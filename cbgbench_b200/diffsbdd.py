"""CUDA (H100) drop-in for the reference's ``DiffSBDD`` model, sampling path (SURVEY.md section 8 row f2).

Mirrors /root/reference repo/models/diffusion/diffsbdd.py:25-46 (constructor, sub-module names => state-dict
keys) and :240-360 (``sample(batch) -> traj``, ``sample_p_xh_given_z0``).  Same denoiser kernels as TargetDiff;
what differs is the reverse step: a variational gamma schedule (``sample_p_zs_given_zt``) applied to the
coordinates AND to continuous type features, with a centre-of-mass projection that also translates the pocket.
One C-ABI call per step (``cbg_sbdd_step_f32``): ligand embedding -> kNN -> edge gate -> 9 x (X2H, H2X) ->
classifier -> fused reverse step + COM projection + pocket shift.

Because the pocket coordinates change every step, the step-invariant R-cache / static neighbour lists of the
TargetDiff path do not apply (distances are translation invariant, their fp32 roundings are not); receptive-field
pruning still does.

Reference quirks reproduced (oracle/diffusion_sbdd.py lists them): the denoiser's output COORDINATES act as eps;
the final ``c_lig`` is 4 x the last state, not the freshly sampled one; gen_flag is ignored by the reverse step.
Random numbers: ``torch.randn`` on the model device in the reference's order (x then c: init, every step, final
stage), or injected through ``noise`` for parity tests.

The eval-mode ``forward(batch)`` (diffsbdd.py:48-191, the validation loss) noises every timestep twice, at t and at 0,
and runs all these copies through ONE C-ABI call (``cbg_sbdd_eval_loss_f32``, DESIGN.md section 15).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .schedulers import DiffsbddVariationalTables
from . import targetdiff
from .targetdiff import BaseDiffB200, register_model

TYPE_NORM = 4.0      # normalize_type / unnormalize_type (diffsbdd.py:95-96, 210-211)
EVAL_NOISE_KEYS = ('x_t', 'c_t', 'x_0', 'c_0')     # the four draws of one eval timestep, in the reference's order


def eval_t_values(num_timesteps, eval_interval=10):
    """Timesteps of DiffSBDD's eval-mode forward (diffsbdd.py:71-77): ``targetdiff.eval_t_values`` from first = 1, i.e.
    ``np.linspace(1, T, eval_interval)`` truncated.  T = 1000 gives [1, 112, 223, ..., 889, 1000]: t = T is included."""
    return targetdiff.eval_t_values(num_timesteps, eval_interval, first=1)


@register_model('diffsbdd')
class DiffSBDDB200(BaseDiffB200):
    allow_rcache = False
    eval_t_first = 1         # the eval timesteps are np.linspace(1, T, eval_interval) (diffsbdd.py:71-77)

    def __init__(self, cfg):
        super().__init__(cfg)
        gen = cfg.generator
        self.pos_scheduler = DiffsbddVariationalTables(self.num_diffusion_timesteps, type=gen.pos_schedule.type)
        self.type_scheduler = DiffsbddVariationalTables(self.num_diffusion_timesteps, type=gen.atom_schedule.type)
        self._build_networks(cfg)
        self.intersect_reg = cfg.get('intersect_reg', True) if hasattr(cfg, 'get') else True

    # ---- validation loss (DiffSBDD.forward with self.training == False, diffsbdd.py:48-191) --------------------------
    def eval_coef(self, t):
        """Host scalars of timestep t (integer in [1, T]) with the reference's fp32 torch expressions: s = (t - 1) / T and
        t / T as in get_loss, gamma at 0 (t_zeros) and at 1 (kl_prior's ones)."""
        T = self.num_diffusion_timesteps
        tt = torch.tensor([t], dtype=torch.int64)
        alpha = lambda g: torch.sqrt(torch.sigmoid(-g))
        sigma = lambda g: torch.sqrt(torch.sigmoid(g))
        v = {}
        for pre, tab in (('pos', self.pos_scheduler), ('type', self.type_scheduler)):
            g_s, g_t, g_0, g_T = (tab.gamma_at(x) for x in ((tt - 1) / T, tt / T, torch.zeros(1), torch.ones(1)))
            s_T = sigma(g_T)
            v.update({f'{pre}_alpha_t': alpha(g_t), f'{pre}_sigma_t': sigma(g_t),
                      f'{pre}_alpha_0': alpha(g_0), f'{pre}_sigma_0': sigma(g_0),
                      f'{pre}_t_weight': -T * 0.5 * (1 - torch.exp(-(g_s - g_t))),               # :883-887
                      f'{pre}_log_const': -(0.5 * g_0) - 0.5 * np.log(2 * np.pi),               # :680-692
                      f'{pre}_alpha_T': alpha(g_T),
                      f'{pre}_log_inv_sigma_T': torch.log(torch.ones_like(s_T) / s_T),          # gaussian_KL, :695-704
                      f'{pre}_sigma2_T': s_T ** 2})
        return _lib.SbddEvalCoef(**{k: float(x[0]) for k, x in v.items()})

    @torch.no_grad()
    def eval_losses(self, batch, t_values, noise=None, max_nodes=None):
        """Validation losses of ``batch`` at the timesteps ``t_values`` (integers in [1, T]; DiffSBDD.get_loss in eval
        mode, diffsbdd.py:87-191, once per t).  Returns ``(loss_dict, results)`` like the reference's eval-mode forward:
        ``loss_dict`` = {'pos', 'atom'} as CPU 0-d float32 tensors (mean over t of the per-t losses), ``results`` one
        dict per t with the device tensors eps_0_pos (the position draw at t), eps_pred_pos (the denoiser's output
        coordinates), score_0_pos, score_pred_pos (both times sigma_t), mask_gen_pos (the generation flag), and the same
        five ``_atom`` keys of the types (eps_pred_atom = the classifier's logits).  ``last_terms`` then holds the
        per-graph terms [n_t, B, 6] (pos_t, pos_0, pos_kl, atom_t, atom_0, atom_kl; B = last ligand graph id + 1).

        Each t is noised twice, at t and at 0.  The denoiser is not conditioned on t, so the 2 R copies go through ONE
        denoiser pass as 2 R * B graphs, split over several launches above ``max_nodes`` composed nodes (default
        ``eval_max_nodes``, a timestep counting twice) or 32 timesteps; the split does not change any result bit.

        ``noise`` = {'x_t', 'c_t', 'x_0', 'c_0'} of [R, n_lig, 3 | K] injects the draws; by default they are drawn with
        torch on the model device in the reference's order (for each t: randn [n_lig,3], [n_lig,K], [n_lig,3],
        [n_lig,K])."""
        t_values = self._eval_t_values(t_values)
        R, K = len(t_values), self.num_classes
        dev, b, n_graphs, x0, v0, gen = self._eval_batch(batch)
        x_rec = b['protein_pos'].float().contiguous()
        n_lig = x0.shape[0]
        dims = {'x_t': 3, 'c_t': K, 'x_0': 3, 'c_0': K}
        if noise is None:
            draws = [[torch.randn(n_lig, dims[k], device=dev) for k in EVAL_NOISE_KEYS] for _ in range(R)]
            noise = {k: torch.stack([d[i] for d in draws]) for i, k in enumerate(EVAL_NOISE_KEYS)}
        noise = {k: noise[k].to(dev, torch.float32).reshape(R, n_lig, dims[k]).contiguous() for k in EVAL_NOISE_KEYS}

        vec_pos = torch.empty(R, 3, n_lig, 3, device=dev)
        vec_atom = torch.empty(R, 3, n_lig, K, device=dev)
        terms = torch.empty(R, n_graphs, 6, device=dev)
        t_loss = torch.empty(R, 2, device=dev)
        L = _lib.lib()

        def launch(r0, r1, state, coefs):
            _lib.check(L.cbg_sbdd_eval_loss_f32(
                C.byref(state['plan']), coefs, r1 - r0, x0.data_ptr(), v0.data_ptr(), x_rec.data_ptr() if x_rec.numel() else None,
                *[noise[k][r0:r1].data_ptr() for k in EVAL_NOISE_KEYS], vec_pos[r0:r1].data_ptr(),
                vec_atom[r0:r1].data_ptr(), terms[r0:r1].data_ptr(), t_loss[r0:r1].data_ptr(), _lib.stream_ptr(dev)))
        self._eval_plans(b, n_graphs, t_values, _lib.SbddEvalCoef, max_nodes, launch, copies=2,
                         protein_feature_scale=TYPE_NORM)
        self.last_terms = terms[:, :int(b['ligand_element_batch'].max()) + 1]
        loss_dict = self._eval_dict_mean(t_loss, ('pos', 'atom'))
        # the reference's key order: pos_info, then atom_info (get_score_loss, diffusion_scheduler.py:944-961)
        results = [{'eps_0_pos': noise['x_t'][r], 'eps_pred_pos': vec_pos[r, 0], 'score_0_pos': vec_pos[r, 1],
                    'score_pred_pos': vec_pos[r, 2], 'mask_gen_pos': gen,
                    'eps_0_atom': noise['c_t'][r], 'eps_pred_atom': vec_atom[r, 0], 'score_0_atom': vec_atom[r, 1],
                    'score_pred_atom': vec_atom[r, 2], 'mask_gen_atom': gen} for r in range(R)]
        return loss_dict, results

    @staticmethod
    def _segment_mean(x, idx, n):
        """scatter_mean(x, idx, dim=0, dim_size=n) for the one-time initialisation (tensor plumbing, once per
        batch).  Deterministic: rows are laid out in a dense [n, max_count, D] block and summed along axis 1
        (index_add_ on CUDA uses atomics, whose order - and so the rounding - changes from run to run)."""
        order = torch.sort(idx, stable=True).indices
        sid = idx[order]
        cnt = torch.bincount(sid, minlength=n)
        start = torch.cumsum(cnt, 0) - cnt
        pos = torch.arange(sid.numel(), device=x.device) - start[sid]
        dense = torch.zeros((n, int(cnt.max()) if sid.numel() else 1, x.shape[1]), dtype=x.dtype, device=x.device)
        dense[sid, pos] = x[order]
        return dense.sum(1) / cnt.clamp(min=1).to(x.dtype).unsqueeze(-1)

    @torch.no_grad()
    def begin(self, batch, noise=None):
        """Initial state (diffsbdd.py:255-262) + device plan.  Ligand ~ N(pocket mean, I) projected to zero ligand
        COM - the projection translates the pocket as well; type features ~ N(0, I).  Returns the state dict of
        ``prepare`` plus the trajectory buffers X [T+1,n_lig,3] / C [T+1,n_lig,K] (slot t+1 = state entering step t)."""
        K = self.num_classes
        dev = next(self.parameters()).device
        if dev.type != 'cuda':
            raise RuntimeError('DiffSBDDB200.sample needs the model on a CUDA device (no CPU fallback)')
        to = lambda t: t.to(dev, torch.float32).contiguous()
        bl = batch['ligand_element_batch'].to(dev).long()
        br = batch['protein_element_batch'].to(dev).long()
        n_lig = int(bl.numel())
        B = max(int(bl.max()) + 1 if n_lig else 0, int(br.max()) + 1 if br.numel() else 0)
        x_rec = batch['protein_pos'].to(dev).float()
        eps_x = to(noise['init_x']) if noise is not None else torch.randn((n_lig, 3), device=dev)
        eps_c = to(noise['init_c']) if noise is not None else torch.randn((n_lig, K), device=dev)
        x_lig = self._segment_mean(x_rec, br, B)[bl] + eps_x
        mean = self._segment_mean(x_lig, bl, B)
        x_lig = (x_lig - mean[bl]).contiguous()
        x_rec = x_rec - mean[br]
        state = self.prepare(batch, device=dev, protein_feature_scale=TYPE_NORM, protein_pos=x_rec)
        state['X'], state['C'] = self._traj_buffers(dev, (x_lig, eps_c))
        return state

    @torch.no_grad()
    def run_steps(self, state, t_seq, noise=None):
        """Enqueue the reverse steps ``t_seq`` (descending t): one ``cbg_sbdd_step_f32`` call each."""
        self.check_state(state)
        K, dev, n_lig, plan = self.num_classes, state['device'], state['n_lig'], state['plan']
        X, Cc = state['X'], state['C']
        to = lambda t: t.to(dev, torch.float32).contiguous()
        L = _lib.lib()
        st = _lib.stream_ptr(dev)
        launches0 = L.cbg_launch_count()
        with torch.cuda.device(dev):
            for t_idx in t_seq:
                x_t, c_t = X[t_idx + 1], Cc[t_idx + 1]
                nx = to(noise['step_x'][t_idx]) if noise is not None else torch.randn((n_lig, 3), device=dev)
                nc = to(noise['step_c'][t_idx]) if noise is not None else torch.randn((n_lig, K), device=dev)
                a, b, s = self.pos_scheduler.step_scalars(t_idx)
                coef = _lib.SbddCoef(a=a, b=b, s=s, mode=0)
                _lib.check(L.cbg_sbdd_step_f32(C.byref(plan), C.byref(coef), x_t.data_ptr(), c_t.data_ptr(),
                                               nx.data_ptr(), nc.data_ptr(), X[t_idx].data_ptr(),
                                               Cc[t_idx].data_ptr(), None, None, st))
        self.last_launches = L.cbg_launch_count() - launches0

    @torch.no_grad()
    def finish(self, state, noise=None):
        """sample_p_xh_given_z0 (diffsbdd.py:323-352): one more denoiser pass at t = 0 -> (x_lig, 4 * c_lig)."""
        self.check_state(state)
        K, dev, n_lig, plan = self.num_classes, state['device'], state['n_lig'], state['plan']
        X, Cc = state['X'], state['C']
        to = lambda t: t.to(dev, torch.float32).contiguous()
        L = _lib.lib()
        with torch.cuda.device(dev):
            nx = to(noise['final_x']) if noise is not None else torch.randn((n_lig, 3), device=dev)
            nc = to(noise['final_c']) if noise is not None else torch.randn((n_lig, K), device=dev)  # drawn, unused
            a, b, s = self.pos_scheduler.final_scalars()
            coef = _lib.SbddCoef(a=a, b=b, s=s, mode=1)
            x_fin = torch.empty((n_lig, 3), dtype=torch.float32, device=dev)
            c_fin = torch.empty((n_lig, K), dtype=torch.float32, device=dev)
            _lib.check(L.cbg_sbdd_step_f32(C.byref(plan), C.byref(coef), X[0].data_ptr(), Cc[0].data_ptr(),
                                           nx.data_ptr(), nc.data_ptr(), x_fin.data_ptr(), c_fin.data_ptr(),
                                           None, None, _lib.stream_ptr(dev)))
        return x_fin, c_fin

    @torch.no_grad()
    def sample(self, batch, noise=None, num_steps=None, traj_mode='full'):
        """DiffSBDD.sample (diffsbdd.py:240-321).

        Returns ``traj``: {t: (x_lig [n_lig,3], c_lig [n_lig,K] continuous, batch_idx_lig)} with keys T-1 ... -1;
        entries >= 0 on the CPU, key -1 on the device, and traj[0] replaced by the final stage
        (x_lig, 4 * c_lig) exactly like the reference (:313-320).

        ``noise`` = {'init_x','init_c','step_x'[t],'step_c'[t],'final_x','final_c'} injects the random numbers;
        ``num_steps`` stops early (testing; the final stage only runs after step t = 0);
        ``traj_mode='final'`` keeps only traj[0] and traj[-1]."""
        T = self.num_diffusion_timesteps
        state = self.begin(batch, noise)
        t_seq = list(reversed(range(T)))
        if num_steps is not None:
            t_seq = t_seq[:num_steps]
        self.run_steps(state, t_seq, noise)
        launches = self.last_launches
        t_last = t_seq[-1]
        x_fin = c_fin = None
        if t_last == 0:
            x_fin, c_fin = self.finish(state, noise)
        self.last_launches = launches
        traj = self._traj((state['X'], state['C']), state['batch_idx_lig'], t_last, traj_mode)
        if x_fin is not None:
            traj[0] = (x_fin.cpu(), c_fin.cpu(), traj[0][2])
        return traj
