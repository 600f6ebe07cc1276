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
"""
import ctypes as C

import torch

from . import _lib
from .schedulers import DiffsbddVariationalTables
from .targetdiff import BaseDiffB200, register_model

TYPE_NORM = 4.0      # normalize_type / unnormalize_type (diffsbdd.py:95-96, 210-211)


@register_model('diffsbdd')
class DiffSBDDB200(BaseDiffB200):
    allow_rcache = False

    def __init__(self, cfg):
        super().__init__(cfg)
        gen = cfg.generator
        self.pos_scheduler = DiffsbddVariationalTables(self.num_diffusion_timesteps, type=gen.pos_schedule.type)
        self.type_scheduler = DiffsbddVariationalTables(self.num_diffusion_timesteps, type=gen.atom_schedule.type)
        self._build_networks(cfg)
        self.intersect_reg = cfg.get('intersect_reg', True) if hasattr(cfg, 'get') else True

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
        state['X'], state['C'] = self._traj_buffers(dev, x_lig, eps_c)
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
        traj = self._traj(state['X'], state['C'], state['batch_idx_lig'], t_last, traj_mode)
        if x_fin is not None:
            traj[0] = (x_fin.cpu(), c_fin.cpu(), traj[0][2])
        return traj
