"""CUDA (H100) drop-in for the reference's ``DiffBP`` model, sampling path (SURVEY.md section 8 row f2).

Mirrors /root/reference repo/models/diffusion/diffbp.py:30-57 (``CoMPredictor`` parameters), :103-130 (constructor,
sub-module names => state-dict keys) and :240-299 (``sample(batch) -> traj``).  Per step ONE C-ABI call
(``cbg_bp_step_f32``): ligand embedding -> kNN -> edge gate -> 9 x (X2H, H2X) -> classifier -> CoM head (its own
gate + 3 x H2X on the final h, from the step's input coordinates) -> fused reverse step (zero-mean noise prediction
+ per-graph CoM shift, score-form VP update, mask-type update).

The pocket is static, so the step-invariant caches of the TargetDiff path (R-cache, static neighbour lists, cached
gates, receptive-field pruning) all apply to the denoiser part unchanged.

Random numbers: ``torch.randn_like`` (positions) then ``torch.rand_like`` over [n_lig] (type change mask) per step,
in the reference's order (diffusion_scheduler.py:158, 486), or injected for parity tests.

The eval-mode ``forward(batch)`` (diffbp.py:133-230, the validation loss) runs the noised copies of the batch for all
its timesteps through ONE C-ABI call (``cbg_bp_eval_loss_f32``, DESIGN.md section 14).
"""
import ctypes as C

import torch
from torch import nn
import torch.nn.functional as F

from . import _lib
from .modules import (GaussianSmearing, H2XAttention, MLP, _NoTorchPath, cfg_get, pack_denoiser_blob)
from .schedulers import CTNVPTables
from .targetdiff import BaseDiffB200, register_model

ABSORBING_STATE = 0      # repo/utils/molecule/constants.py:8


class CoMPredictorB200(_NoTorchPath):
    """Parameter container for CoMPredictor (diffbp.py:30-57)."""

    def __init__(self, cfg):
        super().__init__()
        self.hidden_dim = cfg_get(cfg, 'node_feat_dim', 128)
        self.n_heads = cfg_get(cfg, 'n_heads', 16)
        self.num_r_gaussian = cfg_get(cfg, 'num_r_gaussian', 20)
        self.num_layers = cfg_get(cfg, 'num_layers_com', 3)
        if cfg_get(cfg, 'ew_type', 'global') != 'global' or cfg_get(cfg, 'cutoff_mode', 'knn') != 'knn':
            raise NotImplementedError("CoMPredictorB200 needs ew_type == 'global' and cutoff_mode == 'knn' "
                                      "(the reference's radius branch is broken, diffbp.py:60)")
        self.h2xattentions = nn.ModuleList([H2XAttention(self.hidden_dim, self.n_heads, cfg_get(cfg, 'edge_feat_dim', 4),
                                                         self.num_r_gaussian) for _ in range(self.num_layers)])
        self.dist_emb = nn.Sequential(GaussianSmearing(self.num_r_gaussian),
                                      MLP(self.num_r_gaussian, 1, self.num_r_gaussian * 8))
        self._blob = None
        self._blob_key = None

    def packed_blob(self, device):
        key = (str(device),) + tuple((t.data_ptr(), t._version) for t in self.state_dict(keep_vars=True).values())
        if self._blob is None or key != self._blob_key:
            self._blob = pack_denoiser_blob(dict(self.state_dict()), '', self.num_layers, 1, com_head=True).to(device)
            self._blob_key = key
        return self._blob


class MaskTypeScheduleB200(nn.Module):
    """MaskTypeSchedule (diffusion_scheduler.py:444-450): no parameters, only the change probability of a step."""

    def __init__(self, num_timestep, num_classes, absorbing_state, type='uniform'):
        super().__init__()
        self.num_timestep, self.num_classes = num_timestep, num_classes
        self.absorbing_state, self.schedule_type = absorbing_state, type
        if absorbing_state != 0:
            raise NotImplementedError('the fused reverse step assumes absorbing_state == 0 (constants.py:8)')

    def change_prob(self, t_idx):
        """((T - t) / T).clamp(0, 1) in fp32 like diffusion_scheduler.py:482-484."""
        t = torch.tensor([t_idx], dtype=torch.long)
        return float(((self.num_timestep - t) / self.num_timestep).clamp(max=1., min=0.)[0])


@register_model('diffbp')
class DiffBPB200(BaseDiffB200):
    def __init__(self, cfg):
        super().__init__(cfg)
        gen = cfg.generator
        ps = gen.pos_schedule
        self.pos_scheduler = CTNVPTables(self.num_diffusion_timesteps, beta_start=ps.beta_start,
                                         beta_end=ps.beta_end, type=ps.type)
        self.type_scheduler = MaskTypeScheduleB200(self.num_diffusion_timesteps, num_classes=self.num_classes,
                                                   type=gen.atom_schedule.type, absorbing_state=ABSORBING_STATE)
        self._build_networks(cfg)
        if cfg_get(cfg.encoder, 'cutoff_mode', 'knn') != 'knn':
            raise NotImplementedError('DiffBPB200: the CoM head shares the kNN graph of the denoiser')
        self.com_head = CoMPredictorB200(cfg.encoder)
        self.intersect_reg = cfg.get('intersect_reg', True) if hasattr(cfg, 'get') else True

    def step_coef(self, t_idx):
        ps = self.pos_scheduler
        return _lib.BpCoef(alpha_cumprod=float(ps.host_table('alphas_cumprod')[t_idx]),
                           beta=float(ps.host_table('betas')[t_idx]),
                           nonzero=0.0 if t_idx == 0 else 1.0,
                           change_prob=self.type_scheduler.change_prob(t_idx))

    # ---- validation loss (DiffBP.forward with self.training == False, diffbp.py:133-171) ---------------------------
    def eval_coef(self, t_idx):
        ps = self.pos_scheduler
        mask_prob = torch.tensor([t_idx]).float().clamp(min=0.) / self.num_diffusion_timesteps    # fp32, like :462-466
        return _lib.BpEvalCoef(alphas_cumprod=float(ps.host_table('alphas_cumprod')[t_idx]),
                               beta=float(ps.host_table('betas')[t_idx]), mask_prob=float(mask_prob[0]))

    @torch.no_grad()
    def eval_losses(self, batch, t_values, pos_noise=None, type_uniform=None, max_nodes=None):
        """Validation losses of ``batch`` at the timesteps ``t_values`` (DiffBP.get_loss, diffbp.py:173-230, once per t).
        Returns ``(loss_dict, results)`` like the reference's eval-mode forward: ``loss_dict`` = {'pos', 'atom', 'com',
        'inter'} as CPU 0-d float32 tensors (mean over t of the per-t losses), ``results`` one dict per t with the device
        tensors eps_0, eps_pred, score_0, score_pred, mask_gen (the type mask), v0, vt (one-hot float), c_pred, and
        eps_0_com, eps_pred_com, score_0_com, score_pred_com, mask_gen_com (the generation flag).  A t whose batch has no
        generated atom gets NaN pos / com losses; a t without masked atoms (every t = 0) an atom loss of 0, like the
        reference.  ``last_rep_loss`` then holds the per-t losses [R, 4] in the order pos, atom, com, inter.

        The denoiser is not conditioned on t, so the R = len(t_values) noised copies go through ONE denoiser pass as
        R*B graphs, split over several launches above ``max_nodes`` composed nodes (default ``eval_max_nodes``) or 64
        replicas; the split does not change any result bit.

        ``pos_noise`` [R,n_lig,3] / ``type_uniform`` [R,n_lig] inject the draws; by default they are drawn with torch on
        the model device in the reference's order (for each t: randn [n_lig,3], then rand [n_lig])."""
        if not self.intersect_reg:
            raise NotImplementedError('intersect_reg: False is not supported: the reference\'s DiffBP.get_loss reads the '
                                      'interior loss unconditionally (diffbp.py:222-226) and raises UnboundLocalError')
        t_values = self._eval_t_values(t_values)
        R, K = len(t_values), self.num_classes
        dev, b, n_graphs, x0, v0, gen = self._eval_batch(batch)
        if 'protein_gen_flag' in b and bool(b['protein_gen_flag'].any()):
            raise NotImplementedError('the interior loss reads the pocket at its input coordinates: protein_gen_flag '
                                      'must be all False')
        n_lig = x0.shape[0]
        pos_noise, type_uniform = self._eval_noise(R, dev, pos_noise, type_uniform, (n_lig,))

        com_blob = self.com_head.packed_blob(dev)
        xt = torch.empty(R, n_lig, 3, device=dev)
        vt = torch.empty(R, n_lig, dtype=torch.int64, device=dev)
        mask = torch.empty(R, n_lig, dtype=torch.uint8, device=dev)
        vec = torch.empty(R, 8, n_lig, 3, device=dev)
        c_pred = torch.empty(R, n_lig, K, device=dev)
        rep_loss = torch.empty(R, 4, device=dev)
        L = _lib.lib()

        def launch(r0, r1, state, coefs):
            _lib.check(L.cbg_bp_eval_loss_f32(
                C.byref(state['plan']), com_blob.data_ptr(), self.com_head.num_layers, coefs, r1 - r0, x0.data_ptr(),
                v0.data_ptr(), pos_noise[r0:r1].data_ptr(), type_uniform[r0:r1].data_ptr(), xt[r0:r1].data_ptr(),
                vt[r0:r1].data_ptr(), mask[r0:r1].data_ptr(), vec[r0:r1].data_ptr(), c_pred[r0:r1].data_ptr(),
                rep_loss[r0:r1].data_ptr(), _lib.stream_ptr(dev)))
        self._eval_plans(b, n_graphs, t_values, _lib.BpEvalCoef, max_nodes, launch)
        self.last_rep_loss = rep_loss
        loss_dict = self._eval_dict_mean(rep_loss, ('pos', 'atom', 'com', 'inter'))
        vt_onehot = F.one_hot(vt, K).float()
        # the reference's key order: pos_info, then atom_info (its mask_gen, the type mask, replaces gen), then com_info
        results = [{'eps_0': vec[r, 0], 'eps_pred': vec[r, 1], 'score_0': vec[r, 2], 'score_pred': vec[r, 3],
                    'mask_gen': mask[r].bool(), 'v0': v0, 'vt': vt_onehot[r], 'c_pred': c_pred[r],
                    'eps_0_com': vec[r, 4], 'eps_pred_com': vec[r, 5], 'score_0_com': vec[r, 6],
                    'score_pred_com': vec[r, 7], 'mask_gen_com': gen} for r in range(R)]
        return loss_dict, results

    @torch.no_grad()
    def run_steps(self, state, t_seq, X, Cc, pos_noise=None, type_uniform=None, eps_out=None):
        """Enqueue the reverse steps ``t_seq`` (descending t): one ``cbg_bp_step_f32`` call each.  X / Cc as in
        TargetDiffB200.run_steps (slot t+1 = state entering step t, slot t = its result)."""
        self.check_state(state)
        dev, n_lig, plan = state['device'], state['n_lig'], state['plan']
        com_blob = self.com_head.packed_blob(dev)
        v_scratch = torch.empty(n_lig, dtype=torch.int64, device=dev)
        L = _lib.lib()
        st = _lib.stream_ptr(dev)
        launches0 = L.cbg_launch_count()
        with torch.cuda.device(dev):
            for t_idx in t_seq:
                x_t, c_t = X[t_idx + 1], Cc[t_idx + 1]
                eps = torch.randn_like(x_t) if pos_noise is None else pos_noise[t_idx].to(dev, torch.float32).contiguous()
                uni = (torch.rand((n_lig,), device=dev) if type_uniform is None
                       else type_uniform[t_idx].to(dev, torch.float32).contiguous())
                e_buf = None
                if eps_out is not None:
                    e_buf = eps_out[t_idx] = torch.empty((n_lig, 3), dtype=torch.float32, device=dev)
                coef = self.step_coef(t_idx)
                _lib.check(L.cbg_bp_step_f32(C.byref(plan), com_blob.data_ptr(), self.com_head.num_layers, C.byref(coef),
                                             x_t.data_ptr(), c_t.data_ptr(), eps.data_ptr(), uni.data_ptr(),
                                             X[t_idx].data_ptr(), Cc[t_idx].data_ptr(), v_scratch.data_ptr(),
                                             e_buf.data_ptr() if e_buf is not None else None, None, st))
        self.last_launches = L.cbg_launch_count() - launches0

    @torch.no_grad()
    def sample(self, batch, pos_noise=None, type_uniform=None, num_steps=None, traj_mode='full', eps_out=None):
        """DiffBP.sample (diffbp.py:240-299).  Returns ``traj``: {t: (x_lig, c_lig one-hot, batch_idx_lig)}, keys
        T-1 ... -1, entries >= 0 on the CPU and key -1 on the device like the reference.

        ``pos_noise[t]`` [n_lig,3] / ``type_uniform[t]`` [n_lig] inject the random numbers; ``num_steps`` stops early;
        ``traj_mode='final'`` keeps only traj[0] and traj[-1]; ``eps_out`` (dict) receives eps + eps_com per step."""
        T = self.num_diffusion_timesteps
        state = self.prepare(batch)
        X, Cc = self._traj_buffers(state['device'], (state['x_lig'], state['c_lig']))
        t_seq = list(reversed(range(T)))
        if num_steps is not None:
            t_seq = t_seq[:num_steps]
        self.run_steps(state, t_seq, X, Cc, pos_noise, type_uniform, eps_out)
        return self._traj((X, Cc), state['batch_idx_lig'], t_seq[-1], traj_mode)
