"""CUDA (H100) drop-in for the reference's ``TargetDiff`` model (sampling path).

Mirrors the reference's repo/models/diffusion/targetdiff.py:14-38 (constructor, sub-module
names => state-dict keys) and :127-184 (``sample(batch) -> traj``).  The Python loop over the
T diffusion steps stays here (north-star: host code keeps the outer schedule); each iteration
is ONE C-ABI call (``cbg_sample_step_f32``) that enqueues: ligand embedding -> device kNN ->
edge gate -> 9 x (node GEMMs, fused X2H, fused H2X) -> classifier -> fused reverse step.
Step-invariant work is hoisted out of the loop (SURVEY.md Appendix B): protein embedding,
the compose_context permutation, graph offsets, flag arrays.

Random numbers are drawn with torch on the model device in the reference's order
(positions ``randn_like`` then types ``rand_like``, diffusion_scheduler.py:158-163 /
categorical.py:27), or injected for parity tests.

The eval-mode ``forward(batch)`` (targetdiff.py:41-124, the validation loss) is built too: ``eval_losses`` runs the
noised copies of the batch for all its timesteps through ONE C-ABI call (``cbg_eval_loss_f32``, DESIGN.md section 13).
"""
import ctypes as C
import os

import numpy as np
import torch
from torch import nn
import torch.nn.functional as F

from . import _lib
from .modules import cfg_get, get_e3_gnn, graph_ptr_from_batch, _Workspace
from .schedulers import CTNVPTables, TypeVPTables

N_AA_TYPES = 20        # repo/utils/protein/constants.py:39-41
N_PROTEIN_ATOM_FEAT = 7  # 6 elements + backbone flag, repo/utils/protein/constants.py:37

_MODEL_DICT = {}


def register_model(name):
    def deco(cls):
        _MODEL_DICT[name] = cls
        return cls
    return deco


def get_model(config):
    """Mirror of repo/models/_base.py:10-12."""
    return _MODEL_DICT[config.type](config)


def eval_t_values(num_timesteps, eval_interval=10, first=0):
    """Timesteps of the reference's eval-mode forwards: ``np.linspace(first, T - 1 + first, eval_interval)``, each
    truncated toward zero by ``torch.tensor([t] * B).long()``.  TargetDiff and DiffBP (targetdiff.py:67-71) start at
    first = 0: T = 50 gives [0, 5, 10, 16, 21, 27, 32, 38, 43, 49].  DiffSBDD (diffsbdd.py:71-77) starts at first = 1,
    i.e. ``np.linspace(1, T, eval_interval)``: T = 1000 gives [1, 112, 223, ..., 889, 1000], t = T included."""
    return [int(t) for t in np.linspace(first, num_timesteps - 1 + first, eval_interval).astype(np.int64)]


def replicate_batch(batch, n_rep, n_graphs):
    """``n_rep`` copies of a batch (dict of tensors) as one batch of n_rep * n_graphs graphs: every tensor is tiled along
    dim 0 and copy r's graph ids are offset by r * n_graphs, so the copies stay replica-major and sorted."""
    out = {}
    for k, t in batch.items():
        if k in ('ligand_element_batch', 'protein_element_batch'):
            off = torch.arange(n_rep, device=t.device, dtype=t.dtype).unsqueeze(1) * n_graphs
            out[k] = (t.unsqueeze(0) + off).reshape(-1)
        else:
            out[k] = t.repeat(n_rep, *([1] * (t.dim() - 1)))
    return out


class PLContextEmbedderB200(nn.Module):
    """Parameter container for PLContextEmbedder (context_emb.py:137-177), 'linear' embeddings,
    no time embedding (the only shipped configuration, SURVEY.md A7)."""

    def __init__(self, cfg):
        super().__init__()
        self.num_classes = cfg_get(cfg, 'num_atomtype', 14)
        emb_dim = cfg_get(cfg, 'emb_dim', 128)
        self.emb_dim = emb_dim
        if cfg_get(cfg, 'time', None) is not None or cfg_get(cfg, 'vec', None) is not None:
            # Not only unused by every shipped config: the reference's own time path cannot run.  PLContextEmbedder passes
            # t as [N, 1] (context_emb.py:184-185) into SinusoidalPosEmb, whose x[:, None] (common.py:146) makes the
            # embedding [N, 1, 128]; "h_lig + t_emb_lig" (context_emb.py:224) then broadcasts h to [N, N, 128] and
            # compose_context raises (common.py:209).  Verified against the live reference (DESIGN.md section 9).
            raise NotImplementedError('time / vec embeddings are not used by any shipped CBGBench config (the reference\'s '
                                      'own time-embedding path raises a shape error) and are not implemented on the CUDA path')
        atom = cfg_get(cfg, 'atom', None)
        res = cfg_get(cfg, 'residue', None)
        if atom is None or res is None or cfg_get(atom, 'type') != 'linear' or cfg_get(res, 'type') != 'linear':
            raise NotImplementedError("embedder needs atom.type == residue.type == 'linear'")
        if emb_dim != 128:
            raise NotImplementedError('emb_dim must be 128')
        self.ligand_atom_emb = nn.Linear(self.num_classes, emb_dim)
        self.protein_atom_emb = nn.Linear(N_PROTEIN_ATOM_FEAT, emb_dim)
        self.residue_emb = nn.Linear(N_AA_TYPES, emb_dim)
        self.ligand_indicator = nn.Linear(1, emb_dim)

    @torch.no_grad()
    def static_features(self, v_rec, aa_rec, lig_flag, rec_flag):
        """Step-invariant pieces (tensor plumbing, executed once per batch):
        h_rec (context_emb.py:210-222) and the c_lig-independent part of h_lig."""
        if aa_rec.dim() == 1:
            aa_rec = F.one_hot(aa_rec, num_classes=N_AA_TYPES).float()
        if v_rec.dim() == 1:
            v_rec = F.one_hot(v_rec.long(), num_classes=N_PROTEIN_ATOM_FEAT).float()
        h_rec = self.protein_atom_emb(v_rec.float()) + self.residue_emb(aa_rec) \
            + self.ligand_indicator(rec_flag.float().unsqueeze(-1))
        h_lig_bias = self.ligand_atom_emb.bias.unsqueeze(0) + self.ligand_indicator(lig_flag.float().unsqueeze(-1))
        return h_rec, h_lig_bias.contiguous()


class DiffusionB200(nn.Module):
    """What every CUDA diffusion model shares, whatever its network: the trajectory buffers of ``sample`` and the
    eval-mode ``forward`` (validation losses of replica batches, DESIGN.md section 13).  A subclass provides
    ``num_diffusion_timesteps``, ``cfg``, ``eval_coef(t)`` and ``eval_losses(batch, t_values, *draws, **kw)``."""

    eval_t_first = 0            # first eval timestep of ``eval_t_values``: 0, or 1 for DiffSBDD
    # composed nodes per validation-loss launch: about 9 GB of workspace at ~8.5 KB/node for the denoiser, 8 GB at
    # ~7.6 KB/node for the D3FG encoder at H = 256
    eval_max_nodes = 1 << 20

    # ---- the trajectory of ``sample`` ----------------------------------------------------------------------------
    def _traj_buffers(self, dev, init):
        """One device trajectory [T+1, *v.shape] per initial state tensor v of the tuple ``init`` (x [n_lig,3], c
        [n_lig,K], ...): slot t+1 is the state entering step t, slot t its result; slot T holds the initial state."""
        T = self.num_diffusion_timesteps
        bufs = tuple(torch.empty((T + 1, *v.shape), dtype=torch.float32, device=dev) for v in init)
        for b, v in zip(bufs, init):
            b[T].copy_(v)
        return bufs

    def _traj(self, bufs, bl, t_last, traj_mode):
        """``traj`` of the reference's sample: {t: (*states, batch_idx_lig)} for t = T-1 ... t_last (on the CPU, one
        copy; only t_last when ``traj_mode`` is not 'full') and t_last - 1 (on the device)."""
        T = self.num_diffusion_timesteps
        hi = T if traj_mode == 'full' else t_last + 1
        host = [b[t_last + 1:hi + 1].cpu() for b in bufs]
        bl_cpu = bl.cpu()
        traj = {t: (*(h[t - t_last] for h in host), bl_cpu) for t in range(t_last, hi)}
        traj[t_last - 1] = (*(b[t_last].clone() for b in bufs), bl)
        return traj

    # ---- validation losses: what the eval-mode forwards share (replica batching, DESIGN.md section 13) --------------
    def forward(self, batch, *draws, **kw):
        """The reference's forward in eval mode: ``(loss_dict, results)`` of ``eval_losses`` for the ``eval_interval``
        (default 10) timesteps ``eval_t_values(T, eval_interval, first=eval_t_first)``, exactly like the reference.
        Training mode needs autograd through the network and raises; ``eval_losses`` refuses a model on the CPU."""
        self._check_eval_mode()
        t_values = eval_t_values(self.num_diffusion_timesteps, cfg_get(self.cfg, 'eval_interval', 10),
                                 first=self.eval_t_first)
        return self.eval_losses(batch, t_values, *draws, **kw)

    def _check_eval_mode(self):
        if self.training:
            raise NotImplementedError(f'{type(self).__name__}.forward in training mode needs autograd through the '
                                      'network, which the CUDA path does not provide: training is out of scope '
                                      '(call model.eval() for the validation losses)')

    def _eval_device(self):
        """The model's device, which must be a CUDA device."""
        dev = next(self.parameters()).device
        if dev.type != 'cuda':
            raise NotImplementedError(f'{type(self).__name__}.forward needs the model on a CUDA device: on the CPU '
                                      f'{type(self).__name__} is a sampling build without a validation-loss implementation')
        return dev

    def _eval_t_values(self, t_values):
        """``t_values`` as ints, each in [eval_t_first, T - 1 + eval_t_first]."""
        t_values = [int(t) for t in t_values]
        lo, hi = self.eval_t_first, self.num_diffusion_timesteps - 1 + self.eval_t_first
        if not t_values:
            raise ValueError('t_values is empty')
        if any(t < lo or t > hi for t in t_values):
            raise ValueError(f't_values must lie in [{lo}, {hi}]')
        return t_values

    def _eval_loop(self, n_nodes, t_values, coef_type, max_nodes, launch, make_state, copies=1):
        """Run the timesteps ``t_values`` of a batch of ``n_nodes`` composed nodes in plans of at most 64 replicas and
        ``max_nodes`` composed nodes (default ``eval_max_nodes``): each plan holds timesteps r0 .. r1-1, ``copies``
        noised copies each, and is ``make_state(n_rep)`` with n_rep = (r1 - r0) * copies.  ``launch(r0, r1, state,
        coefs)`` makes the plan's C call, with ``coefs`` the ctypes array of ``eval_coef`` over t_values[r0:r1], on the
        plan's device.  ``last_launches`` counts the kernels of all plans."""
        budget = self.eval_max_nodes if max_nodes is None else int(max_nodes)
        per_launch = max(1, min(_lib.EVAL_MAX_REPLICAS // copies, budget // (copies * n_nodes)))
        L = _lib.lib()
        launches0 = L.cbg_launch_count()
        for r0 in range(0, len(t_values), per_launch):
            r1 = min(len(t_values), r0 + per_launch)
            state = make_state((r1 - r0) * copies)
            coefs = (coef_type * (r1 - r0))(*[self.eval_coef(t) for t in t_values[r0:r1]])
            with torch.cuda.device(state['device']):
                launch(r0, r1, state, coefs)
        self.last_launches = L.cbg_launch_count() - launches0

    @staticmethod
    def _eval_dict_mean(per_t, keys):
        """get_dict_mean (common.py:33-42) of the per-t losses [R, len(keys)]: for each key the mean over t of its column,
        as a CPU float32 0-d tensor."""
        per_t = per_t.cpu()
        return {k: torch.mean(torch.tensor(per_t[:, i].tolist())) for i, k in enumerate(keys)}


class BaseDiffB200(DiffusionB200):
    """What the samplers built on the denoiser share (mirror of repo/models/diffusion/_base.py:4-11 plus the
    hoisting of everything step-invariant): generator flags, context embedder, denoiser, device workspaces and
    ``prepare`` (batch -> device plan)."""

    allow_rcache = True      # samplers whose pocket atoms move between steps (DiffSBDD) turn the R-cache off

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        gen = cfg.generator
        self.num_diffusion_timesteps = gen.num_diffusion_timesteps
        self.denoise_structure = cfg_get(gen, 'denoise_structure', True)
        self.denoise_atom = cfg_get(gen, 'denoise_atom', True)
        self.time_sampler = cfg_get(gen, 'time_sampler', 'symmetric')
        if not (self.denoise_structure and self.denoise_atom):
            raise NotImplementedError('denoise_structure / denoise_atom = False is not implemented')
        self.num_classes = cfg.num_atomtype
        self._ws = _Workspace()
        self._rc = _Workspace()
        self._plan_generation = 0      # the workspace is shared by every prepare() of this model: newest plan wins
        self.last_launches = 0
        # Static lists: atoms without gen_flag never move, so their static-only neighbour lists / edge gates are built
        # once per batch (incremental kNN, cached gates; exact).  On by default wherever the pocket is static.
        self.use_static_lists = self.allow_rcache and os.environ.get('CBG_STATIC_LISTS', '1') != '0'
        # R-cache (for the fp32 SIMT X2H kernels only): step-invariant first-Linear terms of static edges,
        # computed once per batch and streamed from HBM (2*L*N*16 KB).  The default wgmma kernels recompute these
        # terms on the tensor cores and never read it, so it is off unless CBG_RCACHE=1 / use_rcache=True.
        self.use_rcache = self.allow_rcache and os.environ.get('CBG_RCACHE', '0') == '1'
        # receptive-field pruning of the per-step denoiser (exact for the sampled ligand rows)
        self.use_prune = os.environ.get('CBG_PRUNE', '1') != '0'
        # replay each denoise step from a CUDA graph captured once per batch (TargetDiff; exact)
        self.use_graph = os.environ.get('CBG_GRAPH', '1') != '0'

    def _build_networks(self, cfg):
        """context_embedder + denoiser, registered AFTER the schedulers like the reference constructors do
        (state-dict order: targetdiff.py:22-38, diffsbdd.py:32-44, diffbp.py:111-128)."""
        cfg.embedder.num_atomtype = cfg.num_atomtype
        self.context_embedder = PLContextEmbedderB200(cfg.embedder)
        self.denoiser = get_e3_gnn(cfg.encoder, num_classes=self.num_classes)

    def check_state(self, state):
        """A state returned by ``prepare`` owns the model's (single, grow-only) device workspace until the next
        ``prepare``: using an older state would read coordinates / neighbour lists of another batch, so it raises."""
        if state.get('generation') != self._plan_generation:
            raise RuntimeError('stale sampling state: prepare() was called again on this model (its device workspace now '
                               'belongs to the newer batch); finish one batch before preparing the next, or use a second model')

    # ---- validation losses of the denoiser models ----------------------------------------------------------------
    @staticmethod
    def _eval_noise(R, dev, pos_noise, type_uniform, type_shape):
        """pos_noise [R,n_lig,3] / type_uniform [R,*type_shape] on ``dev``; what is not injected is drawn in the
        reference's order (for each of the R timesteps: randn [n_lig,3], then rand type_shape)."""
        n_lig = type_shape[0]
        if pos_noise is None or type_uniform is None:
            draws = [(torch.randn(n_lig, 3, device=dev), torch.rand(*type_shape, device=dev)) for _ in range(R)]
            pos_noise = torch.stack([d[0] for d in draws]) if pos_noise is None else pos_noise
            type_uniform = torch.stack([d[1] for d in draws]) if type_uniform is None else type_uniform
        pos_noise = pos_noise.to(dev, torch.float32).reshape(R, n_lig, 3).contiguous()
        type_uniform = type_uniform.to(dev, torch.float32).reshape(R, *type_shape).contiguous()
        return pos_noise, type_uniform

    _EVAL_KEYS = ('ligand_pos', 'ligand_atom_type', 'protein_pos', 'protein_atom_feature', 'protein_aa_type',
                  'ligand_lig_flag', 'protein_lig_flag', 'ligand_element_batch', 'protein_element_batch',
                  'ligand_gen_flag', 'protein_gen_flag')

    def _eval_batch(self, batch):
        """(dev, b, n_graphs, x0, v0, gen): the model's CUDA device, the batch's tensors on it (dict or attribute batch),
        its graph count, the clean ligand positions x0 [n_lig,3] float32 and types v0 [n_lig] int64, and its generation
        flags (ligand_lig_flag when the batch has no ligand_gen_flag)."""
        dev = self._eval_device()
        g = lambda k, d=None: batch.get(k, d) if hasattr(batch, 'get') else (batch[k] if k in batch else d)
        b = {k: g(k).to(dev) for k in self._EVAL_KEYS if g(k) is not None}
        if b['ligand_pos'].shape[0] == 0:
            raise ValueError('the batch has no ligand atoms')
        n_graphs = int(torch.cat([b['ligand_element_batch'], b['protein_element_batch']]).max()) + 1
        x0 = b['ligand_pos'].float().contiguous()
        v0 = b['ligand_atom_type'].long().contiguous()
        gen = b['ligand_gen_flag'] if 'ligand_gen_flag' in b else b['ligand_lig_flag']
        return dev, b, n_graphs, x0, v0, gen

    def _eval_plans(self, b, n_graphs, t_values, coef_type, max_nodes, launch, copies=1, **prepare_kw):
        """``_eval_loop`` over plans of ``prepare`` (``prepare_kw`` goes to it) on replicas of the batch ``b`` of
        ``n_graphs`` graphs."""
        self._eval_loop(b['ligand_pos'].shape[0] + b['protein_pos'].shape[0], t_values, coef_type, max_nodes, launch,
                        lambda n_rep: self.prepare(replicate_batch(b, n_rep, n_graphs), **prepare_kw), copies)

    # ---- setup of the step-invariant state ------------------------------------------------
    @torch.no_grad()
    def prepare(self, batch, device=None, protein_feature_scale=None, protein_pos=None):
        """Move the batch to the device and hoist everything that does not change over the
        T steps.  Returns a dict holding device tensors (kept alive) and the ctypes plan.

        ``protein_feature_scale`` divides protein_atom_feature (DiffSBDD's normalize_type) and
        ``protein_pos`` replaces batch['protein_pos'] (DiffSBDD starts from a COM-shifted pocket)."""
        dev = torch.device(device) if device is not None else next(self.parameters()).device
        if dev.type != 'cuda':
            raise RuntimeError(f'{type(self).__name__}.sample needs the model on a CUDA device (no CPU fallback)')
        g = lambda k, d=None: batch.get(k, d) if hasattr(batch, 'get') else (batch[k] if k in batch else d)
        to = lambda t: t.to(dev, non_blocking=True)
        x_lig = to(batch['ligand_pos']).float().contiguous()
        v_lig = to(batch['ligand_atom_type'])
        x_rec = to(batch['protein_pos'] if protein_pos is None else protein_pos).float()
        v_rec = to(batch['protein_atom_feature'])
        if protein_feature_scale is not None:
            v_rec = v_rec.float() / protein_feature_scale
        aa_rec = to(batch['protein_aa_type'])
        lig_flag = to(batch['ligand_lig_flag']).bool()
        rec_flag = to(batch['protein_lig_flag']).bool()
        gl = g('ligand_gen_flag', None)
        gen_lig = to(gl).bool() if gl is not None else lig_flag
        gr = g('protein_gen_flag', None)
        gen_rec = to(gr).bool() if gr is not None else torch.zeros_like(rec_flag)
        bl = to(batch['ligand_element_batch']).long()
        br = to(batch['protein_element_batch']).long()
        n_lig, n_rec = x_lig.shape[0], x_rec.shape[0]
        N = n_lig + n_rec

        # compose_context (common.py:189-214): stable sort of [rec | lig] by graph id
        batch_ctx = torch.cat([br, bl], 0)
        sort_idx = torch.sort(batch_ctx, stable=True).indices
        batch_sorted = batch_ctx[sort_idx]
        inv = torch.empty_like(sort_idx)
        inv[sort_idx] = torch.arange(N, device=dev)
        lig_node = inv[n_rec:].to(torch.int32).contiguous()
        if n_lig > 1 and not bool((lig_node[1:] > lig_node[:-1]).all()):
            raise ValueError('ligand_element_batch must be sorted')
        gptr, B, max_n = graph_ptr_from_batch(batch_sorted)

        h_rec, h_lig_bias = self.context_embedder.static_features(v_rec, aa_rec, lig_flag, rec_flag)
        h_static = torch.cat([h_rec, torch.zeros(n_lig, 128, device=dev)], 0)[sort_idx].contiguous()
        x_nodes = torch.cat([x_rec, x_lig], 0)[sort_idx].contiguous()
        lig_nodes = torch.cat([rec_flag, lig_flag], 0)[sort_idx].to(torch.uint8).contiguous()
        gen_nodes_flag = torch.cat([gen_rec, gen_lig], 0)[sort_idx].to(torch.uint8).contiguous()
        gen_node = torch.nonzero(gen_nodes_flag, as_tuple=False).flatten().to(torch.int32).contiguous()
        n_gen = int(gen_node.numel())
        gen_lig8 = gen_lig.to(torch.uint8).contiguous()
        emb_wt = self.context_embedder.ligand_atom_emb.weight.detach().t().contiguous().float()
        blob = self.denoiser.packed_blob(dev)

        L = _lib.lib()
        ws_bytes = L.cbg_workspace_bytes(N, n_gen)
        ws_ptr, ws_have = self._ws.get(ws_bytes, dev)
        den = self.denoiser
        rc_ptr, rc_bytes = None, 0
        if self.use_rcache and self.allow_rcache:
            rc_bytes = L.cbg_rcache_bytes(N, den.num_layers)
            have = self._rc.buf.numel() if self._rc.buf is not None and self._rc.buf.device == dev else 0
            free_b, _ = torch.cuda.mem_get_info(dev)
            if rc_bytes + 256 > have and rc_bytes > 0.6 * (free_b + have):
                import warnings
                warnings.warn(f'R-cache of {rc_bytes / 2**30:.1f} GiB does not fit ({free_b / 2**30:.1f} GiB free): the legacy X2H '
                              'kernels recompute the static first-Linear terms instead (slower)')
                rc_bytes = 0          # batch too large for the cache on this GPU: fall back to recomputing the terms
            else:
                rc_ptr, rc_bytes = self._rc.get(rc_bytes, dev)
        plan = _lib.SamplePlan(
            blob=blob.data_ptr(), num_layers=den.num_layers, num_classes=self.num_classes,
            emb_wt=emb_wt.data_ptr(), h_lig_bias=h_lig_bias.data_ptr(), h_static=h_static.data_ptr(),
            graph_ptr=gptr.data_ptr(), n_graphs=B, max_graph_nodes=max_n, n_nodes=N,
            lig_node=lig_node.data_ptr(), n_lig=n_lig, gen_lig=gen_lig8.data_ptr(),
            gen_node=gen_node.data_ptr() if n_gen else None, n_gen=n_gen,
            mode=den.mode_id, k=den.cut_off, r_max=den.r_max, workspace=ws_ptr, workspace_bytes=ws_have,
            rcache=rc_ptr, rcache_bytes=rc_bytes, prune=1 if self.use_prune else 0,
            static_lists=1 if (self.use_static_lists and self.allow_rcache) else 0)
        with torch.cuda.device(dev):
            _lib.check(L.cbg_sample_begin_f32(C.byref(plan), x_nodes.data_ptr(), lig_nodes.data_ptr(),
                                              gen_nodes_flag.data_ptr(), _lib.stream_ptr(dev)))
        keep = dict(blob=blob, emb_wt=emb_wt, h_lig_bias=h_lig_bias, h_static=h_static, gptr=gptr,
                    lig_node=lig_node, gen_lig8=gen_lig8, gen_node=gen_node, x_nodes=x_nodes,
                    lig_nodes=lig_nodes, gen_nodes_flag=gen_nodes_flag)
        c_lig = F.one_hot(v_lig, num_classes=self.num_classes).float().contiguous()
        self._plan_generation += 1
        return dict(plan=plan, keep=keep, device=dev, generation=self._plan_generation, x_lig=x_lig, c_lig=c_lig, batch_idx_lig=bl,
                    batch_idx_rec=br, n_lig=n_lig, n_nodes=N, n_graphs=B)


@register_model('targetdiff')
class TargetDiffB200(BaseDiffB200):
    def __init__(self, cfg):
        super().__init__(cfg)
        gen = cfg.generator
        ps = gen.pos_schedule
        self.pos_scheduler = CTNVPTables(self.num_diffusion_timesteps, beta_start=ps.beta_start,
                                         beta_end=ps.beta_end, type=ps.type)
        at = gen.atom_schedule
        self.type_scheduler = TypeVPTables(self.num_diffusion_timesteps, num_classes=self.num_classes,
                                           type=at.type, cosine_s=at.cosine_s)
        self._build_networks(cfg)

    def step_coef(self, t_idx):
        ps, ts = self.pos_scheduler, self.type_scheduler
        tm1 = max(t_idx - 1, 0)
        return _lib.StepCoef(
            pos_c0=float(ps.host_table('posterior_mean_c0_coef')[t_idx]),
            pos_ct=float(ps.host_table('posterior_mean_ct_coef')[t_idx]),
            pos_logvar=float(ps.host_table('posterior_logvar')[t_idx]),
            pos_nonzero=0.0 if t_idx == 0 else 1.0,
            log_alphas_cumprod_prev=float(ts.host_table('log_alphas_cumprod_v')[tm1]),
            log_one_minus_alphas_cumprod_prev=float(ts.host_table('log_one_minus_alphas_cumprod_v')[tm1]),
            log_alpha=float(ts.host_table('log_alphas_v')[t_idx]),
            log_one_minus_alpha=float(ts.host_table('log_one_minus_alphas_v')[t_idx]))

    # ---- validation loss (TargetDiff.forward with self.training == False, targetdiff.py:41-80) ----------------------
    def eval_coef(self, t_idx):
        ps, ts = self.pos_scheduler, self.type_scheduler
        tm1 = max(t_idx - 1, 0)
        tab = ts.host_table
        return _lib.EvalCoef(
            alphas_cumprod=float(ps.host_table('alphas_cumprod')[t_idx]),
            log_alphas_cumprod=float(tab('log_alphas_cumprod_v')[t_idx]),
            log_one_minus_alphas_cumprod=float(tab('log_one_minus_alphas_cumprod_v')[t_idx]),
            log_alphas_cumprod_prev=float(tab('log_alphas_cumprod_v')[tm1]),
            log_one_minus_alphas_cumprod_prev=float(tab('log_one_minus_alphas_cumprod_v')[tm1]),
            log_alpha=float(tab('log_alphas_v')[t_idx]),
            log_one_minus_alpha=float(tab('log_one_minus_alphas_v')[t_idx]),
            t_is_zero=1 if t_idx == 0 else 0)

    @torch.no_grad()
    def eval_losses(self, batch, t_values, pos_noise=None, type_uniform=None, max_nodes=None):
        """Validation losses of ``batch`` at the timesteps ``t_values`` (TargetDiff.get_loss, targetdiff.py:82-124, once
        per t).  Returns ``(loss_dict, results)`` like the reference's eval-mode forward: ``loss_dict`` = {'pos', 'atom'}
        as CPU 0-d float32 tensors (mean over t of the per-t losses), ``results`` one dict per t with the device tensors
        x0, xt, x_pred, mask_gen, v0, vt, c_pred.  A t whose batch has no generated atom gets NaN losses, like the
        reference's mean of an empty tensor.  ``last_graph_loss`` then holds the per-graph position and type losses
        [R, B, 2] (means over each graph's generated atoms, 0 for a graph without one).

        The denoiser is not conditioned on t, so the R = len(t_values) noised copies of the batch go through ONE
        denoiser pass as R*B graphs.  When R copies would exceed ``max_nodes`` composed nodes (default
        ``eval_max_nodes``), or more than 64 replicas are asked for, the replicas are split over several launches; graphs
        are processed independently, so the split does not change any result bit.

        ``pos_noise`` [R,n_lig,3] / ``type_uniform`` [R,n_lig,K] inject the draws; by default they are drawn with torch on
        the model device in the reference's order (for each t: randn [n_lig,3], then rand [n_lig,K])."""
        t_values = self._eval_t_values(t_values)
        R, K = len(t_values), self.num_classes
        dev, b, n_graphs, x0, v0, gen = self._eval_batch(batch)
        mask_gen = gen.bool()
        n_lig = x0.shape[0]
        pos_noise, type_uniform = self._eval_noise(R, dev, pos_noise, type_uniform, (n_lig, K))

        xt = torch.empty(R, n_lig, 3, device=dev)
        vt = torch.empty(R, n_lig, dtype=torch.int64, device=dev)
        x_pred = torch.empty(R, n_lig, 3, device=dev)
        c_pred = torch.empty(R, n_lig, K, device=dev)
        rep_loss = torch.empty(R, 2, device=dev)
        graph_loss = torch.empty(R, n_graphs, 2, device=dev)
        L = _lib.lib()

        def launch(r0, r1, state, coefs):
            _lib.check(L.cbg_eval_loss_f32(
                C.byref(state['plan']), coefs, r1 - r0, x0.data_ptr(), v0.data_ptr(), pos_noise[r0:r1].data_ptr(),
                type_uniform[r0:r1].data_ptr(), xt[r0:r1].data_ptr(), vt[r0:r1].data_ptr(), x_pred[r0:r1].data_ptr(),
                c_pred[r0:r1].data_ptr(), graph_loss[r0:r1].data_ptr(), rep_loss[r0:r1].data_ptr(), _lib.stream_ptr(dev)))
        self._eval_plans(b, n_graphs, t_values, _lib.EvalCoef, max_nodes, launch)
        self.last_graph_loss = graph_loss
        loss_dict = self._eval_dict_mean(rep_loss, ('pos', 'atom'))
        results = [{'x0': x0, 'xt': xt[r], 'x_pred': x_pred[r], 'mask_gen': mask_gen,
                    'v0': v0, 'vt': vt[r], 'c_pred': c_pred[r]} for r in range(R)]
        return loss_dict, results

    @torch.no_grad()
    def run_steps(self, state, t_seq, X, Cc, V=None, pos_noise=None, type_uniform=None,
                  x0_out=None, logits_out=None):
        """Enqueue the denoise steps ``t_seq`` (descending t).  X [T+1,n_lig,3] / Cc [T+1,n_lig,K]
        hold the trajectory on the device: slot t+1 is the state ENTERING step t, slot t its
        result (slot 0 = traj[-1])."""
        self.check_state(state)
        L = _lib.lib()
        dev = state['device']
        plan = state['plan']
        n_lig, K = state['n_lig'], self.num_classes
        st = _lib.stream_ptr(dev)
        v_scratch = V if V is not None else torch.empty(n_lig, dtype=torch.int64, device=dev)
        launches0 = L.cbg_launch_count()
        # CUDA-graph replay of the step (bit-identical; CBG_GRAPH=0 or a debug output request keeps the eager path)
        use_graph = self.use_graph and x0_out is None and logits_out is None
        keep = []
        with torch.cuda.device(dev):
            for t_idx in t_seq:
                x_t, c_t = X[t_idx + 1], Cc[t_idx + 1]
                if pos_noise is None:
                    eps = torch.randn_like(x_t)
                else:
                    eps = pos_noise[t_idx].to(dev, torch.float32).contiguous()
                if type_uniform is None:
                    uni = torch.rand_like(c_t)
                else:
                    uni = type_uniform[t_idx].to(dev, torch.float32).contiguous()
                coef = self.step_coef(t_idx)
                if use_graph:
                    _lib.check(L.cbg_sample_step_graph_f32(
                        C.byref(plan), C.byref(coef), x_t.data_ptr(), c_t.data_ptr(), eps.data_ptr(), uni.data_ptr(),
                        X[t_idx].data_ptr(), Cc[t_idx].data_ptr(), v_scratch.data_ptr(), st))
                    keep.append((eps, uni))          # the graph reads them after this Python iteration is over
                    if len(keep) > 80:
                        keep.pop(0)
                    continue
                _lib.check(L.cbg_sample_step_f32(
                    C.byref(plan), C.byref(coef), x_t.data_ptr(), c_t.data_ptr(), eps.data_ptr(), uni.data_ptr(),
                    X[t_idx].data_ptr(), Cc[t_idx].data_ptr(), v_scratch.data_ptr(),
                    x0_out[t_idx].data_ptr() if x0_out is not None else None,
                    logits_out[t_idx].data_ptr() if logits_out is not None else None, st))
        self.last_launches = L.cbg_launch_count() - launches0

    @torch.no_grad()
    def sample(self, batch, pos_noise=None, type_uniform=None, num_steps=None, traj_mode='full'):
        """TargetDiff.sample (targetdiff.py:127-184).

        Returns ``traj``: {t: (x_lig [n_lig,3], c_lig [n_lig,K] one-hot, batch_idx_lig)} with keys
        T-1 ... -1; entries >= 0 live on the CPU and key -1 on the device, exactly like the
        reference (whose consumer, sample.py:194-201, reads traj[0]).  The per-step D2H +
        sync of the reference (targetdiff.py:182) is replaced by one device-side trajectory
        buffer and a single copy at the end.

        Extras (default = reference behaviour): ``pos_noise`` / ``type_uniform`` inject the noise
        (indexable by t); ``num_steps`` stops after that many steps (testing);
        ``traj_mode='final'`` keeps only traj[0] and traj[-1]."""
        T = self.num_diffusion_timesteps
        state = self.prepare(batch)
        X, Cc = self._traj_buffers(state['device'], (state['x_lig'], state['c_lig']))
        t_seq = list(reversed(range(T)))
        if num_steps is not None:
            t_seq = t_seq[:num_steps]
        self.run_steps(state, t_seq, X, Cc, pos_noise=pos_noise, type_uniform=type_uniform)
        return self._traj((X, Cc), state['batch_idx_lig'], t_seq[-1], traj_mode)
