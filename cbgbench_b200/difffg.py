"""CUDA (H100) drop-in for the reference's ``D3FG`` model (``difffg`` / ``difffg_v2``): sampling (DESIGN.md section 16)
and the eval-mode validation losses (section 17).

Mirrors repo/models/diffusion/difffg.py:32-63 (constructor, sub-module names => state-dict keys, including the angular
histograms of the rotation schedule) and :174-246 (``sample(batch) -> traj``).  ``difffg_v2`` differs from ``difffg``
only in its position loss: ``D3FGV2B200`` is the same module with the denoise-form loss.

Once per batch, with torch ops on the device: the protein rows of the composed graph (C-alpha positions, backbone frames
as so3 vectors, FG-type + PerResidueEncoder embeddings), the compose_context permutation and the plan.  Once per model:
the float64 prefix sums of the inverse angular histograms.  Per reverse step: ONE C-ABI call, ``cbg_fg_step_f32``
(csrc/fg.cu), that writes the ligand rows, runs the IPATransformer and applies the position / SO(3) / FG-type updates.

Random numbers: per step, in the reference's order, ``randn [n,3]`` (positions), ``randn [n,3]`` (rotation axes),
``rand [n]`` (the histogram bin, see ``multinomial_bin``), ``rand [n]`` (offset in the bin), ``randn [n]`` (Gaussian
branch), ``rand [n,K]`` (Gumbel), from torch's generator of the model device; or injected for parity tests.

Validation losses (difffg.py:65-171): the R eval timesteps noise R copies of the batch, which run as R * B graphs through
ONE C-ABI call, ``cbg_fg_eval_loss_f32`` (csrc/fg_eval.cu): forward noising, one encoder pass, per-graph losses.
"""
import ctypes as C
import math

import torch
from torch import nn
import torch.nn.functional as F

from . import _lib
from .modules import cfg_get, get_e3_gnn, graph_ptr_from_batch, _Workspace
from .schedulers import CTNVPTables, TypeVPTables, VPTables
from .targetdiff import DiffusionB200, register_model

NUM_AA_TYPES = 21          # repo/utils/protein/constants.py:75: len(AA), the width added to num_fgtype by FGContextEmbedder
NUM_AA_ONEHOT = 20         # len(aa_name_number): the reference one-hots protein_aa with 20 classes (context_emb.py:119)
BB_N, BB_CA, BB_C = 0, 1, 2   # BBHeavyAtom
MAX_AA_TYPES, MAX_NUM_ATOMS = 22, 15   # PerResidueEncoder defaults (res_emb.py:42)
ROT_DRAWS = 6              # axis N(0,1)^3 | bin uniform | in-bin uniform | Gaussian-branch N(0,1)


# ---- rotation schedule (RotVPScheduler, diffusion_scheduler.py:514-529; ApproxAngularDistribution, so3.py:71-109) --------

class ApproxAngularTables(nn.Module):
    """Buffers ``stddevs``, ``approx_flag``, ``X``, ``Y`` [T, num_bins] of ApproxAngularDistribution, computed with the
    reference's fp32 torch expression on the CPU, so a fresh module equals the reference's bit for bit."""

    def __init__(self, stddevs, std_threshold=0.1, num_bins=8192, num_iters=1024):
        super().__init__()
        self.std_threshold = std_threshold
        self.num_bins = num_bins
        self.num_iters = num_iters
        self.register_buffer('stddevs', torch.FloatTensor(stddevs))
        self.register_buffer('approx_flag', self.stddevs <= std_threshold)
        X, Y = [], []
        for std in self.stddevs:
            x = torch.linspace(0, math.pi, num_bins)
            y = torch.nan_to_num(self._pdf(x, std.item(), num_iters)).clamp_min(0)
            X.append(x)
            Y.append(y)
        self.register_buffer('X', torch.stack(X, dim=0))
        self.register_buffer('Y', torch.stack(Y, dim=0))

    @staticmethod
    def _pdf(x, e, L):
        x = x[:, None]
        c = ((1 - torch.cos(x)) / math.pi)
        l = torch.arange(0, L)[None, :]
        a = (2 * l + 1) * torch.exp(-l * (l + 1) * (e ** 2))
        b = (torch.sin((l + 0.5) * x) + 1e-6) / (torch.sin(x / 2) + 1e-6)
        return (c * a * b).sum(dim=1)


class RotVPTables(VPTables):
    """RotVPScheduler: the VP tables plus the forward / inverse angular distributions and the ``_dummy`` buffer."""

    def __init__(self, num_timestep, beta_start=1e-7, beta_end=2e-3, type='sigmoid', cosine_s=0.008):
        super().__init__(num_timestep, beta_start, beta_end, type, cosine_s)
        c1 = torch.sqrt(1 - self.alphas_cumprod.detach())
        self.angular_distrib_fwd = ApproxAngularTables(c1.tolist())
        betas, acp = self.betas.detach(), self.alphas_cumprod.detach()
        sigmas = torch.zeros_like(betas)
        for i in range(1, betas.size(0)):
            sigmas[i] = ((1 - acp[i - 1]) / (1 - acp[i])) * betas[i]
        self.angular_distrib_inv = ApproxAngularTables(torch.sqrt(sigmas).tolist())
        self.register_buffer('_dummy', torch.empty([0, ]))

    def bin_cdf(self, device):
        """Inclusive float64 prefix sums C_t of ``angular_distrib_inv.Y[t, :-1]`` on ``device`` (cached per table
        version).  Summed on the CPU row by row, the same sums the definition of the bin draw uses."""
        return self._prefix_sums('inv', self.angular_distrib_inv.Y, device)

    def fwd_cdf(self, device):
        """The same prefix sums of ``angular_distrib_fwd.Y``: the forward noising of the validation loss draws its angles
        from the forward distribution.  Cached separately from ``bin_cdf``."""
        return self._prefix_sums('fwd', self.angular_distrib_fwd.Y, device)

    def _prefix_sums(self, name, Y, device):
        key = (Y.data_ptr(), Y._version, str(device))
        if self.__dict__.get('_cdf_key_' + name) != key:
            self.__dict__['_cdf_' + name] = Y.detach().cpu()[:, :-1].double().cumsum(-1).to(device).contiguous()
            self.__dict__['_cdf_key_' + name] = key
        return self.__dict__['_cdf_' + name]


def multinomial_bin(prob, u):
    """The histogram-bin draw that stands for ``torch.multinomial(prob, 1)`` (so3.py:123):
    b = min{i : C[i] > u C[-1]}, C the float64 inclusive prefix sum of each row of ``prob``, u ~ U[0,1) per row."""
    cdf = prob.double().cumsum(-1)
    return torch.searchsorted(cdf, (u.double() * cdf[:, -1]).unsqueeze(-1).contiguous(), right=True).squeeze(-1)


# ---- context embedder (FGContextEmbedder, context_emb.py:24-135) -------------------------------------------------------

class AngularEncodingW(nn.Module):
    """res_emb.py:16-37 (buffer ``freq_bands``)."""

    def __init__(self, num_funcs=3):
        super().__init__()
        self.num_funcs = num_funcs
        self.register_buffer('freq_bands', torch.FloatTensor([i + 1 for i in range(num_funcs)] +
                                                             [1. / (i + 1) for i in range(num_funcs)]))


class PerResidueEncoderW(nn.Module):
    """Parameters of PerResidueEncoder (res_emb.py:40-54)."""

    def __init__(self, feat_dim):
        super().__init__()
        self.aatype_embed = nn.Embedding(MAX_AA_TYPES, feat_dim)
        self.dihed_embed = AngularEncodingW()
        infeat = feat_dim + MAX_AA_TYPES * MAX_NUM_ATOMS * 3 + 3 * (1 + 2 * 2 * self.dihed_embed.num_funcs)
        self.mlp = nn.Sequential(nn.Linear(infeat, feat_dim * 2), nn.ReLU(), nn.Linear(feat_dim * 2, feat_dim), nn.ReLU(),
                                 nn.Linear(feat_dim, feat_dim), nn.ReLU(), nn.Linear(feat_dim, feat_dim))


class FGContextEmbedderB200(nn.Module):
    """Parameter container for FGContextEmbedder with fg 'linear' and residue 'frame' embeddings (the shipped D3FG
    embedder, configs/denovo/train/d3fg_fg.yml), plus the once-per-batch protein features."""

    def __init__(self, cfg):
        super().__init__()
        self.num_classes = cfg_get(cfg, 'num_fgtype', 50) + NUM_AA_TYPES
        emb_dim = cfg_get(cfg, 'emb_dim', 128)
        self.emb_dim = emb_dim
        if cfg_get(cfg, 'time', None) is not None or cfg_get(cfg, 'vec', None) is not None:
            raise NotImplementedError('FGContextEmbedderB200: time / vec embeddings are not built (no shipped D3FG config '
                                      'uses them)')
        fg, res = cfg_get(cfg, 'fg', None), cfg_get(cfg, 'residue', None)
        if fg is None or cfg_get(fg, 'type') != 'linear' or res is None or cfg_get(res, 'type') != 'frame':
            raise NotImplementedError("FGContextEmbedderB200: needs fg.type 'linear' and residue.type 'frame'")
        self.ligand_fg_emb = nn.Linear(self.num_classes, emb_dim)
        self.protein_fg_emb = nn.Linear(self.num_classes, emb_dim)
        self.residue_emb = PerResidueEncoderW(emb_dim)
        self.ligand_indicator = nn.Linear(1, emb_dim)

    def protein_features(self, x_rec, v_rec, aa, res_nb, chain_nb, mask_atoms):
        """(xc_rec, o_rec, h_rec) of context_emb.py:73-79, 106-129 for the protein rows (t_emb = 0, rec_flag = 0)."""
        xc = x_rec[:, BB_CA]
        R = construct_3d_basis(xc, x_rec[:, BB_C], x_rec[:, BB_N])
        o_rec = rotation_to_so3vec(R)
        h = self.protein_fg_emb(F.one_hot(v_rec, num_classes=self.num_classes).float())
        h = h + torch.zeros_like(h)                                     # the all-zero time embedding
        h = h + self._residue_features(R, x_rec, aa, res_nb, chain_nb, mask_atoms)
        bias = self.ligand_indicator(torch.zeros(x_rec.shape[0], 1, device=x_rec.device))
        return xc, o_rec, h + bias

    def _residue_features(self, R, pos, aa, res_nb, chain_nb, mask_atoms):
        """PerResidueEncoder.forward (res_emb.py:56-96)."""
        re = self.residue_emb
        N = aa.shape[0]
        mask_res = mask_atoms[:, BB_CA]
        ca = pos[:, BB_CA]
        crd = torch.matmul(R.transpose(-1, -2), pos.transpose(-1, -2) - ca.unsqueeze(-1)).transpose(-1, -2)
        crd = torch.where(mask_atoms[:, :, None], crd, torch.zeros_like(crd))
        crd_feat = torch.zeros(N, MAX_AA_TYPES, MAX_NUM_ATOMS, 3, device=pos.device)
        crd_feat[torch.arange(N, device=pos.device), aa] = crd
        dihed, dmask = backbone_dihedrals(pos, chain_nb, res_nb, mask_res)
        x = dihed[:, :, None]
        fb = re.dihed_embed.freq_bands
        code = torch.cat([x, torch.sin(x * fb), torch.cos(x * fb)], dim=-1) * dmask[:, :, None]
        feat = torch.cat([re.aatype_embed.weight[aa], crd_feat.reshape(N, -1), code.reshape(N, -1)], dim=-1)
        return re.mlp(feat) * mask_res[:, None]


def normalize_vector(v, eps=1e-6):
    return v / (torch.linalg.norm(v, ord=2, dim=-1, keepdim=True) + eps)


def construct_3d_basis(center, p1, p2):
    """geometry.py:53-75: columns e1, e2, e3."""
    e1 = normalize_vector(p1 - center)
    v2 = p2 - center
    e2 = normalize_vector(v2 - (v2 * e1).sum(-1, keepdim=True) * e1)
    e3 = torch.cross(e1, e2, dim=-1)
    return torch.stack([e1, e2, e3], dim=-1)


def rotation_to_so3vec(R):
    """so3.py:10-31, 60-63 (no-grad branch)."""
    cos_t = ((R[..., 0, 0] + R[..., 1, 1] + R[..., 2, 2] - 1) / 2).clamp_min(min=-1.0)
    sin_t = torch.sqrt(1 - cos_t ** 2)
    coef = ((torch.acos(cos_t) + 1e-8) / (2 * sin_t + 2e-8))[..., None, None]
    L = coef * (R - R.transpose(-1, -2))
    return torch.stack([L[..., 1, 2], L[..., 2, 0], L[..., 0, 1]], dim=-1)


def dihedral(p0, p1, p2, p3):
    """geometry.py:271-289."""
    v0, v1, v2 = p2 - p1, p0 - p1, p3 - p2
    u1 = torch.cross(v0, v1, dim=-1)
    n1 = u1 / torch.linalg.norm(u1, dim=-1, keepdim=True)
    u2 = torch.cross(v0, v2, dim=-1)
    n2 = u2 / torch.linalg.norm(u2, dim=-1, keepdim=True)
    sgn = torch.sign((torch.cross(v1, v2, dim=-1) * v0).sum(-1))
    return torch.nan_to_num(sgn * torch.acos((n1 * n2).sum(-1).clamp(min=-0.999999, max=0.999999)))


def backbone_dihedrals(pos, chain_nb, res_nb, mask):
    """get_backbone_dihedral_angles (geometry.py:327-360, topology.py:5-24) over the flattened residue list."""
    n, ca, c = pos[:, BB_N], pos[:, BB_CA], pos[:, BB_C]
    consec = ((res_nb[1:] - res_nb[:-1]).abs() == 1) & (chain_nb[1:] == chain_nb[:-1]) & mask[:-1]
    n_term = F.pad(~consec, pad=(1, 0), value=1)
    c_term = F.pad(~consec, pad=(0, 1), value=1)
    omega = F.pad(dihedral(ca[:-1], c[:-1], n[1:], ca[1:]), pad=(1, 0), value=0)
    phi = F.pad(dihedral(c[:-1], n[1:], ca[1:], c[1:]), pad=(1, 0), value=0)
    psi = F.pad(dihedral(n[:-1], ca[:-1], c[:-1], n[1:]), pad=(0, 1), value=0)
    dmask = torch.stack([~n_term, ~n_term, ~c_term], dim=-1)
    return torch.stack([omega, phi, psi], dim=-1) * dmask, dmask


# ---- the model ---------------------------------------------------------------------------------------------------------

@register_model('difffg')
class D3FGB200(DiffusionB200):
    """D3FG (difffg.py:32-63, 250-280) with CUDA sampling and validation-loss paths."""

    pos_loss_form = _lib.FG_LOSS_SCORE    # difffg: get_score_loss(score_in=False) (difffg.py:145-148)

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        gen = cfg.generator
        self.num_classes = cfg.num_fgtype
        self.num_diffusion_timesteps = gen.num_diffusion_timesteps
        if not cfg_get(gen, 'denoise_structure', True) or not cfg_get(gen, 'denoise_atom', True):
            raise NotImplementedError('D3FGB200: denoise_structure / denoise_atom = False are not built')
        ps, rs, fs = gen.pos_schedule, gen.rot_schedule, gen.fg_schedule
        self.pos_scheduler = CTNVPTables(self.num_diffusion_timesteps, beta_start=cfg_get(ps, 'beta_start', 1e-7),
                                         beta_end=cfg_get(ps, 'beta_end', 2e-3), type=cfg_get(ps, 'type', 'sigmoid'))
        self.rot_scheduler = RotVPTables(self.num_diffusion_timesteps, type=cfg_get(rs, 'type', 'sigmoid'),
                                         cosine_s=cfg_get(rs, 'cosine_s', 0.008))
        self.type_scheduler = TypeVPTables(self.num_diffusion_timesteps, num_classes=self.num_classes,
                                           type=cfg_get(fs, 'type', 'sigmoid'), cosine_s=cfg_get(fs, 'cosine_s', 0.008))
        cfg.embedder.num_fgtype = cfg.num_fgtype
        if cfg_get(cfg.embedder, 'type', 'fa') != 'fg':
            raise NotImplementedError("D3FGB200: embedder.type must be 'fg'")
        self.context_embedder = FGContextEmbedderB200(cfg.embedder)
        self.denoiser = get_e3_gnn(cfg.encoder, num_classes=self.num_classes)
        if self.context_embedder.emb_dim != self.denoiser.hidden_dim:
            raise NotImplementedError('D3FGB200: embedder.emb_dim must equal encoder.node_feat_dim')
        self._ws = _Workspace()
        self.last_launches = 0

    def _device(self):
        dev = next(self.parameters()).device
        if dev.type != 'cuda':
            raise RuntimeError('D3FGB200.sample needs the model on a CUDA device (no CPU fallback)')
        return dev

    # ---- once per batch ------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def _context(self, batch):
        """The batch's tensors on the model's device, checked, and the protein rows of the composed graph.  Computed once
        per batch: the PerResidueEncoder MLP runs through cuBLAS, whose kernel choice depends on the row count, so the
        replicas of the validation loss tile these rows instead of recomputing them on a larger batch."""
        dev = self._device()
        K = self.num_classes
        g = lambda k: batch[k].to(dev)
        xc_lig = g('ligand_pos_heavyatom')[:, BB_CA].float().contiguous()
        v_lig = g('ligand_type_fg').long()
        o_lig = g('ligand_o_fg').float().contiguous()
        lig_flag, rec_flag = g('ligand_lig_flag').bool(), g('protein_lig_flag').bool()
        gen_lig = (batch['ligand_gen_flag'] if 'ligand_gen_flag' in batch else batch['ligand_lig_flag']).to(dev).bool()
        gen_rec = batch['protein_gen_flag'].to(dev).bool() if 'protein_gen_flag' in batch else torch.zeros_like(rec_flag)
        bl, br = g('ligand_type_fg_batch').long(), g('protein_type_fg_batch').long()
        aa = g('protein_aa').long()
        n_lig, n_rec = int(bl.numel()), int(br.numel())
        if n_lig == 0 or n_rec == 0:
            raise ValueError('D3FGB200.sample: the batch needs functional groups and residues')
        if not bool(lig_flag.all()) or bool(rec_flag.any()):
            raise ValueError('D3FGB200.sample: ligand_lig_flag must be all True and protein_lig_flag all False')
        if bool((aa < 0).any()) or bool((aa >= NUM_AA_ONEHOT).any()):
            raise ValueError(f'protein_aa must lie in [0, {NUM_AA_ONEHOT}) (the reference one-hots it with 20 classes)')
        if bool((v_lig < 0).any()) or bool((v_lig >= K).any()):
            raise ValueError(f'ligand_type_fg must lie in [0, {K})')
        # difffg.py:188-192: chain ids offset per graph by protein_num_chains.cumsum - 1 (rows are sorted by graph)
        chain_nb = g('protein_chain_nb').long() + (g('protein_num_chains').long().cumsum(0) - 1)[br]
        xc_rec, o_rec, h_rec = self.context_embedder.protein_features(
            g('protein_pos_heavyatom').float(), g('protein_type_fg').long(), aa, g('protein_res_nb').long(), chain_nb,
            g('protein_mask_heavyatom').bool())
        return {'device': dev, 'n_lig': n_lig, 'n_rec': n_rec, 'bl': bl, 'br': br, 'xc_lig': xc_lig, 'v_lig': v_lig,
                'o_lig': o_lig, 'lig_flag': lig_flag, 'rec_flag': rec_flag, 'gen_lig': gen_lig, 'gen_rec': gen_rec,
                'xc_rec': xc_rec, 'o_rec': o_rec, 'h_rec': h_rec}

    @torch.no_grad()
    def _compose(self, ctx, n_rep, angular, cdf):
        """Composed arrays and the plan of ``n_rep`` replicas of the batch of ``ctx``, replica-major: replica r's graph g is
        graph r * B + g.  The protein rows are written here; the ligand rows of x / o / h are the kernels'.  ``angular``
        (an ApproxAngularTables) and ``cdf`` (its prefix sums) are the angle tables the plan points at."""
        dev = ctx['device']
        K, H = self.num_classes, self.denoiser.hidden_dim
        bl, br = ctx['bl'], ctx['br']
        if n_rep == 1:
            tile = off = lambda v: v
        else:
            B = int(torch.cat([br, bl]).max()) + 1
            steps = torch.arange(n_rep, device=dev).unsqueeze(1) * B
            tile = lambda v: v.repeat(n_rep, *([1] * (v.dim() - 1)))
            off = lambda b: (b.unsqueeze(0) + steps).reshape(-1)
        n_lig, n_rec = ctx['n_lig'] * n_rep, ctx['n_rec'] * n_rep
        # compose_context (common.py:189-214): [protein | ligand] stably sorted by graph id
        batch_ctx = torch.cat([off(br), off(bl)])
        sort_idx = torch.sort(batch_ctx, stable=True).indices
        inv = torch.empty_like(sort_idx)
        inv[sort_idx] = torch.arange(sort_idx.numel(), device=dev)
        N = n_rec + n_lig
        cat = lambda a, b: torch.cat([a, b])[sort_idx].contiguous()
        x = cat(tile(ctx['xc_rec']).float(), tile(ctx['xc_lig']))
        o = cat(tile(ctx['o_rec']).float(), tile(ctx['o_lig']))
        h = cat(tile(ctx['h_rec']).float(), torch.zeros(n_lig, H, device=dev))
        lig8 = cat(tile(ctx['rec_flag']), tile(ctx['lig_flag'])).to(torch.uint8)
        gen8 = cat(tile(ctx['gen_rec']), tile(ctx['gen_lig'])).to(torch.uint8)
        gptr, n_graphs, max_n = graph_ptr_from_batch(batch_ctx[sort_idx])
        lig_node = inv[n_rec:].to(torch.int32).contiguous()
        ce = self.context_embedder
        fg_emb_t = ce.ligand_fg_emb.weight.detach()[:, :K].t().float().contiguous()
        fg_emb_b = ce.ligand_fg_emb.bias.detach().float().contiguous()
        lig_ind = ce.ligand_indicator(torch.ones(1, 1, device=dev))[0].float().contiguous()
        angle_x = angular.X.detach().float().contiguous()
        blob = self.denoiser.packed_blob(dev)
        L = _lib.lib()
        ws_ptr, ws_have = self._ws.get(L.cbg_fg_workspace_bytes(N, H, K), dev)
        gen_lig8 = tile(ctx['gen_lig']).to(torch.uint8).contiguous()
        d = self.denoiser
        plan = _lib.FgPlan(blob=blob.data_ptr(), hidden=H, num_sublayers=d.num_layers * d.num_x2h, num_blocks=d.num_blocks,
                      num_classes=K, k=d.cut_off, graph_ptr=gptr.data_ptr(), n_graphs=n_graphs, max_graph_nodes=max_n,
                      n_nodes=N, lig_flag=lig8.data_ptr(), gen_flag=gen8.data_ptr(), lig_node=lig_node.data_ptr(),
                      gen_lig=gen_lig8.data_ptr(), n_lig=n_lig,
                      x=x.data_ptr(), o=o.data_ptr(), h=h.data_ptr(), fg_emb_t=fg_emb_t.data_ptr(),
                      fg_emb_b=fg_emb_b.data_ptr(), lig_indicator=lig_ind.data_ptr(), angle_x=angle_x.data_ptr(),
                      angle_cdf=cdf.data_ptr(), n_bins=angle_x.shape[1], workspace=ws_ptr, workspace_bytes=ws_have)
        # tensors the plan points into stay alive with the state
        keep = (blob, gptr, lig8, gen8, lig_node, gen_lig8, x, o, h, fg_emb_t, fg_emb_b, lig_ind, angle_x, cdf)
        return {'plan': plan, 'keep': keep, 'device': dev, 'n_lig': n_lig, 'n_graphs': n_graphs, 'n_nodes': N}

    @torch.no_grad()
    def begin(self, batch):
        """Protein features, composed arrays and the step plan for ``batch`` (the reference's FG batch keys)."""
        ctx = self._context(batch)
        rot = self.rot_scheduler
        state = self._compose(ctx, 1, rot.angular_distrib_inv, rot.bin_cdf(ctx['device']))
        state.update(batch_idx_lig=ctx['bl'], x0=ctx['xc_lig'], c0=F.one_hot(ctx['v_lig'], num_classes=self.num_classes).float(),
                     o0=ctx['o_lig'])
        return state

    # ---- per step ------------------------------------------------------------------------------------------------------
    def step_coef(self, t, rot_std, rot_flag):
        """Host scalars of reverse step t, with the reference's fp32 torch expressions; ``rot_std`` / ``rot_flag`` are CPU
        copies of angular_distrib_inv.stddevs / approx_flag."""
        ps, ts = self.pos_scheduler, self.type_scheduler
        a = torch.tensor(ps.host_table('alphas_cumprod')[t])
        b = torch.tensor(ps.host_table('betas')[t])
        nonzero = torch.tensor(0.0 if t == 0 else 1.0)
        tm1 = max(t - 1, 0)
        return _lib.FgCoef(t=t, pos_beta=float(b), pos_sigma=float((1 - a).sqrt()), pos_sqrt_one_minus_beta=float((1 - b).sqrt()),
                      pos_noise_scale=float(nonzero * b.sqrt()), rot_std=float(rot_std[t]),
                      rot_gaussian=int(bool(rot_flag[t])), rot_noise=int(t > 1),
                      log_alphas_cumprod_prev=float(ts.host_table('log_alphas_cumprod_v')[tm1]),
                      log_one_minus_alphas_cumprod_prev=float(ts.host_table('log_one_minus_alphas_cumprod_v')[tm1]),
                      log_alpha=float(ts.host_table('log_alphas_v')[t]),
                      log_one_minus_alpha=float(ts.host_table('log_one_minus_alphas_v')[t]))

    @torch.no_grad()
    def sample(self, batch, pos_noise=None, rot_draws=None, type_uniform=None, num_steps=None, traj_mode='full'):
        """D3FG.sample (difffg.py:174-246).

        Returns ``traj``: {t: (xc_lig [n,3], c_lig [n,K] one-hot, o_lig [n,3], batch_idx_lig)} for t = T-1 ... t_last on
        the CPU and t_last - 1 on the device (t_last = 0 for a full run).  ``traj_mode='final'`` keeps traj[t_last] and
        traj[t_last - 1] only.  Injected draws, indexed by t: ``pos_noise`` [T,n,3] N(0,1), ``rot_draws`` [T,n,6] (axis
        N(0,1)^3, bin uniform, in-bin uniform, Gaussian-branch N(0,1)), ``type_uniform`` [T,n,K] U[0,1); all three or
        none.  ``num_steps`` stops after that many steps (testing)."""
        if (pos_noise is None) != (rot_draws is None) or (pos_noise is None) != (type_uniform is None):
            raise ValueError('inject pos_noise, rot_draws and type_uniform together, or none of them')
        T, K = self.num_diffusion_timesteps, self.num_classes
        t_seq = list(reversed(range(T)))[:num_steps]
        if not t_seq:
            raise ValueError('num_steps must be at least 1')
        state = self.begin(batch)
        rot = self.rot_scheduler.angular_distrib_inv
        rot_std, rot_flag = rot.stddevs.cpu(), rot.approx_flag.cpu()
        dev, n, plan = state['device'], state['n_lig'], state['plan']
        X, Cc, O = self._traj_buffers(dev, (state['x0'], state['c0'], state['o0']))
        to = lambda a: a.to(dev, torch.float32).contiguous()
        L = _lib.lib()
        st = _lib.stream_ptr(dev)
        launches0 = L.cbg_launch_count()
        with torch.cuda.device(dev):
            for t in t_seq:
                if pos_noise is None:
                    pn = torch.randn(n, 3, device=dev)
                    axis = torch.randn(n, 3, device=dev)
                    u_bin, u_off = torch.rand(n, device=dev), torch.rand(n, device=dev)
                    gauss = torch.randn(n, device=dev)
                    tu = torch.rand(n, K, device=dev)
                    rd = torch.cat([axis, u_bin[:, None], u_off[:, None], gauss[:, None]], dim=1).contiguous()
                else:
                    pn, rd, tu = to(pos_noise[t]), to(rot_draws[t]), to(type_uniform[t])
                _lib.check(L.cbg_fg_step_f32(C.byref(plan), self.step_coef(t, rot_std, rot_flag), X[t + 1].data_ptr(), Cc[t + 1].data_ptr(),
                                             O[t + 1].data_ptr(), pn.data_ptr(), rd.data_ptr(), tu.data_ptr(),
                                             X[t].data_ptr(), Cc[t].data_ptr(), O[t].data_ptr(), st))
        self.last_launches = L.cbg_launch_count() - launches0
        return self._traj((X, Cc, O), state['batch_idx_lig'], t_seq[-1], traj_mode)

    # ---- validation losses (D3FG.forward with self.training == False, difffg.py:65-171 / :283-389) -----------------------
    def _check_eval_mode(self):
        """Training mode raises, and so does a model on the CPU: ``eval_losses`` reads the batch's graph ids before its
        own device check, so ``forward`` checks the device first."""
        super()._check_eval_mode()
        self._eval_device()

    def eval_coef(self, t):
        """Host scalars of the validation loss at timestep t, with the reference's fp32 torch expressions."""
        ps, rs, ts = self.pos_scheduler, self.rot_scheduler, self.type_scheduler
        a = torch.tensor(ps.host_table('alphas_cumprod')[t])
        ar = torch.tensor(rs.host_table('alphas_cumprod')[t])
        fwd = rs.angular_distrib_fwd
        tm1 = max(t - 1, 0)
        tab = ts.host_table
        return _lib.FgEvalCoef(
            t=t, pos_sqrt_alphas_cumprod=float(a.sqrt()), pos_sqrt_one_minus_alphas_cumprod=float((1. - a).sqrt()),
            rot_sqrt_alphas_cumprod=float(torch.sqrt(ar)), rot_std=float(fwd.stddevs[t]),
            rot_gaussian=int(bool(fwd.approx_flag[t])),
            log_alphas_cumprod=float(tab('log_alphas_cumprod_v')[t]),
            log_one_minus_alphas_cumprod=float(tab('log_one_minus_alphas_cumprod_v')[t]),
            log_alphas_cumprod_prev=float(tab('log_alphas_cumprod_v')[tm1]),
            log_one_minus_alphas_cumprod_prev=float(tab('log_one_minus_alphas_cumprod_v')[tm1]),
            log_alpha=float(tab('log_alphas_v')[t]), log_one_minus_alpha=float(tab('log_one_minus_alphas_v')[t]),
            t_is_zero=1 if t == 0 else 0)

    @torch.no_grad()
    def eval_losses(self, batch, t_values, pos_noise=None, rot_draws=None, type_uniform=None, max_nodes=None):
        """Validation losses of ``batch`` at the timesteps ``t_values`` (D3FG.get_loss once per t).  Returns
        ``(loss_dict, results)`` like the reference's eval-mode forward: ``loss_dict`` = {'pos', 'rot', 'fg'} as CPU 0-d
        float32 tensors (mean over t of the per-t losses), ``results`` one dict per t of device tensors, keys in the
        reference's order: eps_0, eps_pred, score_0, score_pred (``difffg``) or x0, xt, x_pred (``difffg_v2``), then
        mask_gen, v0, vt, c_pred, R0, R_pred.  A t whose batch has no generated FG gets NaN losses.

        The encoder does not see t, so the R = len(t_values) noised copies of the batch run as R * B graphs through ONE
        encoder pass; above ``max_nodes`` composed nodes (default ``eval_max_nodes``) or 64 copies they are split over
        several launches, which changes no bit.  ``last_ot`` [R,n,3] keeps the noised orientations and
        ``last_graph_loss`` [R*B,4] the per-graph pos / rot / fg means and generated-FG counts.

        Draws, all three or none: ``pos_noise`` [R,n,3] N(0,1), ``rot_draws`` [R,n,6] (axis N(0,1)^3, bin uniform,
        in-bin uniform, Gaussian-branch N(0,1)), ``type_uniform`` [R,n,K] U[0,1).  By default they are drawn with torch on
        the model device in the reference's order (for each t: randn [n,3], randn [n,3], rand [n], rand [n], randn [n],
        rand [n,K]; the bin draw stands for ``torch.multinomial``, see ``multinomial_bin``)."""
        K = self.num_classes
        t_values = self._eval_t_values(t_values)
        if (pos_noise is None) != (rot_draws is None) or (pos_noise is None) != (type_uniform is None):
            raise ValueError('inject pos_noise, rot_draws and type_uniform together, or none of them')
        bl, br = batch['ligand_type_fg_batch'], batch['protein_type_fg_batch']
        if bl.numel() and br.numel() and int(br.max()) > int(bl.max()):
            # the reference sizes t by the last graph with FGs and indexes it with the residues' graph ids (IndexError)
            raise ValueError('D3FGB200.forward: the last graph of the batch has residues but no functional group')
        self._check_eval_mode()
        dev = self._eval_device()
        ctx = self._context(batch)
        R, n = len(t_values), ctx['n_lig']
        if pos_noise is None:
            pos_noise, rot_draws, type_uniform = (torch.empty(R, n, w, device=dev) for w in (3, ROT_DRAWS, K))
            for r in range(R):
                pos_noise[r] = torch.randn(n, 3, device=dev)
                rot_draws[r, :, 0:3] = torch.randn(n, 3, device=dev)
                rot_draws[r, :, 3] = torch.rand(n, device=dev)
                rot_draws[r, :, 4] = torch.rand(n, device=dev)
                rot_draws[r, :, 5] = torch.randn(n, device=dev)
                type_uniform[r] = torch.rand(n, K, device=dev)
        to = lambda a, w: a.to(dev, torch.float32).reshape(R, n, w).contiguous()
        pn, rd, tu = to(pos_noise, 3), to(rot_draws, ROT_DRAWS), to(type_uniform, K)
        score_form = self.pos_loss_form == _lib.FG_LOSS_SCORE
        xt, ot, pred = (torch.empty(R, n, 3, device=dev) for _ in range(3))
        vt = torch.empty(R, n, dtype=torch.int64, device=dev)
        score = torch.empty(R, 2, n, 3, device=dev) if score_form else None
        c_pred = torch.empty(R, n, K, device=dev)
        R_pred = torch.empty(R, n, 3, 3, device=dev)
        R0 = torch.empty(n, 3, 3, device=dev)
        rep_loss = torch.empty(R, 3, device=dev)
        x0, v0, o0 = ctx['xc_lig'], ctx['v_lig'].contiguous(), ctx['o_lig']
        fwd, cdf = self.rot_scheduler.angular_distrib_fwd, self.rot_scheduler.fwd_cdf(dev)
        L = _lib.lib()
        st = _lib.stream_ptr(dev)
        graph_loss = []

        def launch(r0, r1, state, coefs):
            gl = torch.empty(state['n_graphs'], 4, device=dev)
            _lib.check(L.cbg_fg_eval_loss_f32(
                C.byref(state['plan']), coefs, r1 - r0, self.pos_loss_form, x0.data_ptr(), v0.data_ptr(),
                o0.data_ptr(), pn[r0:r1].data_ptr(), rd[r0:r1].data_ptr(), tu[r0:r1].data_ptr(), xt[r0:r1].data_ptr(),
                ot[r0:r1].data_ptr(), vt[r0:r1].data_ptr(), pred[r0:r1].data_ptr(),
                score[r0:r1].data_ptr() if score_form else None, c_pred[r0:r1].data_ptr(), R_pred[r0:r1].data_ptr(),
                R0.data_ptr(), gl.data_ptr(), rep_loss[r0:r1].data_ptr(), st))
            graph_loss.append(gl)
        self._eval_loop(n + ctx['n_rec'], t_values, _lib.FgEvalCoef, max_nodes, launch,
                        lambda n_rep: self._compose(ctx, n_rep, fwd, cdf))
        self.last_ot = ot
        self.last_graph_loss = torch.cat(graph_loss)
        loss_dict = self._eval_dict_mean(rep_loss, ('pos', 'rot', 'fg'))
        mask_gen = ctx['gen_lig']
        results = []
        for r in range(R):
            if score_form:
                res = {'eps_0': pn[r], 'eps_pred': pred[r], 'score_0': score[r, 0], 'score_pred': score[r, 1]}
            else:
                res = {'x0': x0, 'xt': xt[r], 'x_pred': pred[r]}
            res.update({'mask_gen': mask_gen, 'v0': v0, 'vt': vt[r], 'c_pred': c_pred[r], 'R0': R0, 'R_pred': R_pred[r]})
            results.append(res)
        return loss_dict, results


@register_model('difffg_v2')
class D3FGV2B200(D3FGB200):
    """``difffg_v2`` (difffg.py:250-389): the module of ``difffg``; its position loss is get_loss(type='denoise'),
    ||x_pred - x0||^2 on the encoder's position output (difffg.py:363-365)."""

    pos_loss_form = _lib.FG_LOSS_DENOISE
