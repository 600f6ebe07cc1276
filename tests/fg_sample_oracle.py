"""CPU restatement of D3FG.sample (repo/models/diffusion/difffg.py:174-246) in fp32 torch, on the reference's state-dict
keys.  Pinned to the live reference by tests/golden/make_golden_f8.py (oracle == reference at every step).

Followed as written (``/root/reference``):
  repo/modules/context_emb.py:24-135        FGContextEmbedder (fg 'linear', residue 'frame', no time / vec embedding)
  repo/modules/embs/res_emb.py:16-96         AngularEncoding, PerResidueEncoder
  repo/models/utils/geometry.py:32-120, 271-360, topology.py:5-24   basis, global_to_local, backbone dihedrals
  repo/modules/common.py:189-214             compose_context
  repo/models/diffusion/diffusion_scheduler.py:144-165 (score form), 367-441, 558-574; so3.py:111-146
The encoder is oracle/ipa.py.  The histogram-bin draw is ``cbgbench_b200.difffg.multinomial_bin`` (its definition).
"""
import math

import torch
import torch.nn.functional as F

from cbgbench_b200.difffg import multinomial_bin
from oracle import ipa as OI

CA, C_, N_ = 1, 2, 0


def _normalize(v, eps=1e-6):
    return v / (torch.linalg.norm(v, ord=2, dim=-1, keepdim=True) + eps)


def construct_3d_basis(center, p1, p2):
    e1 = _normalize(p1 - center)
    v2 = p2 - center
    u2 = v2 - (e1 * v2).sum(dim=-1, keepdim=True) * e1
    e2 = _normalize(u2)
    e3 = torch.cross(e1, e2, dim=-1)
    return torch.cat([e1.unsqueeze(-1), e2.unsqueeze(-1), e3.unsqueeze(-1)], dim=-1)


def global_to_local(R, t, q):
    q_size = q.size()
    N = q_size[0]
    q = q.reshape(N, -1, 3).transpose(-1, -2)
    p = torch.matmul(R.transpose(-1, -2), (q - t.unsqueeze(-1)))
    return p.transpose(-1, -2).reshape(q_size)


def dihedral_from_four_points(p0, p1, p2, p3):
    v0, v1, v2 = p2 - p1, p0 - p1, p3 - p2
    u1 = torch.cross(v0, v1, dim=-1)
    n1 = u1 / torch.linalg.norm(u1, dim=-1, keepdim=True)
    u2 = torch.cross(v0, v2, dim=-1)
    n2 = u2 / torch.linalg.norm(u2, dim=-1, keepdim=True)
    sgn = torch.sign((torch.cross(v1, v2, dim=-1) * v0).sum(-1))
    return torch.nan_to_num(sgn * torch.acos((n1 * n2).sum(-1).clamp(min=-0.999999, max=0.999999)))


def backbone_dihedrals(pos, chain_nb, res_nb, mask):
    pN, pCA, pC = pos[:, N_], pos[:, CA], pos[:, C_]
    consec = torch.logical_and((res_nb[1:] - res_nb[:-1]).abs() == 1, chain_nb[1:] == chain_nb[:-1])
    consec = torch.logical_and(consec, mask[:-1])
    N_term = F.pad(torch.logical_not(consec), pad=(1, 0), value=1)
    C_term = F.pad(torch.logical_not(consec), pad=(0, 1), value=1)
    omega = F.pad(dihedral_from_four_points(pCA[:-1], pC[:-1], pN[1:], pCA[1:]), pad=(1, 0), value=0)
    phi = F.pad(dihedral_from_four_points(pC[:-1], pN[1:], pCA[1:], pC[1:]), pad=(1, 0), value=0)
    psi = F.pad(dihedral_from_four_points(pN[:-1], pCA[:-1], pC[:-1], pN[1:]), pad=(0, 1), value=0)
    m = torch.stack([~N_term, ~N_term, ~C_term], dim=-1)
    return torch.stack([omega, phi, psi], dim=-1) * m, m


def per_residue_encoder(sd, p, aa_onehot, res_nb, chain_nb, pos, mask_atoms):
    aa = aa_onehot.argmax(-1)
    N = aa.size()[0]
    aa_feat = F.embedding(aa, sd[p + 'aatype_embed.weight'])
    mask_residue = mask_atoms[:, CA]
    R = construct_3d_basis(pos[:, CA], pos[:, C_], pos[:, N_])
    crd = global_to_local(R, pos[:, CA], pos)
    crd = torch.where(mask_atoms[:, :, None].expand_as(crd), crd, torch.zeros_like(crd))
    aa_expand = aa[:, None, None, None].expand(N, 22, 15, 3)
    rng_expand = torch.arange(0, 22)[None, :, None, None].expand(N, 22, 15, 3)
    crd_expand = crd[:, None, :, :].expand(N, 22, 15, 3)
    crd_feat = torch.where(aa_expand == rng_expand, crd_expand, torch.zeros_like(crd_expand)).reshape(N, 22 * 15 * 3)
    dihed, mdihed = backbone_dihedrals(pos, chain_nb, res_nb, mask_residue)
    x = dihed[:, :, None].unsqueeze(-1)
    fb = sd[p + 'dihed_embed.freq_bands']
    code = torch.cat([x, torch.sin(x * fb), torch.cos(x * fb)], dim=-1).reshape(N, 3, -1)
    dihed_feat = (code * mdihed[:, :, None]).reshape(N, -1)
    h = torch.cat([aa_feat, crd_feat, dihed_feat], dim=-1)
    for i, last in ((0, False), (2, False), (4, False), (6, True)):
        h = F.linear(h, sd[p + f'mlp.{i}.weight'], sd[p + f'mlp.{i}.bias'])
        if not last:
            h = F.relu(h)
    return h * mask_residue[:, None]


def so3vec_to_rotation(w):
    return OI.so3vec_to_rotation(w)


def rotation_to_so3vec(R):
    return OI.rotation_to_so3vec(R)


def sample(sd, batch, T, pos_noise, rot_draws, type_uniform, num_classes=28, num_steps=None, hidden=256):
    """traj {t: (xc, c, o)} of D3FG.sample for t = T-1 ... T-1-num_steps with the injected draws (indexed by t)."""
    K = num_classes
    emb_classes = K + 21
    pre = 'context_embedder.'
    xc = batch['ligand_pos_heavyatom'][:, CA].float()
    c = F.one_hot(batch['ligand_type_fg'], K).float()
    o = batch['ligand_o_fg'].float()
    lig_flag, rec_flag = batch['ligand_lig_flag'], batch['protein_lig_flag']
    gen_lig = batch.get('ligand_gen_flag', lig_flag)
    gen_rec = torch.zeros_like(rec_flag)
    bl, br = batch['ligand_type_fg_batch'], batch['protein_type_fg_batch']
    x_rec = batch['protein_pos_heavyatom'].float()
    chain_cumsum = batch['protein_num_chains'].cumsum(0)
    chain_nb = torch.cat([batch['protein_chain_nb'][br == i] + chain_cumsum[i] - 1 for i in br.unique()])
    # protein part of FGContextEmbedder.forward: independent of the step
    xc_rec = x_rec[:, CA]
    o_rec = rotation_to_so3vec(construct_3d_basis(x_rec[:, CA], x_rec[:, C_], x_rec[:, N_]))
    h_rec = F.linear(F.one_hot(batch['protein_type_fg'], emb_classes).float(), sd[pre + 'protein_fg_emb.weight'],
                     sd[pre + 'protein_fg_emb.bias'])
    h_aa = per_residue_encoder(sd, pre + 'residue_emb.', F.one_hot(batch['protein_aa'], 20).float(),
                               batch['protein_res_nb'], chain_nb, x_rec, batch['protein_mask_heavyatom'])
    ind = lambda f: F.linear(f.float().unsqueeze(-1), sd[pre + 'ligand_indicator.weight'], sd[pre + 'ligand_indicator.bias'])
    h_rec = h_rec + torch.zeros_like(h_rec) + h_aa + ind(rec_flag)
    batch_ctx = torch.cat([br, bl])
    sort_idx = torch.sort(batch_ctx, stable=True).indices
    is_lig = torch.cat([rec_flag, lig_flag])[sort_idx]
    traj = {T - 1: (xc, c, o)}
    steps = list(reversed(range(T)))[:num_steps]
    for t_idx in steps:
        xc_l, c_l, o_l = traj[t_idx]
        t = torch.full((int(bl.max()) + 1,), t_idx, dtype=torch.long)
        v49 = F.one_hot(c_l.argmax(-1), emb_classes).float()
        h_lig = F.linear(v49, sd[pre + 'ligand_fg_emb.weight'], sd[pre + 'ligand_fg_emb.bias'])
        h_lig = h_lig + torch.zeros_like(h_lig) + ind(lig_flag)
        cat = lambda a, b: torch.cat([a, b])[sort_idx]
        eps, _, o_pred, _, logits = OI.ipatransformer_forward(
            sd, cat(xc_rec, xc_l), cat(o_rec, o_l.clone()), cat(h_rec, h_lig), batch_ctx[sort_idx], is_lig,
            cat(gen_rec, gen_lig), prefix='denoiser.')
        eps, o_pred, logits = eps[is_lig], o_pred[is_lig], logits[is_lig]
        x_next, v_next, o_next, _ = reverse_step(sd, t_idx, bl, xc_l, c_l, o_l, eps, o_pred, logits, gen_lig,
                                                 pos_noise[t_idx], rot_draws[t_idx], type_uniform[t_idx])
        traj[t_idx - 1] = (x_next, F.one_hot(v_next, K).float(), o_next)
    return traj


def reverse_step(sd, t_idx, bl, xc_l, c_l, o_l, eps, o_pred, logits, gen_lig, pos_noise, rd, type_u, theta=None):
    """The position / SO(3) / FG-type update of one reverse step t_idx for the ligand rows, in the dtype of ``xc_l``
    (fp32: the expressions of D3FG.sample; float64: a high-precision reference of the same step; the schedule tables
    stay the fp32 values they hold).  ``theta``: use this rotation angle instead of drawing it (a float64 composition
    with a given fp32 angle).  -> (x_next, v_next, o_next, (theta, bin, log_prob + gumbel))."""
    dt = xc_l.dtype
    K = c_l.shape[-1]
    pf = 'pos_scheduler.'
    ts = 'type_scheduler.'
    rot = 'rot_scheduler.angular_distrib_inv.'
    acp, betas = sd[pf + 'alphas_cumprod'].to(dt), sd[pf + 'betas'].to(dt)
    eps, o_pred, logits, c_l = eps.to(dt), o_pred.to(dt), logits.to(dt), c_l.to(dt)
    pos_noise, rd, type_u = pos_noise.to(dt), rd.to(dt), type_u.to(dt)
    t = torch.full((int(bl.max()) + 1,), t_idx, dtype=torch.long)
    # positions: CTNVPScheduler.backward_remove_noise, type='score'
    a = acp.index_select(0, t)[:, None][bl].expand_as(xc_l)
    b = betas.index_select(0, t)[:, None][bl].expand_as(xc_l)
    nonzero = (1 - (t == 0).to(dt))[bl].unsqueeze(-1)
    xs = (xc_l + b * (-eps / (1 - a).sqrt())) / (1 - b).sqrt()
    xs = xs + nonzero * b.sqrt() * pos_noise
    x_next = torch.where(gen_lig.unsqueeze(-1), xs, xc_l)
    # orientation: RotVPScheduler.backward_remove_noise with ApproxAngularDistribution.sample
    tt = t[bl]
    u = F.normalize(rd[:, 0:3], dim=-1)
    X, Y, std = sd[rot + 'X'].to(dt), sd[rot + 'Y'], sd[rot + 'stddevs'].to(dt)
    b_idx = multinomial_bin(Y[tt][:, :-1], rd[:, 3])
    if theta is None:
        start = X[tt, b_idx]
        s_hist = start + rd[:, 4] * (X[tt, b_idx + 1] - start)
        s_gauss = (std[tt] * 2 + rd[:, 5] * std[tt]).abs() % math.pi
        theta = torch.where(sd[rot + 'approx_flag'][tt], s_gauss, s_hist)
    e = u * theta.to(dt)[:, None]
    e = torch.where((tt > 1)[:, None].expand(-1, 3), e, torch.zeros_like(e))
    R_next = so3vec_to_rotation(e) @ so3vec_to_rotation(o_pred)
    o_next = torch.where(gen_lig[:, None].expand(-1, 3), rotation_to_so3vec(R_next), o_l)
    # FG type: TypeVPScheduler.backward_remove_noise
    tm1 = torch.clamp(t - 1, min=0)
    lv = lambda name, tt_: sd[ts + name].to(dt)[tt_][bl].unsqueeze(-1)
    lae = lambda p_, q_: torch.max(p_, q_) + torch.log(torch.exp(p_ - torch.max(p_, q_)) + torch.exp(q_ - torch.max(p_, q_)))
    log_pred = F.log_softmax(logits, dim=-1)
    log_ct = torch.log(c_l + 1e-8)
    A = lae(log_pred + lv('log_alphas_cumprod_v', tm1), lv('log_one_minus_alphas_cumprod_v', tm1) - math.log(K))
    B_ = lae(log_ct + lv('log_alphas_v', t), lv('log_one_minus_alphas_v', t) - math.log(K))
    un = A + B_
    log_prob = un - torch.logsumexp(un, dim=-1, keepdim=True)
    gumbel = -torch.log(-torch.log(type_u + 1e-30) + 1e-30)
    score = gumbel + log_prob
    v_next = torch.where(gen_lig, score.argmax(-1), c_l.argmax(-1))
    return x_next, v_next, o_next, (theta, b_idx, score)
