"""CPU restatement of the reference's eval-mode D3FG.forward (the validation losses of ``difffg`` / ``difffg_v2``).

TEST INFRASTRUCTURE, like oracle/: written from the reference as it reads, one timestep at a time with materialised
tensors, on top of the sampling oracle's protein-feature restatement (tests/fg_sample_oracle.py) and the encoder
restatement oracle/ipa.py.  Pinned to the live reference by tests/golden/make_golden_f9.py.

Reference code followed (``repo/`` of the reference checkout):
  models/diffusion/difffg.py:16-31                  rotation_matrix_cosine_loss
  models/diffusion/difffg.py:65-171 / :283-389      D3FG.forward (eval branch) / get_loss of difffg and difffg_v2
  models/diffusion/diffusion_scheduler.py:117-134   CTNVPScheduler.forward_add_noise
  models/diffusion/diffusion_scheduler.py:185-220   CTNVPScheduler.get_loss (type='denoise') / get_score_loss
  models/diffusion/diffusion_scheduler.py:339-418   TypeVPScheduler.forward_add_noise / get_loss / q_v_posterior
  models/diffusion/diffusion_scheduler.py:531-556   RotVPScheduler.forward_add_noise
  models/utils/so3.py:111-146                       ApproxAngularDistribution.sample, random_normal_so3
  modules/context_emb.py:24-135, modules/common.py:189-214, :33-42   embedder, compose_context, get_dict_mean

Randomness is INJECTED: for timestep r, ``pos_noise[r]`` [n,3] replaces the position ``randn_like``, ``rot_draws[r]``
[n,6] the axis ``randn``, the multinomial bin (by its definition ``multinomial_bin``), the in-bin ``rand_like`` and the
Gaussian-branch ``randn_like``, and ``type_uniform[r]`` [n,K] the Gumbel ``rand_like``.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from cbgbench_b200.difffg import multinomial_bin
from oracle import ipa as OI
from oracle.graph_ops import scatter_mean
import fg_sample_oracle as OF

CA, C_, N_ = 1, 2, 0


def log_onehot(v, K):
    return torch.log(F.one_hot(v, K).float().clamp(min=1e-30))


def log_add_exp(a, b):
    m = torch.max(a, b)
    return m + torch.log(torch.exp(a - m) + torch.exp(b - m))


def q_v_posterior(sd, log_v0, log_vt, t, K):
    p = 'type_scheduler.'
    tm1 = max(t - 1, 0)
    a = log_add_exp(log_v0 + sd[p + 'log_alphas_cumprod_v'][tm1], sd[p + 'log_one_minus_alphas_cumprod_v'][tm1] - np.log(K))
    b = log_add_exp(log_vt + sd[p + 'log_alphas_v'][t], sd[p + 'log_one_minus_alphas_v'][t] - np.log(K))
    un = a + b
    return un - torch.logsumexp(un, dim=-1, keepdim=True)


def forward_angle(sd, t, rd):
    """theta of ApproxAngularDistribution.sample on angular_distrib_fwd at t for the draws rd [n,6]."""
    rot = 'rot_scheduler.angular_distrib_fwd.'
    X, Y, std = sd[rot + 'X'], sd[rot + 'Y'], sd[rot + 'stddevs']
    tt = torch.full((rd.shape[0],), t, dtype=torch.long)
    b = multinomial_bin(Y[tt][:, :-1], rd[:, 3])
    start = X[tt, b]
    s_hist = start + rd[:, 4] * (X[tt, b + 1] - start)
    s_gauss = (std[tt] * 2 + rd[:, 5] * std[tt]).abs() % math.pi
    return torch.where(sd[rot + 'approx_flag'][tt], s_gauss, s_hist)


def protein_rows(sd, batch, K):
    """(xc_rec, o_rec, h_rec) of FGContextEmbedder for the protein rows (independent of t)."""
    pre = 'context_embedder.'
    br = batch['protein_type_fg_batch']
    x_rec = batch['protein_pos_heavyatom'].float()
    chain_cumsum = batch['protein_num_chains'].cumsum(0)
    chain_nb = torch.cat([batch['protein_chain_nb'][br == i] + chain_cumsum[i] - 1 for i in br.unique()])
    xc_rec = x_rec[:, CA]
    o_rec = OF.rotation_to_so3vec(OF.construct_3d_basis(x_rec[:, CA], x_rec[:, C_], x_rec[:, N_]))
    h_rec = F.linear(F.one_hot(batch['protein_type_fg'], K + 21).float(), sd[pre + 'protein_fg_emb.weight'],
                     sd[pre + 'protein_fg_emb.bias'])
    h_aa = OF.per_residue_encoder(sd, pre + 'residue_emb.', F.one_hot(batch['protein_aa'], 20).float(),
                                  batch['protein_res_nb'], chain_nb, x_rec, batch['protein_mask_heavyatom'])
    h_rec = h_rec + torch.zeros_like(h_rec) + h_aa + indicator(sd, batch['protein_lig_flag'])
    return xc_rec, o_rec, h_rec


def indicator(sd, flag):
    pre = 'context_embedder.ligand_indicator.'
    return F.linear(flag.float().unsqueeze(-1), sd[pre + 'weight'], sd[pre + 'bias'])


def rotation_cosine_loss(R_pred, R0):
    """rotation_matrix_cosine_loss per FG: sum over the three columns of F.cosine_embedding_loss (target 1)."""
    n = R_pred.shape[0]
    a = R_pred.transpose(-2, -1).reshape(n * 3, 3)
    b = R0.transpose(-2, -1).reshape(n * 3, 3)
    loss = F.cosine_embedding_loss(a, b, torch.ones(n * 3, dtype=torch.long), reduction='none')
    return loss.reshape(n, 3).sum(dim=-1)


def eval_losses(sd, batch, t_values, pos_noise, rot_draws, type_uniform, form='score', num_classes=28):
    """Returns (loss_dict, results, per_t, ot): loss_dict / results as the reference's eval-mode forward returns them
    (``form`` 'score' = difffg, 'denoise' = difffg_v2), per_t [R,3] the per-timestep (pos, rot, fg) losses and ot [R,n,3]
    the noised orientations."""
    K = num_classes
    xc0 = batch['ligand_pos_heavyatom'][:, CA].float()
    v0 = batch['ligand_type_fg']
    o0 = batch['ligand_o_fg'].float()
    lig_flag, rec_flag = batch['ligand_lig_flag'], batch['protein_lig_flag']
    gen = batch.get('ligand_gen_flag', lig_flag)
    gen_rec = torch.zeros_like(rec_flag)
    bl, br = batch['ligand_type_fg_batch'], batch['protein_type_fg_batch']
    B = int(bl.max()) + 1
    xc_rec, o_rec, h_rec = protein_rows(sd, batch, K)
    batch_ctx = torch.cat([br, bl])
    sort_idx = torch.sort(batch_ctx, stable=True).indices
    is_lig = torch.cat([rec_flag, lig_flag])[sort_idx]
    cat = lambda a, b: torch.cat([a, b])[sort_idx]
    results, per_t, ots = [], [], []
    for r, t_idx in enumerate(t_values):
        t = torch.full((B,), t_idx, dtype=torch.long)
        # positions (diffusion_scheduler.py:117-134)
        a = sd['pos_scheduler.alphas_cumprod'].index_select(0, t)[bl].unsqueeze(-1)
        noise = pos_noise[r]
        xt = torch.where(gen.unsqueeze(-1), a.sqrt() * xc0 + (1. - a).sqrt() * noise, xc0)
        # orientations (:531-556): o_t = log(exp(e) exp(sqrt(abar) o0)), e ~ angular_distrib_fwd at t
        ar = sd['rot_scheduler.alphas_cumprod'][t[bl]]
        rd = rot_draws[r]
        e = F.normalize(rd[:, 0:3], dim=-1) * forward_angle(sd, t_idx, rd)[:, None]
        R_noisy = OF.so3vec_to_rotation(e) @ OF.so3vec_to_rotation(torch.sqrt(ar).unsqueeze(-1) * o0)
        ot = torch.where(gen[:, None].expand(-1, 3), OF.rotation_to_so3vec(R_noisy), o0)
        # types (:339-346, :380-396)
        log_c0 = log_onehot(v0, K)
        lq = log_add_exp(log_c0 + sd['type_scheduler.log_alphas_cumprod_v'][t][bl].unsqueeze(-1),
                         sd['type_scheduler.log_one_minus_alphas_cumprod_v'][t][bl].unsqueeze(-1) - np.log(K))
        gumbel = -torch.log(-torch.log(type_uniform[r] + 1e-30) + 1e-30)
        vt = torch.where(gen, (gumbel + lq).argmax(dim=-1), v0)
        # embedder, compose, encoder
        h_lig = F.linear(F.one_hot(vt, K + 21).float(), sd['context_embedder.ligand_fg_emb.weight'],
                         sd['context_embedder.ligand_fg_emb.bias'])
        h_lig = h_lig + torch.zeros_like(h_lig) + indicator(sd, lig_flag)
        x, _, _, R, v = OI.ipatransformer_forward(sd, cat(xc_rec, xt), cat(o_rec, ot), cat(h_rec, h_lig),
                                                  batch_ctx[sort_idx], is_lig, cat(gen_rec, gen), prefix='denoiser.')
        x_pred, logits, R_pred = x[is_lig], v[is_lig], R[is_lig]
        # position loss
        if form == 'score':
            sigma = (1 - a.expand_as(x_pred)).sqrt()
            mse = ((x_pred - noise) ** 2).sum(-1)
            pos_info = {'eps_0': noise, 'eps_pred': x_pred, 'score_0': noise * sigma, 'score_pred': x_pred * sigma,
                        'mask_gen': gen}
        else:
            mse = ((x_pred - xc0) ** 2).sum(-1)
            pos_info = {'x0': xc0, 'xt': xt, 'x_pred': x_pred, 'mask_gen': gen}
        loss_pos = scatter_mean(mse[gen], bl[gen], dim=0).mean()
        # rotation loss (difffg.py:16-31)
        R0 = OF.so3vec_to_rotation(o0)
        loss_rot = scatter_mean(rotation_cosine_loss(R_pred, R0)[gen], bl[gen], dim=0).mean()
        # type loss (:348-418)
        log_c_pred = F.log_softmax(logits, dim=-1)
        log_ct = log_onehot(vt, K)
        lp_pred = q_v_posterior(sd, log_c_pred, log_ct, t_idx, K)
        lp_true = q_v_posterior(sd, log_c0, log_ct, t_idx, K)
        kl = (lp_true.exp() * (lp_true - lp_pred)).sum(dim=1)
        nll = -(log_c0.exp() * lp_pred).sum(dim=1)
        mask = (t == 0).float()[bl]
        loss_fg = scatter_mean((mask * nll + (1. - mask) * kl)[gen], bl[gen], dim=0).mean()
        res = dict(pos_info)
        res.update({'v0': v0, 'vt': vt, 'c_pred': log_c_pred.exp(), 'mask_gen': gen})
        res.update({'R0': R0, 'R_pred': R_pred, 'mask_gen': gen})
        results.append(res)
        per_t.append([float(loss_pos), float(loss_rot), float(loss_fg)])
        ots.append(ot)
    per_t = torch.tensor(per_t, dtype=torch.float32)
    loss_dict = {k: torch.mean(torch.tensor(per_t[:, i].tolist())) for i, k in enumerate(('pos', 'rot', 'fg'))}
    return loss_dict, results, per_t, torch.stack(ots)


def noised_angles_f64(sd, batch, t_values, rot_draws):
    """Rotation angle of exp(e) exp(sqrt(abar) o0) in float64 for every timestep and FG [R,n] (with the fp32 draws)."""
    o0 = batch['ligand_o_fg'].double()
    out = []
    for r, t in enumerate(t_values):
        rd = rot_draws[r].double()
        theta = forward_angle(sd, t, rot_draws[r]).double()
        e = F.normalize(rd[:, 0:3], dim=-1) * theta[:, None]
        c0 = sd['rot_scheduler.alphas_cumprod'][t].double().sqrt()
        R = OF.so3vec_to_rotation(e) @ OF.so3vec_to_rotation(c0 * o0)
        out.append(torch.acos(((R.diagonal(dim1=-2, dim2=-1).sum(-1) - 1) / 2).clamp(-1, 1)))
    return torch.stack(out)
