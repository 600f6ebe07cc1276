"""CPU restatement of the reference's TargetDiff sampling loop around the denoiser.

TEST INFRASTRUCTURE (see oracle/__init__.py).

Reference code followed (``/root/reference``):
  repo/models/diffusion/diffusion_scheduler.py:27-100   VPScheduler tables / init_betas
  repo/models/diffusion/diffusion_scheduler.py:137-165  CTNVPScheduler.qxs_x0_xt /
                                                        backward_remove_noise('denoise')
  repo/models/diffusion/diffusion_scheduler.py:320-337  TypeVPScheduler tables
  repo/models/diffusion/diffusion_scheduler.py:367-378  TypeVPScheduler.backward_remove_noise
  repo/models/diffusion/diffusion_scheduler.py:407-441  q_v_posterior / q_v_pred / q_v_pred_one_timestep
  repo/models/utils/categorical.py:26-37                log_sample_categorical / log_add_exp
  repo/modules/context_emb.py:179-231                   PLContextEmbedder.forward (no time emb)
  repo/modules/common.py:189-214                        compose_context (stable sort by graph)
  repo/models/diffusion/targetdiff.py:127-184           TargetDiff.sample

Randomness: the reference draws ``torch.randn_like`` (positions) then ``torch.rand_like``
(type Gumbel) on the model device every step; here both are INJECTED
(``pos_noise[t]``, ``type_uniform[t]``) so CPU oracle and CUDA path see identical noise.
"""
import math
import numpy as np
import torch
import torch.nn.functional as F

from .denoiser import unitransformer_forward

N_AA = 20          # repo/utils/protein/constants.py:39-41 (aa_name_number)


def vp_tables(num_timestep, beta_start=1e-7, beta_end=2e-3, kind='sigmoid', cosine_s=0.008):
    """float64 numpy schedule -> dict of fp32 tensors (diffusion_scheduler.py:27-100)."""
    if kind == 'sigmoid':
        b = np.linspace(-6, 6, num_timestep)
        betas = 1.0 / (np.exp(-b) + 1.0) * (beta_end - beta_start) + beta_start
    elif kind == 'cosine':
        steps = num_timestep + 1
        x = np.linspace(0, steps, steps)
        ac = np.cos(((x / steps) + cosine_s) / (1 + cosine_s) * np.pi * 0.5) ** 2
        ac = ac / ac[0]
        alphas = np.clip(ac[1:] / ac[:-1], a_min=0.001, a_max=1.0)
        betas = 1.0 - np.sqrt(alphas)
    elif kind == 'linear':
        betas = np.linspace(beta_start, beta_end, num_timestep, dtype=np.float64)
    else:
        raise NotImplementedError(kind)
    alphas = 1.0 - betas
    ac = np.cumprod(alphas, axis=0)
    ac_prev = np.append(1.0, ac[:-1])
    post_var = betas * (1.0 - ac_prev) / (1.0 - ac)
    t = {
        'betas': betas, 'alphas': alphas, 'alphas_cumprod': ac, 'alphas_cumprod_prev': ac_prev,
        'sqrt_alphas_cumprod': np.sqrt(ac), 'sqrt_one_minus_alphas_cumprod': np.sqrt(1.0 - ac),
        'sqrt_recip_alphas_cumprod': np.sqrt(1.0 / ac), 'sqrt_recipm1_alphas_cumprod': np.sqrt(1.0 / ac - 1),
        'posterior_mean_c0_coef': betas * np.sqrt(ac_prev) / (1.0 - ac),
        'posterior_mean_ct_coef': (1.0 - ac_prev) * np.sqrt(alphas) / (1.0 - ac),
        'posterior_var': post_var,
    }
    out = {k: torch.from_numpy(np.asarray(v)).float() for k, v in t.items()}
    # diffusion_scheduler.py:54: the log uses the ALREADY fp32-rounded posterior_var parameter
    pv32 = out['posterior_var'].numpy()
    out['posterior_logvar'] = torch.from_numpy(np.log(np.append(pv32[1], pv32[1:]))).float()
    return out


def type_tables(vp):
    """diffusion_scheduler.py:320-337 (computed from the fp32 ``alphas`` parameter)."""
    alphas_v = vp['alphas'].numpy()
    log_a = np.log(alphas_v)
    log_ac = np.cumsum(log_a)
    f = lambda a: np.log(1 - np.exp(a) + 1e-40)
    return {
        'log_alphas_v': torch.from_numpy(log_a).float(),
        'log_one_minus_alphas_v': torch.from_numpy(f(log_a)).float(),
        'log_alphas_cumprod_v': torch.from_numpy(log_ac).float(),
        'log_one_minus_alphas_cumprod_v': torch.from_numpy(f(log_ac)).float(),
    }


def log_add_exp(a, b):
    m = torch.max(a, b)
    return m + torch.log(torch.exp(a - m) + torch.exp(b - m))


def _scalar(v, dtype):
    return torch.as_tensor(v, dtype=dtype)


def pos_reverse_update(x0_pred, x_t, c0, ct, logvar, nonzero, gen_flag, noise):
    """The position update of CTNVPScheduler.backward_remove_noise(type='denoise') for the step's scalars
    (posterior_mean_c0_coef[t], posterior_mean_ct_coef[t], posterior_logvar[t], 0 at t == 0 else 1), in the dtype of
    ``x_t``: fp32 is the reference's expression, float64 a high-precision reference of it on the same inputs."""
    dt = x_t.dtype
    c0, ct, logvar, nonzero = (_scalar(v, dt) for v in (c0, ct, logvar, nonzero))
    mean = c0 * x0_pred.to(dt) + ct * x_t
    xs = mean + nonzero * (0.5 * logvar).exp() * noise.to(dt)
    return torch.where(gen_flag.unsqueeze(-1), xs, x_t)


def pos_reverse_step(sd, x0_pred, x_t, t_idx, gen_flag, noise, prefix='pos_scheduler.'):
    """CTNVPScheduler.backward_remove_noise(type='denoise'), all graphs at the same t."""
    return pos_reverse_update(x0_pred, x_t, sd[prefix + 'posterior_mean_c0_coef'][t_idx],
                              sd[prefix + 'posterior_mean_ct_coef'][t_idx], sd[prefix + 'posterior_logvar'][t_idx],
                              0.0 if t_idx == 0 else 1.0, gen_flag, noise)


def type_reverse_update(logits, c_t, lac, l1mac, la, l1ma, gen_flag, uniform, num_classes):
    """The type update of TypeVPScheduler.backward_remove_noise(pred_logit=True) for the step's scalars
    (log_alphas_cumprod_v / log_one_minus_alphas_cumprod_v at max(t - 1, 0), log_alphas_v / log_one_minus_alphas_v at
    t), in the dtype of ``logits``.  -> (one-hot c_next, v_next, Gumbel score gumbel + log posterior)."""
    K = num_classes
    dt = logits.dtype
    lac, l1mac, la, l1ma = (_scalar(v, dt) for v in (lac, l1mac, la, l1ma))
    c_t, uniform = c_t.to(dt), uniform.to(dt)
    log_c_pred = F.log_softmax(logits, dim=-1)
    log_ct = torch.log(c_t + 1e-8)
    log_qvt1_v0 = log_add_exp(log_c_pred + lac, l1mac - np.log(K))
    log_qvs1_vt = log_add_exp(log_ct + la, l1ma - np.log(K))
    un = log_qvt1_v0 + log_qvs1_vt
    log_post = un - torch.logsumexp(un, dim=-1, keepdim=True)
    gumbel = -torch.log(-torch.log(uniform + 1e-30) + 1e-30)
    score = gumbel + log_post
    v_next = torch.where(gen_flag, score.argmax(dim=-1), c_t.argmax(-1))
    return F.one_hot(v_next, num_classes=K).float(), v_next, score


def type_reverse_step(sd, logits, c_t, t_idx, gen_flag, uniform, num_classes, prefix='type_scheduler.'):
    """TypeVPScheduler.backward_remove_noise(pred_logit=True)."""
    tm1 = max(t_idx - 1, 0)
    c_next, v_next, _ = type_reverse_update(
        logits, c_t, sd[prefix + 'log_alphas_cumprod_v'][tm1], sd[prefix + 'log_one_minus_alphas_cumprod_v'][tm1],
        sd[prefix + 'log_alphas_v'][t_idx], sd[prefix + 'log_one_minus_alphas_v'][t_idx], gen_flag, uniform, num_classes)
    return c_next, v_next


def context_embed(sd, c_lig, v_rec, aa_rec, lig_flag, rec_flag, prefix='context_embedder.'):
    """PLContextEmbedder.forward with time_emb None, atom/residue 'linear' (context_emb.py:179-231)."""
    lin = lambda name, x: F.linear(x, sd[prefix + name + '.weight'], sd[prefix + name + '.bias'])
    if aa_rec.dim() == 1:
        aa_rec = F.one_hot(aa_rec, num_classes=N_AA).float()
    h_lig = lin('ligand_atom_emb', c_lig) + lin('ligand_indicator', lig_flag.float().unsqueeze(-1))
    h_rec = lin('protein_atom_emb', v_rec) + lin('residue_emb', aa_rec) \
        + lin('ligand_indicator', rec_flag.float().unsqueeze(-1))
    return h_lig, h_rec


def compose(batch_idx_lig, batch_idx_rec):
    """compose_context (common.py:189-214): per graph [protein atoms | ligand atoms]."""
    batch_ctx = torch.cat([batch_idx_rec, batch_idx_lig], dim=0)
    sort_idx = torch.sort(batch_ctx, stable=True).indices
    is_lig = torch.cat([torch.zeros_like(batch_idx_rec, dtype=torch.bool),
                        torch.ones_like(batch_idx_lig, dtype=torch.bool)])[sort_idx]
    return sort_idx, batch_ctx[sort_idx], is_lig


def denoise_once(sd, batch, x_lig, c_lig, k=32, cutoff_mode='knn', r_max=10.0):
    """One embed -> compose -> denoiser pass (targetdiff.py:155-165). Returns (x0_pred, logits) on ligand rows."""
    lig_flag = batch['ligand_lig_flag']
    rec_flag = batch['protein_lig_flag']
    gen_lig = batch.get('ligand_gen_flag', lig_flag)
    gen_rec = batch.get('protein_gen_flag', torch.zeros_like(rec_flag))
    bl, br = batch['ligand_element_batch'], batch['protein_element_batch']
    h_lig, h_rec = context_embed(sd, c_lig, batch['protein_atom_feature'], batch['protein_aa_type'],
                                 lig_flag, rec_flag)
    sort_idx, batch_idx, _ = compose(bl, br)
    x = torch.cat([batch['protein_pos'], x_lig], 0)[sort_idx]
    h = torch.cat([h_rec, h_lig], 0)[sort_idx]
    gen = torch.cat([gen_rec, gen_lig], 0)[sort_idx]
    lig = torch.cat([rec_flag, lig_flag], 0)[sort_idx]
    x_o, h_o, c_o = unitransformer_forward(sd, x, h, batch_idx, lig, gen, k=k,
                                           cutoff_mode=cutoff_mode, r_max=r_max)
    return x_o[lig], c_o[lig]


def sample(sd, batch, num_steps, pos_noise, type_uniform, num_classes=13, k=32,
           cutoff_mode='knn', r_max=10.0, stop_after=None):
    """TargetDiff.sample (targetdiff.py:127-184) with injected noise.

    pos_noise[t] [N_lig,3], type_uniform[t] [N_lig,K] indexed by the step's t_idx.
    Returns traj dict t -> (x_lig, c_lig) with keys T-1 ... -1 (or down to the last
    executed step when ``stop_after`` limits the number of steps)."""
    x = batch['ligand_pos'].float()
    c = F.one_hot(batch['ligand_atom_type'], num_classes=num_classes).float()
    gen_lig = batch.get('ligand_gen_flag', batch['ligand_lig_flag'])
    traj = {num_steps - 1: (x, c)}
    done = 0
    for t_idx in reversed(range(num_steps)):
        x, c = traj[t_idx]
        x0, logits = denoise_once(sd, batch, x, c, k=k, cutoff_mode=cutoff_mode, r_max=r_max)
        x_next = pos_reverse_step(sd, x0, x, t_idx, gen_lig, pos_noise[t_idx])
        c_next, _ = type_reverse_step(sd, logits, c, t_idx, gen_lig, type_uniform[t_idx], num_classes)
        traj[t_idx - 1] = (x_next, c_next)
        done += 1
        if stop_after is not None and done >= stop_after:
            break
    return traj
