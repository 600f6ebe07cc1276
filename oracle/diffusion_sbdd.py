"""CPU restatement of the reference's DiffSBDD sampling loop (SURVEY.md section 8 row f2).

TEST INFRASTRUCTURE (see oracle/__init__.py).

Reference code followed (``/root/reference``):
  repo/models/diffusion/schedule_utils.py:7-21,45-96      clip_noise_schedule, polynomial_schedule,
                                                          PredefinedNoiseSchedule (gamma lookup table)
  repo/models/diffusion/diffusion_scheduler.py:706-710    remove_mean_batch (ligand COM, applied to the pocket too)
  repo/models/diffusion/diffusion_scheduler.py:721-729    sigma / alpha from gamma
  repo/models/diffusion/diffusion_scheduler.py:963-976    sample_normal_zero_com
  repo/models/diffusion/diffusion_scheduler.py:978-1003   sigma_and_alpha_t_given_s
  repo/models/diffusion/diffusion_scheduler.py:1005-1039  sample_p_zs_given_zt
  repo/models/diffusion/diffsbdd.py:92-96,207-211         normalize / unnormalize (pos: identity, type: /4, *4)
  repo/models/diffusion/diffsbdd.py:240-321               DiffSBDD.sample
  repo/models/diffusion/diffsbdd.py:323-360               sample_p_xh_given_z0 / compute_pred

Reference quirks kept on purpose:
  * the denoiser's OUTPUT coordinates of the ligand atoms are used as the noise prediction eps_t
    (diffsbdd.py:299-305; ``zero_com_translate`` is defined but never called);
  * the pocket moves: every COM projection subtracts the ligand mean from the pocket atoms too;
  * the final ``c_lig`` returned is 4 x the INPUT of the last stage - the freshly sampled ``v_lig_in`` is
    discarded (diffsbdd.py:348-352), its random numbers are still drawn;
  * nothing in the reverse step looks at ``gen_flag`` (only the denoiser's coordinate update does).

Randomness: the reference calls ``torch.randn`` (init: x then c; every step: x then c; final stage: x then c).
Here all of it is INJECTED: noise = {'init_x','init_c','step_x'[t],'step_c'[t],'final_x','final_c'}.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import graph_ops as G
from .denoiser import unitransformer_forward
from .diffusion import context_embed, compose

TYPE_NORM = 4.0     # diffsbdd.py:95-96 normalize_type(std=4)


def gamma_table(timesteps, power=2.0, precision=5e-4):
    """'polynomial_<power>' schedule -> gamma[T+1] fp32 (schedule_utils.py:45-96)."""
    steps = timesteps + 1
    x = np.linspace(0, steps, steps)
    alphas2 = (1 - np.power(x / steps, power)) ** 2
    a2 = np.concatenate([np.ones(1), alphas2], axis=0)
    step = np.clip(a2[1:] / a2[:-1], a_min=0.001, a_max=1.0)
    alphas2 = np.cumprod(step, axis=0)
    alphas2 = (1 - 2 * precision) * alphas2 + precision
    sigmas2 = 1 - alphas2
    return torch.from_numpy(-(np.log(alphas2) - np.log(sigmas2))).float()


def gamma_at(gamma, t, timesteps):
    """PredefinedNoiseSchedule.forward (schedule_utils.py:94-96): t in [0,1] -> gamma[round(t*T)]."""
    return gamma[torch.round(t * timesteps).long()]


def step_scalars(gamma, t_idx, timesteps):
    """Per-step scalars of sample_p_zs_given_zt (all graphs share s, t): fp32 0-d tensors
    alpha_ts, k_eps = sigma2_ts / alpha_ts / sigma_t, sigma = sigma_ts * sigma_s / sigma_t."""
    s = torch.tensor([t_idx], dtype=torch.int64) / timesteps            # diffsbdd.py:283-287 (int / int -> fp32)
    t = (torch.tensor([t_idx], dtype=torch.int64) + 1) / timesteps
    g_s, g_t = gamma_at(gamma, s, timesteps), gamma_at(gamma, t, timesteps)
    sigma2_ts = -torch.expm1(F.softplus(g_s) - F.softplus(g_t))
    alpha_ts = torch.exp(0.5 * (F.logsigmoid(-g_t) - F.logsigmoid(-g_s)))
    sigma_ts = torch.sqrt(sigma2_ts)
    sigma_s, sigma_t = torch.sqrt(torch.sigmoid(g_s)), torch.sqrt(torch.sigmoid(g_t))
    return alpha_ts[0], (sigma2_ts / alpha_ts / sigma_t)[0], (sigma_ts * sigma_s / sigma_t)[0]


def final_scalars(gamma, timesteps):
    """sample_p_xh_given_z0 (diffsbdd.py:326-329, 354-360): 1/alpha_0 is applied as ``1. / alpha * (...)``."""
    g0 = gamma_at(gamma, torch.zeros(1), timesteps)
    return torch.sqrt(torch.sigmoid(-g0))[0], torch.sqrt(torch.sigmoid(g0))[0], torch.exp(0.5 * g0)[0]


def remove_mean_batch(x_lig, x_rec, bl, br, num_graphs=None):
    """diffusion_scheduler.py:706-710.  ``num_graphs`` sizes the mean table: without it a trailing graph without ligand
    atoms indexes past the table when its pocket is moved (the reference's own behaviour); with it such a graph's
    mean is 0 and its pocket does not move."""
    mean = G.scatter_mean(x_lig, bl, dim=0, dim_size=num_graphs)
    return x_lig - mean[bl], x_rec - mean[br]


def reverse_update(z_t, eps, a, b, s, noise, mode=0):
    """z_s before the COM projection, for the step's scalars, in the dtype of ``z_t``:
    mode 0  sample_p_zs_given_zt (a = alpha_t|s, b = sigma2_t|s / alpha_t|s / sigma_t, s = sigma_t|s sigma_s / sigma_t):
            z_t / a - b eps + s noise
    mode 1  sample_p_xh_given_z0 (a = 1 / alpha_0, b = sigma_0, s = exp(0.5 gamma_0)): a (z_t - b eps) + s noise."""
    dt = z_t.dtype
    a, b, s = (torch.as_tensor(v, dtype=dt) for v in (a, b, s))
    eps, noise = eps.to(dt), noise.to(dt)
    mu = z_t / a - b * eps if mode == 0 else a * (z_t - b * eps)
    return mu + s * noise


def denoise(sd, batch, x_lig, c_lig, x_rec, v_rec, k, cutoff_mode, r_max):
    """embed -> compose -> denoiser with the CURRENT pocket coordinates (diffsbdd.py:289-300)."""
    lig_flag, rec_flag = batch['ligand_lig_flag'], batch['protein_lig_flag']
    gen_lig = batch.get('ligand_gen_flag', lig_flag)
    gen_rec = batch.get('protein_gen_flag', torch.zeros_like(rec_flag))
    bl, br = batch['ligand_element_batch'], batch['protein_element_batch']
    h_lig, h_rec = context_embed(sd, c_lig, v_rec, batch['protein_aa_type'], lig_flag, rec_flag)
    sort_idx, batch_idx, _ = compose(bl, br)
    x = torch.cat([x_rec, x_lig], 0)[sort_idx]
    h = torch.cat([h_rec, h_lig], 0)[sort_idx]
    gen = torch.cat([gen_rec, gen_lig], 0)[sort_idx]
    lig = torch.cat([rec_flag, lig_flag], 0)[sort_idx]
    x_o, _, c_o = unitransformer_forward(sd, x, h, batch_idx, lig, gen, k=k, cutoff_mode=cutoff_mode, r_max=r_max)
    return x_o[lig], c_o[lig]


def sample(sd, batch, num_steps, noise, num_classes=13, k=32, cutoff_mode='knn', r_max=10.0, stop_after=None):
    """DiffSBDD.sample with injected noise.  Returns (traj, x_rec_final): traj t -> (x_lig, c_lig) for keys
    T-1 ... -1, and - when the loop ran to the end - traj[0] overwritten by the final stage like the reference."""
    T = num_steps
    gamma = sd['pos_scheduler.gamma.gamma']
    bl, br = batch['ligand_element_batch'], batch['protein_element_batch']
    x_rec = batch['protein_pos'].float()
    v_rec = batch['protein_atom_feature'].float() / TYPE_NORM
    mu = G.scatter_mean(x_rec, br, dim=0)[bl]
    x_lig, x_rec = remove_mean_batch(mu + noise['init_x'], x_rec, bl, br)     # sigma = 1 (diffsbdd.py:258)
    c_lig = torch.zeros_like(noise['init_c']) + noise['init_c']
    traj = {T - 1: (x_lig, c_lig)}
    done = 0
    complete = True
    for t_idx in reversed(range(T)):
        x_lig, c_lig = traj[t_idx]
        x_pred, c_out = denoise(sd, batch, x_lig, c_lig, x_rec, v_rec, k, cutoff_mode, r_max)
        a_ts, k_eps, sig = step_scalars(gamma, t_idx, T)
        zs = reverse_update(x_lig, x_pred, a_ts, k_eps, sig, noise['step_x'][t_idx])
        x_next, x_rec = remove_mean_batch(zs, x_rec, bl, br)
        c_next = reverse_update(c_lig, c_out, a_ts, k_eps, sig, noise['step_c'][t_idx])
        traj[t_idx - 1] = (x_next, c_next)
        done += 1
        if stop_after is not None and done >= stop_after:
            complete = t_idx == 0
            break
    if complete:
        x_lig, c_lig = traj[-1]
        x_pred, _ = denoise(sd, batch, x_lig, c_lig, x_rec, v_rec, k, cutoff_mode, r_max)
        alpha0, sigma0, sigma_x = final_scalars(gamma, T)
        zs = reverse_update(x_lig, x_pred, 1.0 / alpha0, sigma0, sigma_x, noise['final_x'], mode=1)
        x_fin, _ = remove_mean_batch(zs, x_rec, bl, br)
        traj[0] = (x_fin, c_lig * TYPE_NORM)
    return traj, x_rec
