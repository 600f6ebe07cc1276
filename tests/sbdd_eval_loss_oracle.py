"""CPU restatement of the reference's eval-mode DiffSBDD.forward (the validation losses).

TEST INFRASTRUCTURE, like oracle/: written from the reference as it reads, one timestep at a time with materialised
tensors, on top of the sampling oracle's embed / compose / denoiser restatement (oracle/diffusion_sbdd.py: denoise).

Reference code followed (``repo/`` of the reference checkout):
  models/diffusion/diffsbdd.py:48-191                DiffSBDD.forward (eval branch) / get_loss: two noised copies per t,
                                                     at t and at 0, each through the denoiser
  models/diffusion/diffusion_scheduler.py:670-963    DiffsbddVariationalScheduler: remove_mean_batch,
                                                     forward_pos_center_noise, forward_type_add_noise, kl_prior,
                                                     log_constants_p_x_given_z0, log_ph_given_z0_discrete,
                                                     calculate_loss_t_non_training, calculate_loss_0_non_training,
                                                     get_score_loss (eval branch)
  modules/common.py:33-42                            get_dict_mean

Randomness is INJECTED: ``noise['x_t'][j]``, ``noise['c_t'][j]``, ``noise['x_0'][j]``, ``noise['c_0'][j]`` replace the four
``randn_like`` draws of timestep j, in that (the reference's) order.

The per-graph terms have B = (last ligand graph id) + 1 rows like the reference's scatter_add.  Pocket atoms of a graph
after the last ligand graph (where the reference's ``mean[batch_idx_rec]`` would index past B) keep their input
coordinates here: the means of a graph without ligand atoms are 0.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import diffusion_sbdd as OS
from oracle.graph_ops import scatter_add, scatter_mean

TYPE_NORM = 4
LOG_2PI_HALF = 0.5 * np.log(2 * np.pi)
RESULT_KEYS = ('eps_0_pos', 'eps_pred_pos', 'score_0_pos', 'score_pred_pos', 'mask_gen_pos',
               'eps_0_atom', 'eps_pred_atom', 'score_0_atom', 'score_pred_atom', 'mask_gen_atom')
TERM_NAMES = ('pos_t', 'pos_0', 'pos_kl', 'atom_t', 'atom_0', 'atom_kl')


def eval_t_values(num_timesteps, eval_interval=10):
    """diffsbdd.py:71-77: np.linspace(1, T, eval_interval), then torch.tensor([t] * B).long() (truncation)."""
    return [int(torch.tensor([t]).long()) for t in np.linspace(1, num_timesteps, eval_interval)]


def cdf_standard_gaussian(x):
    return 0.5 * (1. + torch.erf(x / math.sqrt(2)))


def schedule(gamma, t_int, T):
    """gamma at s = (t-1)/T, t/T, 0 and 1 (fp32, like get_loss's s / t and the t_zeros / ones of the scheduler)."""
    tt = torch.tensor([t_int]).long()
    g = lambda v: OS.gamma_at(gamma, v, T)
    return g((tt - 1) / T), g(tt / T), g(torch.zeros(1)), g(torch.ones(1))


def alpha_sigma(g):
    return torch.sqrt(torch.sigmoid(-g)), torch.sqrt(torch.sigmoid(g))


def gaussian_kl(mu2, sigma_T, d):
    """gaussian_KL(mu2, q_sigma=sigma_T, p_sigma=1, d) (diffusion_scheduler.py:695-704)."""
    p = torch.ones_like(sigma_T)
    return d * torch.log(p / sigma_T) + 0.5 * (d * sigma_T ** 2 + mu2) / (p ** 2) - 0.5 * d


def eval_losses(sd, batch, t_values, noise, T, num_classes=13, k=32):
    """Returns (loss_dict, results, per_t, terms): loss_dict / results as the reference's eval-mode forward returns them,
    per_t = [(pos, atom)] the per-timestep losses and terms [n_t, B, 6] the per-graph TERM_NAMES."""
    K = num_classes
    g_pos, g_type = sd['pos_scheduler.gamma.gamma'], sd['type_scheduler.gamma.gamma']
    x0 = batch['ligand_pos'].float()
    v0 = batch['ligand_atom_type']
    gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag'])
    bl, br = batch['ligand_element_batch'], batch['protein_element_batch']
    n_graphs = int(torch.cat([bl, br]).max()) + 1
    B = int(bl.max()) + 1
    x_rec = batch['protein_pos'].float()
    v_rec = batch['protein_atom_feature'].float() / TYPE_NORM
    # clean state: zero ligand CoM (the pocket moves with it), continuous types onehot / 4
    mean = scatter_mean(x0, bl, dim=0, dim_size=n_graphs)
    x0c, xrc = x0 - mean[bl], x_rec - mean[br]
    c0 = F.one_hot(v0, K) / TYPE_NORM
    n = torch.bincount(bl)
    dof_pos, dof_type = (n - 1) * 3, (n - 1) * K

    def noised(x_eps, c_eps, g_p, g_c):
        """forward_pos_center_noise (zero_center=False) + forward_type_add_noise at one gamma pair."""
        a, s = alpha_sigma(g_p)
        xn = a * x0c + s * x_eps
        m = scatter_mean(xn, bl, dim=0, dim_size=n_graphs)
        x_lig = torch.where(gen.unsqueeze(-1), xn - m[bl], x0c)
        ac, sc = alpha_sigma(g_c)
        c = torch.where(gen.unsqueeze(-1), ac * c0 + sc * c_eps, c0)
        return x_lig, xrc - m[br], c

    results, per_t, terms = [], [], []
    for j, t in enumerate(t_values):
        gs_p, gt_p, g0_p, gT_p = schedule(g_pos, t, T)
        gs_c, gt_c, g0_c, gT_c = schedule(g_type, t, T)
        ex_t, ec_t, ex_0, ec_0 = noise['x_t'][j], noise['c_t'][j], noise['x_0'][j], noise['c_0'][j]
        x_lig, x_r, c_t = noised(ex_t, ec_t, gt_p, gt_c)
        xp_t, cp_t = OS.denoise(sd, batch, x_lig, c_t, x_r, v_rec, k, 'knn', 10.0)
        x_lig, x_r, c_z = noised(ex_0, ec_0, g0_p, g0_c)
        xp_0, _ = OS.denoise(sd, batch, x_lig, c_z, x_r, v_rec, k, 'knn', 10.0)   # its logits are not read
        err = lambda p, q: scatter_add(((q - p) ** 2).sum(-1), bl, dim=0)
        # positions: loss_t with the SNR weight, loss_0 of the t = 0 copy, KL to the prior at T
        pos_t = -T * 0.5 * (1 - torch.exp(-(gs_p - gt_p))) * err(xp_t, ex_t)
        pos_0 = -(-0.5 * err(xp_0, ex_0)) + -(dof_pos * (-(0.5 * g0_p) - LOG_2PI_HALF))
        aT, sT = alpha_sigma(gT_p)
        pos_kl = gaussian_kl(scatter_add(((aT * x0c) ** 2).sum(-1), bl, dim=0), sT, dof_pos)
        # types: loss_t as above; loss_0 is the discretised likelihood of the t = 0 copy's noised types
        atom_t = -T * 0.5 * (1 - torch.exp(-(gs_c - gt_c))) * err(cp_t, ec_t)
        sigma0 = torch.sqrt(torch.sigmoid(g0_c)) * TYPE_NORM
        centered = (c_z * TYPE_NORM + 0.0) - 1
        lp = torch.log(cdf_standard_gaussian((centered + 0.5) / sigma0) - cdf_standard_gaussian((centered - 0.5) / sigma0)
                       + 1e-10)
        logp = lp - torch.logsumexp(lp, dim=1, keepdim=True)
        log_ph = scatter_add((logp * (c0 * TYPE_NORM + 0.0)).sum(-1), bl, dim=0)
        atom_0 = -log_ph + -(dof_type * (-(0.5 * g0_c) - LOG_2PI_HALF))
        aTc, sTc = alpha_sigma(gT_c)
        atom_kl = gaussian_kl(scatter_add(((aTc * c0) ** 2).sum(-1), bl, dim=0), sTc, 1)
        per_t.append(((pos_t + pos_0 + pos_kl).mean(), (atom_t + atom_0 + atom_kl).mean()))
        terms.append(torch.stack([pos_t, pos_0, pos_kl, atom_t, atom_0, atom_kl], 1))
        assert terms[-1].shape == (B, 6)
        sp, sc = alpha_sigma(gt_p)[1], alpha_sigma(gt_c)[1]
        results.append({'eps_0_pos': ex_t, 'eps_pred_pos': xp_t, 'score_0_pos': ex_t * sp, 'score_pred_pos': xp_t * sp,
                        'mask_gen_pos': gen, 'eps_0_atom': ec_t, 'eps_pred_atom': cp_t, 'score_0_atom': ec_t * sc,
                        'score_pred_atom': cp_t * sc, 'mask_gen_atom': gen})
    loss_dict = {name: torch.mean(torch.tensor([float(p[i]) for p in per_t])) for i, name in enumerate(('pos', 'atom'))}
    return loss_dict, results, per_t, torch.stack(terms)
