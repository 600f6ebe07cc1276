"""CPU restatement of the reference's eval-mode TargetDiff.forward (the validation losses).

TEST INFRASTRUCTURE, like oracle/: written from the reference as it reads, one timestep at a time with materialised
tensors, on top of the sampling oracle's embed / compose / denoiser restatement (oracle/diffusion.py: denoise_once).

Reference code followed (``repo/`` of the reference checkout):
  models/diffusion/targetdiff.py:41-124             TargetDiff.forward (eval branch) / get_loss
  models/diffusion/diffusion_scheduler.py:117-134   CTNVPScheduler.forward_add_noise
  models/diffusion/diffusion_scheduler.py:185-201   CTNVPScheduler.get_loss (type='denoise')
  models/diffusion/diffusion_scheduler.py:339-418   TypeVPScheduler.forward_add_noise / get_loss / qct_c0_* /
                                                    compute_loss / q_v_posterior
  models/utils/categorical.py:5-37                  index_to_log_onehot, categorical_kl, log_categorical,
                                                    log_sample_categorical, log_add_exp
  modules/common.py:33-42                           get_dict_mean

Randomness is INJECTED: ``pos_noise[r]`` replaces the ``randn_like`` of timestep r and ``type_uniform[r]`` its
``rand_like``.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import diffusion as OD
from oracle.graph_ops import scatter_mean


def eval_t_values(num_timesteps, eval_interval=10):
    """targetdiff.py:67-71: np.linspace, then torch.tensor([t] * B).long() (truncation toward zero)."""
    return [int(torch.tensor([t]).long()) for t in np.linspace(0, num_timesteps - 1, eval_interval)]


def log_onehot(v, K):
    return torch.log(F.one_hot(v, K).float().clamp(min=1e-30))


def q_v_posterior(sd, log_v0, log_vt, t, K, prefix='type_scheduler.'):
    tm1 = max(t - 1, 0)
    lac, l1mac = sd[prefix + 'log_alphas_cumprod_v'][tm1], sd[prefix + 'log_one_minus_alphas_cumprod_v'][tm1]
    la, l1ma = sd[prefix + 'log_alphas_v'][t], sd[prefix + 'log_one_minus_alphas_v'][t]
    a = OD.log_add_exp(log_v0 + lac, l1mac - np.log(K))
    b = OD.log_add_exp(log_vt + la, l1ma - np.log(K))
    un = a + b
    return un - torch.logsumexp(un, dim=-1, keepdim=True)


def eval_losses(sd, batch, t_values, pos_noise, type_uniform, num_classes=13, k=32, cutoff_mode='knn', r_max=10.0):
    """Returns (loss_dict, results, per_t) with loss_dict / results as the reference's eval-mode forward returns them
    and per_t = [(pos, atom)] the per-timestep losses."""
    K = num_classes
    x0 = batch['ligand_pos'].float()
    v0 = batch['ligand_atom_type']
    gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag'])
    bl = batch['ligand_element_batch']
    results, per_t = [], []
    for r, t in enumerate(t_values):
        # forward noising of positions (diffusion_scheduler.py:117-134)
        a = sd['pos_scheduler.alphas_cumprod'][t]
        x_noisy = a.sqrt() * x0 + (1. - a).sqrt() * pos_noise[r]
        xt = torch.where(gen.unsqueeze(-1), x_noisy, x0)
        # forward noising of types: q(v_t | v_0) Gumbel sample (:339-346, :380-396)
        log_c0 = log_onehot(v0, K)
        lq = OD.log_add_exp(log_c0 + sd['type_scheduler.log_alphas_cumprod_v'][t],
                            sd['type_scheduler.log_one_minus_alphas_cumprod_v'][t] - np.log(K))
        gumbel = -torch.log(-torch.log(type_uniform[r] + 1e-30) + 1e-30)
        vt = torch.where(gen, (gumbel + lq).argmax(dim=-1), v0)
        # embed -> compose -> denoiser on the ligand rows
        x_pred, logits = OD.denoise_once(sd, batch, xt, F.one_hot(vt, K).float(), k=k, cutoff_mode=cutoff_mode, r_max=r_max)
        # position loss (:185-201, type='denoise')
        mse = ((x_pred - x0) ** 2).sum(-1)
        loss_pos = scatter_mean(mse[gen], bl[gen], dim=0).mean()
        # type loss (:348-418)
        log_c_pred = F.log_softmax(logits, dim=-1)
        log_ct = log_onehot(vt, K)
        lp_pred = q_v_posterior(sd, log_c_pred, log_ct, t, K)
        lp_true = q_v_posterior(sd, log_c0, log_ct, t, K)
        kl = (lp_true.exp() * (lp_true - lp_pred)).sum(dim=1)
        nll = -(log_c0.exp() * lp_pred).sum(dim=1)
        mask = 1.0 if t == 0 else 0.0
        loss_atom = scatter_mean((mask * nll + (1. - mask) * kl)[gen], bl[gen], dim=0).mean()
        per_t.append((loss_pos, loss_atom))
        results.append({'x0': x0, 'xt': xt, 'x_pred': x_pred, 'mask_gen': gen, 'v0': v0, 'vt': vt,
                        'c_pred': log_c_pred.exp()})
    loss_dict = {'pos': torch.mean(torch.tensor([p for p, _ in per_t])),
                 'atom': torch.mean(torch.tensor([a for _, a in per_t]))}
    return loss_dict, results, per_t


def auroc(results, true_key='v0', pred_key='c_pred', mask_key='mask_gen'):
    """The reference's AUROC evaluator (utils/evaluate.py: merge_list_of_dict + AUROC.cal_auroc), restated."""
    from sklearn.metrics import roc_auc_score
    merged = {k: torch.cat([res[k] for res in results], dim=0) for k in results[0]}
    y_true, y_pred = merged[true_key], merged[pred_key]
    mask = merged[mask_key] if mask_key is not None else torch.ones_like(y_true, dtype=torch.bool)
    y_true = y_true[mask].cpu().numpy()
    y_pred = y_pred[mask].cpu().numpy()
    total = 0.
    for c in set(y_true):
        try:
            total += roc_auc_score(y_true == c, y_pred[:, c]) * np.sum(y_true == c)
        except ValueError:
            pass
    return np.divide(total, len(y_true))
