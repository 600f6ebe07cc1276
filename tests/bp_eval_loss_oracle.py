"""CPU restatement of the reference's eval-mode DiffBP.forward (the validation losses).

TEST INFRASTRUCTURE, like oracle/: written from the reference as it reads, one timestep at a time with materialised
tensors, on top of the sampling oracle's embed / compose / denoiser / CoM-head restatement (oracle/diffusion_bp.py).

Reference code followed (``repo/`` of the reference checkout):
  models/diffusion/diffbp.py:19-30                  interior_loss (torch_geometric.nn.knn, k = 48, rho = 2, gamma = 5)
  models/diffusion/diffbp.py:133-230                DiffBP.forward (eval branch) / get_loss / get_mean_xs_lig
  models/diffusion/diffusion_scheduler.py:117-134   CTNVPScheduler.forward_add_noise(zero_center=True)
  models/diffusion/diffusion_scheduler.py:167-182   CTNVPScheduler.xs_mean (type='score')
  models/diffusion/diffusion_scheduler.py:203-219   CTNVPScheduler.get_score_loss
  models/diffusion/diffusion_scheduler.py:452-511   MaskTypeSchedule.forward_add_noise / get_loss
  modules/common.py:33-42                           get_dict_mean

Randomness is INJECTED: ``pos_noise[r]`` [n_lig,3] replaces the ``randn_like`` of timestep r and ``type_uniform[r]``
[n_lig] its ``rand_like``.

``knn`` below restates ``torch_geometric.nn.knn`` (pytorch-cluster), which the reference imports unpinned like
``knn_graph`` (oracle/graph_ops.py).  Our definition: for every y[j], the min(k, n_x_g) nearest x of the same graph by
the fp32 squared distance of oracle.graph_ops.pairwise_sqdist_f32, nearest first, ties to the lower x index; the edge
index is [2,E] = [y index ; x index], grouped by y.
"""
import torch
import torch.nn.functional as F

from oracle import diffusion_bp as OB
from oracle.graph_ops import pairwise_sqdist_f32, scatter_add, scatter_mean

from eval_loss_oracle import auroc, eval_t_values  # noqa: F401  (same timesteps and evaluator as TargetDiff)

INTER_K, INTER_RHO, INTER_GAMMA = 48, 2, 5
RESULT_KEYS = ('eps_0', 'eps_pred', 'score_0', 'score_pred', 'mask_gen', 'v0', 'vt', 'c_pred',
               'eps_0_com', 'eps_pred_com', 'score_0_com', 'score_pred_com', 'mask_gen_com')


def knn(x, y, k, batch_x=None, batch_y=None, **_):
    """torch_geometric.nn.knn(x, y, k, batch_x, batch_y) with the definition of the module docstring."""
    x, y = x.detach().float().cpu(), y.detach().float().cpu()
    bx = torch.zeros(x.shape[0], dtype=torch.int64) if batch_x is None else batch_x.cpu().long()
    by = torch.zeros(y.shape[0], dtype=torch.int64) if batch_y is None else batch_y.cpu().long()
    rows, cols = [], []
    for g in torch.unique(by).tolist():
        iy = torch.nonzero(by == g).flatten()
        ix = torch.nonzero(bx == g).flatten()
        if ix.numel() == 0:
            continue
        d2 = pairwise_sqdist_f32(y[iy], x[ix])
        order = torch.sort(d2, dim=1, stable=True).indices[:, :min(k, ix.numel())]     # stable: lower index on ties
        rows.append(iy[:, None].expand_as(order).reshape(-1))
        cols.append(ix[order].reshape(-1))
    if not rows:
        return torch.zeros(2, 0, dtype=torch.int64)
    return torch.stack([torch.cat(rows), torch.cat(cols)], 0)


def interior_loss(x_ligand, x_protein, batch_ligand, batch_protein, k=INTER_K, rho=INTER_RHO, gamma=INTER_GAMMA):
    """diffbp.py:19-30, with ``knn`` above."""
    protein_idx, ligand_idx = knn(x_ligand, x_protein, k, batch_ligand, batch_protein)
    dist2 = torch.square(x_ligand[ligand_idx] - x_protein[protein_idx]).sum(dim=-1)
    s = scatter_add(torch.divide(-dist2, rho).exp(), ligand_idx, dim=0, dim_size=x_ligand.size(0))
    return torch.clamp(gamma - (-rho * (s + 1e-3).log()), min=0.).mean()


def mask_prob(t, T):
    """MaskTypeSchedule.forward_add_noise: t.float().clamp(min=0) / num_timestep in fp32."""
    return (torch.tensor([t]).float().clamp(min=0.) / T)[0]


def eval_losses(sd, batch, t_values, pos_noise, type_uniform, T, num_classes=13, k=32):
    """Returns (loss_dict, results, per_t): loss_dict / results as the reference's eval-mode forward returns them and
    per_t = [(pos, atom, com, inter)] the per-timestep losses."""
    K = num_classes
    x0 = batch['ligand_pos'].float()
    v0 = batch['ligand_atom_type']
    gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag'])
    bl, br = batch['ligand_element_batch'], batch['protein_element_batch']
    results, per_t = [], []
    for r, t in enumerate(t_values):
        a = sd['pos_scheduler.alphas_cumprod'][t]
        b = sd['pos_scheduler.betas'][t]
        sigma = (1 - a).sqrt()
        # positions: raw noise in x_t, zero-centred noise as the target, its graph mean as the CoM target
        eps = pos_noise[r]
        com_noise = scatter_mean(eps, bl, dim=0)[bl]
        pos_noise_t = eps - com_noise
        xt = torch.where(gen.unsqueeze(-1), a.sqrt() * x0 + (1. - a).sqrt() * eps, x0)
        # types: absorbing-state mask with probability t / T
        mask = (type_uniform[r] < mask_prob(t, T)) & gen.bool()
        vt = torch.where(mask, 0, v0)
        eps_pred, com_pred, logits = OB.denoise(sd, batch, xt, F.one_hot(vt, K).float(), k=k)
        # score losses (score_in=False: the targets are the noises themselves)
        loss_pos = scatter_mean(((eps_pred - pos_noise_t) ** 2).sum(-1)[gen], bl[gen], dim=0).mean()
        loss_com = scatter_mean(((com_pred - com_noise) ** 2).sum(-1)[gen], bl[gen], dim=0).mean()
        # masked-type cross-entropy of the softmax probabilities (pred_logit=True)
        c_pred = F.softmax(logits, dim=-1)
        la = scatter_mean(F.cross_entropy(c_pred, v0, reduction='none')[mask], bl[mask], dim=0)
        if len(la) == 0:
            la = torch.zeros_like(v0).float()
        loss_atom = la.mean()
        # interior loss on the posterior mean of x_{t-1}
        xs = (xt + b * (-(eps_pred + com_pred) / sigma)) / (1 - b).sqrt()
        xs_mean = torch.where(gen.unsqueeze(-1), xs, xt)
        loss_inter = interior_loss(xs_mean, batch['protein_pos'].float(), bl, br)
        per_t.append((loss_pos, loss_atom, loss_com, loss_inter))
        results.append({'eps_0': pos_noise_t, 'eps_pred': eps_pred, 'score_0': pos_noise_t * sigma,
                        'score_pred': eps_pred * sigma, 'mask_gen': mask, 'v0': v0,
                        'vt': F.one_hot(vt, K).float(), 'c_pred': c_pred,
                        'eps_0_com': com_noise, 'eps_pred_com': com_pred, 'score_0_com': com_noise * sigma,
                        'score_pred_com': com_pred * sigma, 'mask_gen_com': gen})
    names = ('pos', 'atom', 'com', 'inter')
    loss_dict = {n: torch.mean(torch.tensor([float(p[i]) for p in per_t])) for i, n in enumerate(names)}
    return loss_dict, results, per_t
