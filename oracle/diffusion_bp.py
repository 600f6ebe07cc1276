"""CPU restatement of the reference's DiffBP sampling loop (SURVEY.md section 8 row f2).

TEST INFRASTRUCTURE (see oracle/__init__.py).

Reference code followed (``/root/reference``):
  repo/models/diffusion/diffbp.py:30-101     CoMPredictor (own kNN graph on the step's INPUT coordinates, own edge
                                             gate, 3 x H2XAttention on the denoiser's FINAL h, gen-masked updates;
                                             returns the zero-mean noise prediction and the per-graph mean shift)
  repo/models/diffusion/diffbp.py:236-238    get_xs_lig -> pos_scheduler.backward_remove_noise(eps + eps_com, x_t, ...)
  repo/models/diffusion/diffbp.py:240-299    DiffBP.sample
  repo/models/diffusion/diffusion_scheduler.py:144-165   CTNVPScheduler.backward_remove_noise, type='score' branch
  repo/models/diffusion/diffusion_scheduler.py:444-498   MaskTypeSchedule.backward_remove_noise
  repo/utils/molecule/constants.py:8                     absorbing_state = 0

The com head's kNN graph is built from the same coordinates and the same k as the denoiser's graph of the step, so the
neighbour table is shared (cfg.encoder.k feeds both, diffbp.py:42,128; unitransformer.py:79-80).

Randomness: ``torch.randn_like`` (positions, diffusion_scheduler.py:158) then ``torch.rand_like`` (type change mask,
:486) per step; both INJECTED here (``pos_noise[t]`` [N_lig,3], ``type_uniform[t]`` [N_lig]).
"""
import torch
import torch.nn.functional as F

from . import graph_ops as G
from .denoiser import build_edge_type, edge_gate, h2x_attention, unitransformer_forward
from .diffusion import context_embed, compose

ABSORBING_STATE = 0


def num_com_layers(sd, prefix='com_head.'):
    n = 0
    while (prefix + f'h2xattentions.{n}.xk_func.net.0.weight') in sd:
        n += 1
    return n


def com_head(sd, x_lig_pred, bl, x, h, gen, lig, batch_idx, k=32, prefix='com_head.'):
    """CoMPredictor.forward (diffbp.py:80-101) on composed tensors."""
    ptr = G.graph_ptr_from_batch(batch_idx)
    nbr = G.neighbor_table(x, ptr, k=k)
    src, dst = G.table_to_edge_index(nbr)
    etype = build_edge_type(src, dst, lig.bool())
    e_w = edge_gate(sd, prefix, x, src, dst)
    x_out = x.clone()
    for l in range(num_com_layers(sd, prefix)):
        dx = h2x_attention(sd, prefix + f'h2xattentions.{l}.', x_out, h, src, dst, etype, e_w)
        x_out = x_out + dx * gen.unsqueeze(-1).to(x.dtype)
    return com_eps(x_lig_pred, x[lig], x_out[lig], bl)


def com_eps(x_pred, x_t, x_com, bl, num_graphs=None):
    """The two outputs of CoMPredictor.forward (diffbp.py:80-101) on the ligand rows, in the dtype of the inputs:
    the zero-mean noise prediction (x_pred - x_t) - mean_g(x_pred - x_t) and the per-graph shift mean_g(x_com - x_t),
    where x_com are the CoM head's output coordinates.  ``num_graphs`` sizes the per-graph tables."""
    noise = x_pred - x_t
    noise = noise - G.scatter_mean(noise, bl, dim=0, dim_size=num_graphs)[bl]
    delta = x_com - x_t
    return noise, G.scatter_mean(delta, bl, dim=0, dim_size=num_graphs)[bl]


def pos_score_update(eps, x_t, abar, beta, nonzero, gen_flag, noise):
    """The position update of CTNVPScheduler.backward_remove_noise(type='score') for the step's scalars
    (alphas_cumprod[t], betas[t], 0 at t == 0 else 1), in the dtype of ``x_t``."""
    dt = x_t.dtype
    a, b, nonzero = (torch.as_tensor(v, dtype=dt) for v in (abar, beta, nonzero))
    eps, noise = eps.to(dt), noise.to(dt)
    sigma = (1 - a).sqrt()
    score = -eps / sigma
    xs = (x_t + b * score) / (1 - b).sqrt()
    xs = xs + nonzero * b.sqrt() * noise
    return torch.where(gen_flag.unsqueeze(-1), xs, x_t)


def pos_reverse_step_score(sd, eps, x_t, t_idx, gen_flag, noise, prefix='pos_scheduler.'):
    """CTNVPScheduler.backward_remove_noise(type='score'), all graphs at the same t."""
    return pos_score_update(eps, x_t, sd[prefix + 'alphas_cumprod'][t_idx], sd[prefix + 'betas'][t_idx],
                            0.0 if t_idx == 0 else 1.0, gen_flag, noise)


def mask_type_update(logits, c_t, prob, gen_flag, uniform, num_classes):
    """MaskTypeSchedule.backward_remove_noise(pred_logit=True, fix_pred=True) for the change probability ``prob`` of
    the step, in the dtype of ``logits``.  -> (one-hot c_next, v_next, softmax(logits))."""
    dt = logits.dtype
    c_pred = F.softmax(logits, dim=-1)
    vt = c_t.argmax(-1)
    change = (uniform.to(dt) < torch.as_tensor(prob, dtype=dt)) & gen_flag & (vt == ABSORBING_STATE)
    v_next = torch.where(change, c_pred.argmax(-1), vt)
    return F.one_hot(v_next, num_classes=num_classes).float(), v_next, c_pred


def mask_type_reverse_step(logits, c_t, t_idx, num_steps, gen_flag, uniform, num_classes):
    """MaskTypeSchedule.backward_remove_noise(pred_logit=True, fix_pred=True)."""
    t = torch.full((c_t.shape[0],), t_idx, dtype=torch.long)
    prob = ((num_steps - t) / num_steps).clamp(max=1., min=0.)
    c_next, v_next, _ = mask_type_update(logits, c_t, prob, gen_flag, uniform, num_classes)
    return c_next, v_next


def denoise(sd, batch, x_lig, c_lig, k=32):
    """embed -> compose -> denoiser -> com head (diffbp.py:268-283).  Returns (eps, eps_com, logits) on ligand rows."""
    lig_flag, rec_flag = batch['ligand_lig_flag'], batch['protein_lig_flag']
    gen_lig = batch.get('ligand_gen_flag', lig_flag)
    gen_rec = batch.get('protein_gen_flag', torch.zeros_like(rec_flag))
    bl, br = batch['ligand_element_batch'], batch['protein_element_batch']
    h_lig, h_rec = context_embed(sd, c_lig, batch['protein_atom_feature'], batch['protein_aa_type'], lig_flag, rec_flag)
    sort_idx, batch_idx, _ = compose(bl, br)
    x = torch.cat([batch['protein_pos'], x_lig], 0)[sort_idx]
    h = torch.cat([h_rec, h_lig], 0)[sort_idx]
    gen = torch.cat([gen_rec, gen_lig], 0)[sort_idx]
    lig = torch.cat([rec_flag, lig_flag], 0)[sort_idx]
    x_o, h_o, c_o = unitransformer_forward(sd, x, h, batch_idx, lig, gen, k=k)
    eps, eps_com = com_head(sd, x_o[lig], bl, x, h_o, gen, lig, batch_idx, k=k)
    return eps, eps_com, c_o[lig]


def sample(sd, batch, num_steps, pos_noise, type_uniform, num_classes=13, k=32, stop_after=None):
    """DiffBP.sample with injected noise.  Returns traj t -> (x_lig, c_lig) with keys T-1 ... -1."""
    x = batch['ligand_pos'].float()
    c = F.one_hot(batch['ligand_atom_type'], num_classes=num_classes).float()
    gen_lig = batch.get('ligand_gen_flag', batch['ligand_lig_flag'])
    traj = {num_steps - 1: (x, c)}
    done = 0
    for t_idx in reversed(range(num_steps)):
        x, c = traj[t_idx]
        eps, eps_com, logits = denoise(sd, batch, x, c, k=k)
        x_next = pos_reverse_step_score(sd, eps + eps_com, x, t_idx, gen_lig, pos_noise[t_idx])
        c_next, _ = mask_type_reverse_step(logits, c, t_idx, num_steps, gen_lig, type_uniform[t_idx], num_classes)
        traj[t_idx - 1] = (x_next, c_next)
        done += 1
        if stop_after is not None and done >= stop_after:
            break
    return traj
