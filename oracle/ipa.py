"""CPU restatement of the D3FG encoder `IPATransformer` (SURVEY.md section 8 row f4) - fp32 torch.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Functional style on the reference's own state-dict keys, as-written
formulation ([E, 2H + 84] edge inputs, per-edge k / v, scatter ops).  Pinned to the live reference by
tests/golden/make_golden_f4.py (which also asserts oracle == reference on every stored case).

Reference code followed (``/root/reference``):
  repo/modules/e3nn/itatransformer.py:88-99    _connect_edge (knn_graph k = 32; the radius branch reads an undefined name)
  repo/modules/e3nn/itatransformer.py:101-112  _build_edge_type
  repo/modules/e3nn/itatransformer.py:115-145  forward: shared blocks, edge gate, heads, SO(3) update
  repo/modules/e3nn/itatransformer.py:147-188  InvAttentionLayer (num_x2h x X2HAttention, x fixed)
  repo/modules/attention/x2h_attention.py:43-97
  repo/models/utils/geometry.py:232-250        quaternion_1ijk_to_rotation_matrix
  repo/models/utils/geometry.py:82-99,133-134  apply_rotation_to_vector = R p
  repo/models/utils/so3.py:10-63               log_rotation (no-grad branch: min_cos = -1), exp_skewsym, so3vec maps
"""
import math

import torch
import torch.nn.functional as F

from . import graph_ops as G
from .denoiser import build_edge_type, edge_gate, gaussian_smearing, mlp

N_HEADS = 16


def x2h_attention(sd, lp, x, h, src, dst, etype, e_w):
    """x2h_attention.py:43-97 at the width of ``h`` (ew_net_type='global', out_fc=False)."""
    N, H = h.shape
    rel = x[dst] - x[src]
    dist = torch.norm(rel, p=2, dim=-1, keepdim=True)
    g = gaussian_smearing(dist, sd[lp + 'distance_expansion.offset'])
    onehot = F.one_hot(etype, 4).to(x.dtype)
    r_feat = (onehot[:, :, None] * g[:, None, :]).reshape(len(src), 4 * g.shape[-1])   # explicit width: E may be 0
    kv = torch.cat([onehot, r_feat, h[dst], h[src]], dim=-1)
    k = mlp(sd, lp + 'hk_func.', kv).view(-1, N_HEADS, H // N_HEADS)
    v = (mlp(sd, lp + 'hv_func.', kv) * e_w).view(-1, N_HEADS, H // N_HEADS)
    q = mlp(sd, lp + 'hq_func.', h).view(-1, N_HEADS, H // N_HEADS)
    logits = (q[dst] * k / math.sqrt(k.shape[-1])).sum(-1)
    alpha = G.scatter_softmax(logits, dst, dim=0, dim_size=N)
    out = G.scatter_sum(alpha.unsqueeze(-1) * v, dst, dim=0, dim_size=N).view(N, H)
    return out + h


def quaternion_1ijk_to_rotation_matrix(q):
    b, c, d = torch.unbind(q, dim=-1)
    s = torch.sqrt(1 + b ** 2 + c ** 2 + d ** 2)
    a, b, c, d = 1 / s, b / s, c / s, d / s
    o = torch.stack((a ** 2 + b ** 2 - c ** 2 - d ** 2, 2 * b * c - 2 * a * d, 2 * b * d + 2 * a * c,
                     2 * b * c + 2 * a * d, a ** 2 - b ** 2 + c ** 2 - d ** 2, 2 * c * d - 2 * a * b,
                     2 * b * d - 2 * a * c, 2 * c * d + 2 * a * b, a ** 2 - b ** 2 - c ** 2 + d ** 2), -1)
    return o.reshape(q.shape[:-1] + (3, 3))


def so3vec_to_rotation(w):
    x, y, z = torch.unbind(w, dim=-1)
    o = torch.zeros_like(x)
    S = torch.stack([o, z, -y, -z, o, x, y, -x, o], dim=-1).reshape(w.shape[:-1] + (3, 3))
    n = torch.linalg.norm(w, dim=-1)
    b = (torch.sin(n) + 1e-8) / (n + 1e-8)
    c = (1 - torch.cos(n) + 1e-8) / (n ** 2 + 2e-8)
    return torch.eye(3).to(S) + b[..., None, None] * S + c[..., None, None] * (S @ S)


def rotation_to_so3vec(R):
    trace = R[..., range(3), range(3)].sum(-1)
    cos_theta = ((trace - 1) / 2).clamp_min(min=-1.0)            # sampling runs under no_grad
    sin_theta = torch.sqrt(1 - cos_theta ** 2)
    theta = torch.acos(cos_theta)
    coef = ((theta + 1e-8) / (2 * sin_theta + 2e-8))[..., None, None]
    logR = coef * (R - R.transpose(-1, -2))
    return torch.stack([logR[..., 1, 2], logR[..., 2, 0], logR[..., 0, 1]], dim=-1)


def seq3(sd, p, x):
    """Linear ReLU Linear ReLU Linear (itatransformer.py:54-66)."""
    y = F.relu(F.linear(x, sd[p + '0.weight'], sd[p + '0.bias']))
    y = F.relu(F.linear(y, sd[p + '2.weight'], sd[p + '2.bias']))
    return F.linear(y, sd[p + '4.weight'], sd[p + '4.bias'])


def ipatransformer_forward(sd, x, o, h, batch_idx, lig_flag, gen_flag, prefix='', k=32, num_blocks=1, nbr=None):
    """itatransformer.py:115-145 -> (eps_pos, h, o_next, R_next, c).

    Runs in the dtype of ``x`` / ``h`` / ``sd``.  ``nbr``: a precomputed neighbour table (G.neighbor_table) instead of the
    kNN of ``x``, so that a float64 pass sees exactly the graph of an fp32 one (no tie flips)."""
    ptr = G.graph_ptr_from_batch(batch_idx)
    n_layers = 0
    while (prefix + f'blocks.{n_layers}.x2h_layers.0.hk_func.net.0.weight') in sd:
        n_layers += 1
    table = nbr
    for _ in range(num_blocks):
        nbr = G.neighbor_table(x, ptr, k=k, r_max=None) if table is None else table
        src, dst = G.table_to_edge_index(nbr)
        etype = build_edge_type(src, dst, lig_flag.bool())
        e_w = edge_gate(sd, prefix, x, src, dst)
        for l in range(n_layers):
            s = 0
            while (prefix + f'blocks.{l}.x2h_layers.{s}.hk_func.net.0.weight') in sd:
                h = x2h_attention(sd, prefix + f'blocks.{l}.x2h_layers.{s}.', x, h, src, dst, etype, e_w)
                s += 1
    eps_rot = seq3(sd, prefix + 'eps_rot_net.', h)
    U = quaternion_1ijk_to_rotation_matrix(eps_rot)
    R_o = so3vec_to_rotation(o)
    R_next = R_o @ U
    g = gen_flag.bool()[:, None]
    o_next = torch.where(g.expand(-1, 3), rotation_to_so3vec(R_next), o)
    eps_crd = seq3(sd, prefix + 'eps_crd_net.', h)
    eps_pos = torch.matmul(R_o, eps_crd.unsqueeze(-1)).squeeze(-1)
    eps_pos = torch.where(g.expand(-1, 3), eps_pos, torch.zeros_like(eps_pos))
    c = F.linear(h, sd[prefix + 'classifier.0.weight'], sd[prefix + 'classifier.0.bias'])
    c = F.softplus(c) - math.log(2.0)
    c = F.linear(c, sd[prefix + 'classifier.2.weight'], sd[prefix + 'classifier.2.bias'])
    return eps_pos, h, o_next, R_next, c
