"""Operand magnitudes outside the synthetic weights' comfortable range.

The f16 tensor-core kernels get fp32 accuracy by splitting every operand into (hi, lo) f16 halves after multiplying it by
a power of two.  That split only works inside a window: above it hi overflows to inf (NaN results), below it lo goes
subnormal (the error grows far past fp32's).  Weights and LayerNorm activations are bounded when the blob is packed;
h is data, so the f16 node GEMM scales every row of its A tile by its own power of two.  These tests push h and the
weights across many decades and compare every kernel family with a float64 reference: per row for the node
projections, so one badly rounded small row cannot hide under a large one.
Run on an H100:  python -m pytest tests/test_operand_range.py -m gpu
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cbgbench_b200 import _lib, synthetic
from cbgbench_b200.diffbp import DiffBPB200
from cbgbench_b200.modules import pack_denoiser_blob
from helpers import FORWARD_CASES, assert_close, composed_inputs, make_model, rel_err

torch.set_grad_enabled(False)
gpu = pytest.mark.gpu
NODE_IMPLS = {0: 'simt', 1: 'wgmma-tf32', 2: 'wgmma-f16'}
ROW_TOL = 2e-6          # per-row bar of the node projections: max |got - want| <= ROW_TOL * max |want| of that row
LAYER = 3


def dev():
    return torch.device('cuda:0')


@pytest.fixture
def edge_impl_reset():
    yield
    _lib.check(_lib.lib().cbg_set_edge_impl(0, 12))
    _lib.check(_lib.lib().cbg_set_edge_impl(_lib.DEFAULT_EDGE_IMPL, 0))     # library default


# ---------------------------------------------------------------------------------------------
# node projections, row by row, against float64
ROW_EXPONENTS = [-40, -24, -16, -12, -10, -8, -4, 0, 4, 8, 10, 11, 12, 14, 20, 40]
# positions in the row list (= rows of the 128-row tiles) of the special rows; zero rows at a warpgroup / CTA edge
SPECIAL_ROWS = {5: 'zero', 127: 'zero', 128: 'zero', 130: 'constant', 200: 'spike', 260: 'subnormal'}
N_LISTED, N_NODES = 333, 400


def _sub_names(sublayer):
    return ('x2h_layers.0.', 'hk_func', 'hv_func', 'hq_func') if sublayer == 0 else \
           ('h2x_layers.0.', 'xk_func', 'xv_func', 'xq_func')


def _rows(exponents, seed):
    """h [N_NODES, 128] fp32, the unsorted list of N_LISTED rows, and a label per listed row.  Listed row i is N(0, 1)
    scaled by 2^exponents[i % len], except the special rows (zero, constant, one spike of 2^12 among 2^-12, fp32
    subnormals mixed into O(1) values).  Neighbouring rows of a tile differ by many decades."""
    rs = np.random.RandomState(seed)
    row_idx = rs.permutation(N_NODES)[:N_LISTED].astype(np.int32)
    assert not bool((row_idx[1:] > row_idx[:-1]).all())
    h = rs.normal(size=(N_NODES, 128))
    labels = []
    for i, node in enumerate(row_idx):
        kind = SPECIAL_ROWS.get(i) if len(exponents) > 1 else None
        if kind == 'zero':
            h[node] = 0.0
        elif kind == 'constant':
            h[node] = 3.0
        elif kind == 'spike':
            h[node] = 2.0 ** -12
            h[node, 37] = 2.0 ** 12
        elif kind == 'subnormal':
            sub = rs.rand(128) < 0.5
            h[node, sub] = rs.choice([-1.0, 1.0], size=int(sub.sum())) * rs.uniform(1e-45, 1e-38, size=int(sub.sum()))
        else:
            e = exponents[i % len(exponents)]
            h[node] *= 2.0 ** e
            kind = f's={e}'
        labels.append(kind)
    h32 = torch.from_numpy(h.astype(np.float32))
    if len(exponents) > 1:
        assert bool((h32[row_idx[260]].abs() < 1.2e-38).any() & (h32[row_idx[260]] != 0).any())   # subnormals survive
    return h32, torch.from_numpy(row_idx), labels


def _node_proj_want(sd, layer, sublayer, h64):
    """float64 planes (Pj_k, Pj_v, Pi_k, Pi_v, q) and the bias part of each (the packer centres the first Linear of the
    edge MLPs over the output features, so every plane is minus its row mean)."""
    pre, kn, vn, qn = _sub_names(sublayer)
    pre = f'denoiser.blocks.{layer}.' + pre
    d = lambda k: sd[pre + k].double()
    w0k, w0v = d(kn + '.net.0.weight'), d(vn + '.net.0.weight')
    w0k, w0v = w0k - w0k.mean(0, keepdim=True), w0v - w0v.mean(0, keepdim=True)
    bk, bv = d(kn + '.net.0.bias'), d(vn + '.net.0.bias')
    bk, bv = bk - bk.mean(), bv - bv.mean()
    zero = torch.zeros(128, dtype=torch.float64)
    terms = [h64 @ w0k[:, 212:340].T, h64 @ w0v[:, 212:340].T, h64 @ w0k[:, 84:212].T, h64 @ w0v[:, 84:212].T]
    bias = [zero, zero, bk, bv]
    qh = F.layer_norm(h64 @ d(qn + '.net.0.weight').T + d(qn + '.net.0.bias'), (128,), d(qn + '.net.1.weight'),
                      d(qn + '.net.1.bias'), 1e-5).relu()
    terms.append((qh @ d(qn + '.net.3.weight').T + d(qn + '.net.3.bias')) / math.sqrt(8.0))
    bias.append(zero)
    return terms, bias


def _run_node_proj(blob, layer, sublayer, impl, h, row_idx):
    L = _lib.lib()
    lay = _lib.blob_layout()
    base_ptr = blob.data_ptr() + 4 * (lay['global_floats'] + layer * lay['layer_floats'])
    planes = torch.full((5, h.shape[0], 128), float('nan'), device=dev())
    ridx = row_idx.to(dev())
    hd = h.to(dev())
    assert L.cbg_node_proj_f32(base_ptr, sublayer, impl, hd.data_ptr(), ridx.data_ptr(), int(row_idx.numel()),
                               h.shape[0], planes.data_ptr(), None) == 0, L.cbg_last_error()
    torch.cuda.synchronize()
    return planes.cpu().double()


def _row_failures(got, terms, bias, row_idx, labels):
    """Rows of the list that miss the bar, summarised per row label.  The bar of every row is ROW_TOL times the
    row's largest h term (the plane without its bias), so a bias-dominated row cannot hide its h term, plus one fp32
    ulp of each output (the rounding of the stored result, which no kernel can avoid).  NaN fails."""
    sel = row_idx.long()
    bad = []
    for p in range(5):
        g, t, b = got[p][sel], terms[p][sel], bias[p]
        want = t + b
        scale = t.abs().amax(1, keepdim=True)
        err = (g - want).abs()
        ok = err <= ROW_TOL * scale + 2.0 ** -23 * want.abs()
        for i in torch.nonzero(~ok.all(1)).flatten().tolist():
            ratio = float(((err[i] - 2.0 ** -23 * want[i].abs()) / scale[i].clamp(min=1e-300)).max())
            bad.append((labels[i], p, ratio))
    summary = {}
    for label, p, ratio in bad:       # label: (row planes, planes, worst err / row scale; NaN counts as worst)
        n, planes, worst = summary.get(label, (0, set(), 0.0))
        summary[label] = (n + 1, planes | {p}, ratio if math.isnan(ratio) or math.isnan(worst) else max(worst, ratio))
    return [f'{label}: {n} row planes (planes {sorted(planes)}), worst {worst:.1e}'
            for label, (n, planes, worst) in summary.items()]


@gpu
@pytest.mark.parametrize('impl', list(NODE_IMPLS), ids=list(NODE_IMPLS.values()))
@pytest.mark.parametrize('sublayer', [0, 1], ids=['x2h', 'h2x'])
def test_node_projections_per_row_across_magnitudes(impl, sublayer):
    model, sd = make_model(10, device=dev())
    h, row_idx, labels = _rows(ROW_EXPONENTS, seed=23 + sublayer)
    got = _run_node_proj(model.denoiser.packed_blob(dev()), LAYER, sublayer, impl, h, row_idx)
    terms, bias = _node_proj_want(sd, LAYER, sublayer, h.double())
    bad = _row_failures(got, terms, bias, row_idx, labels)
    assert not bad, f'{NODE_IMPLS[impl]} sublayer {sublayer}, rows that miss the bar: ' + '; '.join(bad)
    # zero rows give exactly the stored (fp32) bias; rows not listed stay untouched
    zero = [int(row_idx[i]) for i, k in SPECIAL_ROWS.items() if k == 'zero']
    for p in range(4):
        assert torch.equal(got[p][zero], bias[p].float().double().expand(len(zero), 128)), p
    mask = torch.ones(h.shape[0], dtype=torch.bool)
    mask[row_idx.long()] = False
    assert torch.isnan(got[:, mask]).all()


def _scaled_layer_weights(sd, layer, k):
    """Copy of ``sd`` with the weight matrices of layer ``layer``'s X2H and H2X MLPs scaled by 2^k (LayerNorm gains and
    shifts and the biases unchanged)."""
    sd = dict(sd)
    for sublayer in (0, 1):
        pre, *mlps = _sub_names(sublayer)
        for m in mlps:
            for lin in ('0', '3'):
                key = f'denoiser.blocks.{layer}.{pre}{m}.net.{lin}.weight'
                sd[key] = sd[key] * 2.0 ** k
    return sd


@gpu
@pytest.mark.parametrize('k', [-8, -4, 4, 6])
@pytest.mark.parametrize('impl', list(NODE_IMPLS), ids=list(NODE_IMPLS.values()))
def test_node_projections_per_row_across_weight_magnitudes(impl, k):
    """Weights packed through the normal path (the model's blob cache) at 2^k times their seeded scale."""
    model, sd = make_model(10)
    sd = _scaled_layer_weights(sd, LAYER, k)
    model.load_state_dict(sd, strict=True)
    model = model.to(dev())
    blob = model.denoiser.packed_blob(dev())
    for sublayer in (0, 1):
        h, row_idx, labels = _rows([0], seed=41 + sublayer)
        got = _run_node_proj(blob, LAYER, sublayer, impl, h, row_idx)
        terms, bias = _node_proj_want(sd, LAYER, sublayer, h.double())
        bad = _row_failures(got, terms, bias, row_idx, labels)
        assert not bad, f'{NODE_IMPLS[impl]} sublayer {sublayer} weights x 2^{k}, rows that miss the bar: ' + '; '.join(bad)


# ---------------------------------------------------------------------------------------------
# the denoiser against float64
EDGE_IMPLS = {6: 'wgmma', 0: 'simt'}
RAGGED = next(c for c in FORWARD_CASES if c[0] == 'ragged_small')
_ORACLE64 = {}


def _oracle64(sd, key, x, h, bidx, lig, gen):
    """float64 reference (one layer and the full forward), memoised per input: the CPU forward dominates the run time."""
    from oracle import denoiser as ODn
    if key not in _ORACLE64:
        sd64 = {k: v.double() for k, v in sd.items()}
        xo, ho, co, tr = ODn.unitransformer_forward(sd64, x, h, bidx, lig, gen, return_trace=True, dtype=torch.float64)
        _ORACLE64[key] = (tr['h'][0], xo, ho, co)
    return _ORACLE64[key]


def _check_denoiser(model, sd, key, h_scale, impl):
    _, n_prot, n_lig, seed, gen_mode, enc = RAGGED
    batch = synthetic.make_batch(n_prot, n_lig, seed=seed, gen_mode=gen_mode)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    h = h * h_scale                                           # a power of two: exact
    h1_want, x_want, h_want, c_want = _oracle64(sd, key, x, h, bidx, lig, gen)
    args = [t.to(dev()) for t in (x, h, bidx, lig, gen)]
    _lib.check(_lib.lib().cbg_set_edge_impl(impl, 0))
    h1 = model.denoiser(*args, stop_after_layers=1)[1].cpu()
    xg, hg, cg = (t.cpu() for t in model.denoiser(*args))
    what = f'{key} edge impl {EDGE_IMPLS[impl]}'
    for name, t in (('h after one layer', h1), ('x', xg), ('h', hg), ('c', cg)):
        assert torch.isfinite(t).all(), f'{what}: {name} not finite'
    e1 = rel_err(h1, h1_want)
    errs = {n: rel_err(a, b) for n, a, b in (('x', xg, x_want), ('h', hg, h_want), ('c', cg, c_want))}
    report = f'{what}: h after one layer {e1:.1e}, ' + ', '.join(f'{n} {e:.1e}' for n, e in errs.items())
    assert e1 < 1e-5, report
    assert all(e < 1e-4 for e in errs.values()), report
    assert_close(xg, x_want, what=f'{what}: x')


@gpu
@pytest.mark.parametrize('c', [-12, -6, 0, 6, 12])
def test_denoiser_matches_float64_across_h_magnitudes(c, edge_impl_reset):
    model, sd = make_model(10, device=dev())
    for impl in EDGE_IMPLS:
        _check_denoiser(model, sd, f'h x 2^{c}', 2.0 ** c, impl)


@gpu
def test_denoiser_matches_float64_with_large_layernorm_gains(edge_impl_reset):
    """X2H / H2X LayerNorm gains x 8 (activation bound ~ 8 x sqrt(127) x max gamma: inside the packer's limit)."""
    model, sd = make_model(10)
    sd = {k: (v * 8.0 if ('x2h_layers' in k or 'h2x_layers' in k) and k.endswith('.net.1.weight') else v)
          for k, v in sd.items()}
    model.load_state_dict(sd, strict=True)
    model = model.to(dev())
    for impl in EDGE_IMPLS:
        _check_denoiser(model, sd, 'LayerNorm gamma x 8', 1.0, impl)


# ---------------------------------------------------------------------------------------------
# sampling path: large context features through the merged source / destination launch, pruned row lists, graph replay
CONTEXT_EMBEDDERS = ('protein_atom_emb', 'ligand_atom_emb', 'residue_emb', 'ligand_indicator')


@gpu
@pytest.mark.parametrize('gen_mode', ['denovo', 'partial'])
def test_sampling_with_large_context_features(gen_mode):
    from oracle import diffusion as OD
    T = 3
    model, sd = make_model(T)
    sd = {k: (v * 2.0 ** 12 if k.startswith(tuple(f'context_embedder.{m}.' for m in CONTEXT_EMBEDDERS)) else v)
          for k, v in sd.items()}
    model.load_state_dict(sd, strict=True)
    model = model.to(dev())
    batch = synthetic.make_batch([150, 60, 20], [20, 12, 5], seed=151, gen_mode=gen_mode)
    h = composed_inputs(sd, batch)[1]
    assert float(h.abs().amax()) >= 4096.0       # past the fixed x16 window of the f16 split (|h| < 4095)
    n_lig = int(batch['ligand_pos'].shape[0])
    pn, tu = synthetic.make_noise(T, n_lig, 13, seed=19)
    traj = model.sample(batch, pos_noise=pn, type_uniform=tu)
    want = OD.sample(sd, batch, T, pn, tu)
    for t in range(-1, T):
        xg, cg = traj[t][0].cpu(), traj[t][1].cpu()
        assert torch.isfinite(xg).all() and torch.isfinite(cg).all(), t
        assert torch.equal(cg.argmax(-1), want[t][1].argmax(-1)), t
        assert rel_err(xg, want[t][0]) < 1e-4, (t, rel_err(xg, want[t][0]))


# ---------------------------------------------------------------------------------------------
# packer bounds (CPU): images that would turn into inf / NaN on the tensor cores are refused
F16_MAX = 65504.0


def _denoiser_sd():
    model, sd = make_model(10)
    return {k[len('denoiser.'):]: v.clone() for k, v in sd.items() if k.startswith('denoiser.')}, model.denoiser


def _pack(sd, den):
    return pack_denoiser_blob(sd, '', den.num_layers, den.out_classes)


def _ln_gamma_for_bound(sd, key, bound):
    """LayerNorm gains whose activation bound sqrt(127) max|gamma| + max|beta| is ``bound`` (one gain set)."""
    g = sd[key + '.weight'].clone()
    g[17] = (bound - float(sd[key + '.bias'].abs().max())) / math.sqrt(127.0)
    assert float(g.abs().max()) == float(g[17].abs())
    return g


CASES = {
    # (key, how to set it just outside the limit, just inside, field named in the message)
    'node_tch': ('blocks.2.x2h_layers.0.hk_func.net.0.weight', lambda sd, k: 300.0, lambda sd, k: 255.0,
                 'layer 2 X2H_NODE_TCH'),
    'tcw1': ('blocks.5.h2x_layers.0.xk_func.net.3.weight', lambda sd, k: 1100.0, lambda sd, k: 1020.0,
             'layer 5 H2X_K_TCW1'),
    'k_ln': ('blocks.1.x2h_layers.0.hk_func.net.1', lambda sd, k: _ln_gamma_for_bound(sd, k, F16_MAX / 64 * 1.0001),
             lambda sd, k: _ln_gamma_for_bound(sd, k, F16_MAX / 64 * 0.999), 'layer 1 X2H_K_LN'),
    'v_ln': ('blocks.4.h2x_layers.0.xv_func.net.1', lambda sd, k: _ln_gamma_for_bound(sd, k, F16_MAX / 64 * 1.0001),
             lambda sd, k: _ln_gamma_for_bound(sd, k, F16_MAX / 64 * 0.999), 'layer 4 H2X_V_LN'),
    'q_ln': ('blocks.7.h2x_layers.0.xq_func.net.1', lambda sd, k: _ln_gamma_for_bound(sd, k, F16_MAX / 16 * 1.0001),
             lambda sd, k: _ln_gamma_for_bound(sd, k, F16_MAX / 16 * 0.999), 'layer 7 H2X_Q_LN'),
}


def _apply(sd, case, which):
    key, outside, inside, _ = CASES[case]
    sd = dict(sd)
    fn = outside if which == 'outside' else inside
    if key.endswith('.weight'):
        w = sd[key].clone()
        w[3, 250 if 'net.0' in key else 40] = fn(sd, key)       # net.0: a Pj column of the first Linear
        sd[key] = w
    else:
        sd[key + '.weight'] = fn(sd, key)
    return sd


@pytest.mark.parametrize('case', list(CASES))
def test_packer_refuses_operands_outside_the_f16_window(case):
    sd, den = _denoiser_sd()
    with pytest.raises(ValueError, match=CASES[case][3]):
        _pack(_apply(sd, case, 'outside'), den)
    blob = _pack(_apply(sd, case, 'inside'), den)
    assert torch.isfinite(blob).all()


def test_packer_bounds_keep_seeded_weights_and_com_head():
    sd, den = _denoiser_sd()
    assert torch.isfinite(_pack(sd, den)).all()
    model = DiffBPB200(synthetic.diffbp_config(num_steps=10))
    model.load_state_dict(synthetic.seeded_state_dict(model, seed=0), strict=True)
    com = model.com_head
    assert torch.isfinite(com.packed_blob(torch.device('cpu'))).all()
    sd = dict(com.state_dict())
    w = sd['h2xattentions.1.xk_func.net.0.weight'].clone()
    w[0, 300] = 300.0
    sd['h2xattentions.1.xk_func.net.0.weight'] = w
    with pytest.raises(ValueError, match='layer 1 H2X_NODE_TCH'):
        pack_denoiser_blob(sd, '', com.num_layers, 1, com_head=True)
