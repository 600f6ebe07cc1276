"""The TargetDiff, DiffSBDD and DiffBP reverse steps against float64 at their per-graph edges (DESIGN.md section 10,
"Checks").

- sbdd_reverse_kernel through the cbg_sbdd_reverse_f32 hook and bp_reverse_kernel through cbg_bp_reverse_f32, one CTA
  of 128 threads per graph: graphs of 1, 127, 128, 129, 256, 257 and 1500 ligand atoms, graphs without ligand atoms
  between and after others, zero-node graphs, a ligand-only graph, 3000 graphs of 1 to 3 atoms and n_lig = 0; every
  case at K in {1, 13, 16} and at the scalars of t in {0, 1, T/2, T - 1} of a T = 1000 schedule (plus the DiffSBDD final
  stage).  The float64 references are the dtype-generic step functions of oracle/diffusion_sbdd.py and
  oracle/diffusion_bp.py, which the fp32 sample loops use too.
- reverse_kernel (TargetDiff) through cbg_reverse_step_f32: positions against float64, the type against the float64
  Gumbel-max class on crafted rows (u at 0 and 1 - 2^-24, equal logits, logits over +-80, all-zero and soft c_t, rows
  where the 1e-8 of log(c_t + 1e-8) decides the class).
- each production step (cbg_sbdd_step_f32, cbg_bp_step_f32, cbg_sample_step_f32) on a batch whose first graph has more
  than 128 ligand atoms, against float64 from the call's own denoiser outputs.
CPU: the argument refusals of the three hooks.

Bars (per element, float64): ULPS fp32 ulps of the element's largest term, plus for a per-graph mean
(ceil(n_g / 128) + 8) * 2^-24 * mean_g |z| (the depth of the kernel's fixed-order sum: a strided loop of
ceil(n_g / 128) terms per thread, five warp levels, two block levels and the division) plus the largest
per-element bar of the graph."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cbgbench_b200 import _lib, synthetic
from cbgbench_b200.diffbp import DiffBPB200
from cbgbench_b200.diffsbdd import DiffSBDDB200
from cbgbench_b200.schedulers import DiffsbddVariationalTables
from oracle import diffusion as OD, diffusion_bp as OB, diffusion_sbdd as OS
from helpers import WEIGHT_SEED, make_model

torch.set_grad_enabled(False)
DEV = 'cuda:0'
T_SCHED = 1000
T_STEPS = (0, 1, T_SCHED // 2, T_SCHED - 1)
KS = (1, 13, 16)
ULPS = 6                       # fp32 ulps of the largest term of an element: the few roundings of the step's formula
U32 = 2.0 ** -24
OFFSET = np.array([812.0, -655.0, 431.0])     # common coordinate offset: |x| up to about 1e3
F64 = torch.float64
PAD = 3                        # sentinel rows after every output (and one after every input)

# (pocket atoms, ligand atoms) per graph
LAYOUTS = {
    'lig1': [(6, 1)],
    'lig127': [(40, 127)],
    'lig128': [(33, 128)],
    'lig129': [(20, 129)],
    'lig256': [(17, 256)],
    'lig257': [(64, 257)],
    'lig1500': [(300, 1500)],
    'ligandless_between_and_after': [(30, 20), (25, 0), (10, 140), (12, 0)],
    'zero_node': [(10, 5), (0, 0), (7, 130), (0, 0)],
    'ligand_only': [(0, 200), (3, 4), (0, 1)],
    'n_lig_0': [(10, 0), (5, 0), (0, 0)],
}


def _many_graphs(rs, n=3000):
    out = []
    for _ in range(n):
        size = rs.randint(1, 4)
        nl = rs.randint(0, size + 1)
        out.append((size - nl, nl))
    return out


def _layout(graphs, salt):
    """Node layout of ``graphs``: per graph pocket first, ligand first or interleaved (rotating with ``salt``), so that
    a graph's last node is sometimes a ligand atom and sometimes a pocket atom.
    -> (graph_ptr int32 [B+1], lig_node int32 [n_lig] ascending, is_lig bool [N], bl [n_lig], bn [N])."""
    rs = np.random.RandomState(salt)
    kinds, ptr = [], [0]
    for g, (npk, nl) in enumerate(graphs):
        k = [0] * npk + [1] * nl
        m = (g + salt) % 3
        if m == 1:
            k = [1] * nl + [0] * npk
        elif m == 2:
            k = list(rs.permutation(k))
        kinds += k
        ptr.append(len(kinds))
    is_lig = np.array(kinds, dtype=bool)
    bn = np.repeat(np.arange(len(graphs)), np.diff(ptr))
    lig_node = np.nonzero(is_lig)[0]
    return (np.array(ptr, np.int32), lig_node.astype(np.int32), is_lig, bn[lig_node].astype(np.int64),
            bn.astype(np.int64))


def _sp(v):
    """fp32 ulp of |v| (float64 tensor in, float64 tensor out)."""
    a = np.abs(v.double().numpy()).astype(np.float32)
    return torch.from_numpy(np.spacing(a).astype(np.float64))


def _seg(vals, idx, B, how='mean'):
    """Per-graph mean / amax of the rows of ``vals`` (float64 [n, w]) over the ids ``idx`` (B graphs, 0 if empty)."""
    out = torch.zeros((B, vals.shape[1]), dtype=F64)
    if how == 'amax':
        return out.scatter_reduce_(0, idx[:, None].expand_as(vals), vals, 'amax', include_self=True)
    out.index_add_(0, idx, vals)
    cnt = torch.bincount(idx, minlength=B).clamp(min=1).to(F64)
    return out / cnt[:, None]


def _depth(bl, B):
    n = torch.bincount(bl, minlength=B).to(F64)
    return torch.ceil(n / 128) + 8


def _d(a, dt=torch.float32, pad=1, fill=float('nan')):
    """Device copy of ``a`` with ``pad`` sentinel rows: a NULL-free pointer even for zero rows."""
    a = torch.as_tensor(a)
    shape = (a.shape[0] + pad,) + tuple(a.shape[1:])
    out = torch.full(shape, fill, dtype=dt) if dt.is_floating_point else torch.full(shape, int(fill), dtype=dt)
    out[: a.shape[0]] = a.to(dt)
    return out.to(DEV).contiguous()


def _out(n, w, dt=torch.float32):
    if dt.is_floating_point:
        return torch.full((n + PAD, w), float('nan'), dtype=dt, device=DEV)
    return torch.full((n + PAD,), -7, dtype=dt, device=DEV)


def _check_pad(t, n, what):
    tail = t[n:].cpu()
    ok = bool(torch.isnan(tail).all()) if tail.is_floating_point() else bool((tail == -7).all())
    assert ok, f'{what}: rows past n_lig were written'


_CACHE = {}


def _sbdd_coefs():
    if 'sbdd' not in _CACHE:
        tab = DiffsbddVariationalTables(T_SCHED, 'polynomial_2')
        cs = [(f't{t}', _lib.SbddCoef(*tab.step_scalars(t), mode=0)) for t in T_STEPS]
        _CACHE['sbdd'] = cs + [('final', _lib.SbddCoef(*tab.final_scalars(), mode=1))]
    return _CACHE['sbdd']


def _bp_model():
    if 'bp' not in _CACHE:
        _CACHE['bp'] = DiffBPB200(synthetic.diffbp_config(num_steps=T_SCHED))
    return _CACHE['bp']


def _td_model():
    if 'td' not in _CACHE:
        _CACHE['td'] = make_model(T_SCHED)[0]
    return _CACHE['td']


# ---- inputs ---------------------------------------------------------------------------------------------------------

def _inputs(graphs, K, seed):
    """Random per-graph inputs (CPU fp32): x4 [N,4] (ligand rows: eps_pred / x_com near the ligand, flag float 1 or 3;
    pocket rows at the offset, flag 0), x_t at the offset, types, noise, generation flags."""
    ptr, lig_node, is_lig, bl, bn = _layout(graphs, seed)
    rs = np.random.RandomState(seed)
    N, n = int(ptr[-1]), int(lig_node.shape[0])
    f = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))
    x_t = OFFSET + rs.normal(0, 40, size=(n, 3))
    x4 = np.zeros((N, 4))
    x4[:, :3] = OFFSET + rs.normal(0, 40, size=(N, 3))
    x4[lig_node, :3] = rs.normal(0, 3, size=(n, 3))
    x4[is_lig, 3] = np.where(rs.random_sample(n) < 0.5, 1.0, 3.0)
    ct_onehot = np.eye(K)[np.where(rs.random_sample(n) < 0.6, 0, rs.randint(0, K, size=n))]
    return dict(ptr=ptr, lig_node=lig_node, is_lig=torch.from_numpy(is_lig), bl=torch.from_numpy(bl),
                bn=torch.from_numpy(bn), B=len(graphs), N=N, n=n, K=K, x4=f(x4), x_t=f(x_t),
                x_com=f(x_t + rs.normal(0, 2, size=(n, 3))), x_pred=f(x_t + rs.normal(0, 3, size=(n, 3))),
                c_t=f(rs.normal(0, 1, size=(n, K))), c_onehot=f(ct_onehot), logits=f(rs.normal(0, 3, size=(n, K))),
                xn=f(rs.normal(size=(n, 3))), cn=f(rs.normal(size=(n, K))), gen=torch.from_numpy(rs.random_sample(n) < 0.8),
                u=f(rs.random_sample(n)))


def _graph_args(st):
    x4 = torch.full((st['N'] + 5, 4), float('nan'))          # five rows past the last graph: never touched
    x4[: st['N']] = st['x4']
    lig = np.concatenate([st['lig_node'], [1 << 30]])
    return x4.to(DEV).contiguous(), torch.from_numpy(st['ptr']).to(DEV), torch.from_numpy(lig.astype(np.int32)).to(DEV)


# ---- DiffSBDD -------------------------------------------------------------------------------------------------------

def _run_sbdd(st, coef):
    x4, ptr, lig = _graph_args(st)
    n, K = st['n'], st['K']
    keep = [_d(st[k]) for k in ('logits', 'x_t', 'c_t', 'xn', 'cn')]
    xo, co = _out(n, 3), _out(n, K)
    with torch.cuda.device(DEV):
        _lib.check(_lib.lib().cbg_sbdd_reverse_f32(x4.data_ptr(), ptr.data_ptr(), st['B'], lig.data_ptr(), n, K,
                                                   C.byref(coef), *[t.data_ptr() for t in keep], xo.data_ptr(),
                                                   co.data_ptr(), _lib.stream_ptr(torch.device(DEV))))
    torch.cuda.synchronize()
    _check_pad(xo, n, 'x_next')
    _check_pad(co, n, 'c_next')
    return xo[:n].cpu(), co[:n].cpu(), x4.cpu()


def _sbdd_check(st, coef, got):
    """All SBDD assertions for one call; -> {output: largest |error| / bar, ...} and the largest absolute errors."""
    x_next, c_next, x4o = got
    n, B, bl = st['n'], st['B'], st['bl']
    a, b, s, mode = coef.a, coef.b, coef.s, coef.mode
    x_t, eps, xn = st['x_t'].double(), st['x4'][torch.from_numpy(st['lig_node']).long(), :3].double(), st['xn'].double()
    pocket = ~st['is_lig']
    bp = st['bn'][pocket]
    rec = st['x4'][pocket][:, :3].double()
    zs = OS.reverse_update(x_t, eps, a, b, s, xn, mode)
    want, rec_want = OS.remove_mean_batch(zs, rec, bl, bp, num_graphs=B)
    a64, b64, s64 = (torch.tensor(v, dtype=F64) for v in (a, b, s))
    term = torch.maximum(torch.maximum((x_t / a64 if mode == 0 else a64 * x_t).abs(), (b64 * eps).abs()
                                       * (1 if mode == 0 else a64.abs())), (s64 * xn).abs())
    e_zs = ULPS * _sp(term)
    e_mean = _depth(bl, B)[:, None] * U32 * _seg(zs.abs(), bl, B) + _seg(e_zs, bl, B, 'amax')
    bar = e_zs + e_mean[bl] + _sp(want)
    err = (x_next.double() - want).abs()
    assert bool((err <= bar).all()), ('x_next', int((err > bar).sum()), float((err / bar).max()))
    rep = {'x_next': float((err / bar).max()) if n else 0.0}
    absmax = {'x_next': float(err.max()) if n else 0.0}
    # the ligand mean of x_next per graph is 0 within the summation bar
    mean_next = _seg(x_next.double(), bl, B)
    mbar = _depth(bl, B)[:, None] * U32 * _seg(zs.abs(), bl, B) + _seg(_sp(x_next.double()), bl, B, 'amax')
    assert bool((mean_next.abs() <= mbar).all()), ('ligand mean', float((mean_next.abs() / mbar).max()))
    # pocket rows: shifted by their graph's float64 mean; graphs without ligand atoms do not move
    has_lig = torch.bincount(bl, minlength=B) > 0
    moved = has_lig[bp]
    got_rec = x4o[: st['N']][pocket][:, :3].double()
    perr = (got_rec - rec_want).abs()
    pbar = e_mean[bp] + _sp(rec_want)
    assert bool((perr[moved] <= pbar[moved]).all()), ('pocket', float((perr / pbar)[moved].max()))
    rep['pocket'] = float((perr / pbar)[moved].max()) if bool(moved.any()) else 0.0
    absmax['pocket'] = float(perr[moved].max()) if bool(moved.any()) else 0.0
    assert torch.equal(x4o[: st['N']][pocket][~moved], st['x4'][pocket][~moved])
    # ligand rows (eps_pred) and every flag float bit for bit; the rows past the last graph untouched
    assert torch.equal(x4o[: st['N']][st['is_lig']], st['x4'][st['is_lig']])
    assert torch.equal(x4o[: st['N'], 3], st['x4'][:, 3])
    assert bool(torch.isnan(x4o[st['N']:]).all())
    if mode == 1:
        assert torch.equal(c_next, st['c_t'] * 4.0)
    else:
        c_t, lg, cn = st['c_t'].double(), st['logits'].double(), st['cn'].double()
        cw = OS.reverse_update(c_t, lg, a, b, s, cn, 0)
        cterm = torch.maximum(torch.maximum((c_t / a64).abs(), (b64 * lg).abs()), (s64 * cn).abs())
        cerr = (c_next.double() - cw).abs()
        cbar = ULPS * _sp(cterm) + _sp(cw)
        assert bool((cerr <= cbar).all()), ('c_next', float((cerr / cbar).max()))
        rep['c_next'] = float((cerr / cbar).max()) if n else 0.0
        absmax['c_next'] = float(cerr.max()) if n else 0.0
    return rep, absmax


def _report(name, rows):
    worst, absmax = {}, {}
    for rep, ab in rows:
        for k, v in rep.items():
            worst[k] = max(worst.get(k, 0.0), v)
        for k, v in ab.items():
            absmax[k] = max(absmax.get(k, 0.0), v)
    print(f'{name}: largest error / bar {worst}; largest |error| {absmax}')


def _cases():
    return list(LAYOUTS.items()) + [('many_3000', _many_graphs(np.random.RandomState(77)))]


@pytest.mark.gpu
@pytest.mark.parametrize('K', KS)
@pytest.mark.parametrize('name,graphs', _cases(), ids=[c[0] for c in _cases()])
def test_sbdd_reverse_float64(name, graphs, K):
    rows = []
    for i, (label, coef) in enumerate(_sbdd_coefs()):
        st = _inputs(graphs, K, seed=1000 * K + i)
        rows.append(_sbdd_check(st, coef, _run_sbdd(st, coef)))
    _report(f'sbdd {name} K={K}', rows)


# ---- DiffBP ---------------------------------------------------------------------------------------------------------

def _run_bp(st, coef, eps_out=True, **over):
    st = dict(st, **over)
    x4, ptr, lig = _graph_args(dict(st, x4=_bp_x4(st)))
    n, K = st['n'], st['K']
    keep = [_d(st['x_pred']), _d(st['logits']), _d(st['x_t']), _d(st['c_onehot']), _d(st['gen'], torch.uint8, fill=0),
            _d(st['xn']), _d(st['u'])]
    xo, co, vo = _out(n, 3), _out(n, K), _out(n, 1, torch.int64)
    eo = _out(n, 3) if eps_out else None
    with torch.cuda.device(DEV):
        _lib.check(_lib.lib().cbg_bp_reverse_f32(x4.data_ptr(), ptr.data_ptr(), st['B'], lig.data_ptr(), n, K,
                                                 C.byref(coef), *[t.data_ptr() for t in keep], xo.data_ptr(),
                                                 co.data_ptr(), vo.data_ptr(), eo.data_ptr() if eo is not None else None,
                                                 _lib.stream_ptr(torch.device(DEV))))
    torch.cuda.synchronize()
    for t, w in ((xo, 'x_next'), (co, 'c_next'), (vo, 'v_next')) + (((eo, 'eps_out'),) if eo is not None else ()):
        _check_pad(t, n, w)
    return xo[:n].cpu(), co[:n].cpu(), vo[:n].cpu(), (eo[:n].cpu() if eo is not None else None), x4.cpu()


def _bp_x4(st):
    """x4 with the ligand rows holding x_com."""
    x4 = st['x4'].clone()
    x4[torch.from_numpy(st['lig_node']).long(), :3] = st['x_com']
    return x4


def _bp_types_check(st, coef, v, c):
    """The DiffBP type rule, exact where the kernel's fp32 comparisons are exact and against the float64 softmax argmax
    where the top two probabilities differ by more than 2^-14 of the larger (fp32 softmax error: about (K + 3) 2^-24)."""
    K = st['K']
    _, _, pr = OB.mask_type_update(st['logits'].double(), st['c_onehot'], coef.change_prob, st['gen'], st['u'], K)
    vt = st['c_onehot'].argmax(-1)                               # torch: first maximum, all-zero rows -> 0
    change = (st['u'] < torch.tensor(coef.change_prob, dtype=torch.float32)) & st['gen'] & (vt == 0)
    assert torch.equal(v[~change], vt[~change])
    top = pr.topk(min(2, K), dim=-1).values
    margin = (top[:, 0] - top[:, 1]) if K > 1 else torch.full((pr.shape[0],), 1.0, dtype=F64)
    lg = st['logits']
    tie = lg.topk(min(2, K), dim=-1).values
    exact_tie = (tie[:, 0] == tie[:, 1]) if K > 1 else torch.zeros(pr.shape[0], dtype=torch.bool)
    clear = (margin > 2.0 ** -14 * top[:, 0]) | exact_tie
    sel = change & clear
    assert torch.equal(v[sel], pr.argmax(-1)[sel]), int((v[sel] != pr.argmax(-1)[sel]).sum())
    assert torch.equal(c, F.one_hot(v, K).float())
    return int((change & ~clear).sum())


def _bp_check(st, coef, got):
    x_next, c_next, v_next, eps, x4o = got
    n, B, bl = st['n'], st['B'], st['bl']
    x_t, x_pred, x_com = st['x_t'].double(), st['x_pred'].double(), st['x_com'].double()
    noise, eps_com = OB.com_eps(x_pred, x_t, x_com, bl, num_graphs=B)
    eps64 = noise + eps_com
    L = torch.maximum(torch.maximum(x_pred.abs(), x_t.abs()), x_com.abs())
    e_el = ULPS * _sp(L)
    d1, d2 = (x_pred - x_t).abs(), (x_com - x_t).abs()
    e_mean = _depth(bl, B)[:, None] * U32 * (_seg(d1, bl, B) + _seg(d2, bl, B)) + _seg(e_el, bl, B, 'amax')
    ebar = e_el + e_mean[bl] + _sp(eps64)
    rep, absmax = {}, {}
    if eps is not None:
        err = (eps.double() - eps64).abs()
        assert bool((err <= ebar).all()), ('eps_out', int((err > ebar).sum()), float((err / ebar).max()))
        rep['eps_out'] = float((err / ebar).max()) if n else 0.0
        absmax['eps_out'] = float(err.max()) if n else 0.0
    want = OB.pos_score_update(eps64, x_t, coef.alpha_cumprod, coef.beta, coef.nonzero, st['gen'], st['xn'].double())
    ab, be, nz = (torch.tensor(v, dtype=F64) for v in (coef.alpha_cumprod, coef.beta, coef.nonzero))
    sig, den = (1 - ab).sqrt(), (1 - be).sqrt()
    term = torch.maximum(torch.maximum(x_t.abs() / den, (be * eps64 / sig).abs() / den), (nz * be.sqrt() * st['xn'].double()).abs())
    xbar = (be / sig / den) * ebar + ULPS * _sp(term) + _sp(want)
    gen = st['gen']
    err = (x_next.double() - want).abs()
    assert bool((err[gen] <= xbar[gen]).all()), ('x_next', float((err / xbar)[gen].max()))
    assert torch.equal(x_next[~gen], st['x_t'][~gen])                   # non-generated rows keep x_t bit for bit
    rep['x_next'] = float((err / xbar)[gen].max()) if bool(gen.any()) else 0.0
    absmax['x_next'] = float(err[gen].max()) if bool(gen.any()) else 0.0
    near = _bp_types_check(st, coef, v_next, c_next)
    assert torch.equal(x4o[: st['N']], _bp_x4(st)) and bool(torch.isnan(x4o[st['N']:]).all())   # x4 is only read
    return rep, absmax, near


@pytest.mark.gpu
@pytest.mark.parametrize('K', KS)
@pytest.mark.parametrize('name,graphs', _cases(), ids=[c[0] for c in _cases()])
def test_bp_reverse_float64(name, graphs, K):
    model = _bp_model()
    rows, near = [], 0
    for i, t in enumerate(T_STEPS):
        coef = model.step_coef(t)
        st = _inputs(graphs, K, seed=2000 * K + i)
        got = _run_bp(st, coef)
        rep, ab, nr = _bp_check(st, coef, got)
        rows.append((rep, ab))
        near += nr
        # eps_out NULL: the same step
        got2 = _run_bp(st, coef, eps_out=False)
        for a_, b_ in zip(got[:3], got2[:3]):
            assert torch.equal(a_, b_)
        if t == 0:                                                      # nonzero = 0: no noise
            assert coef.nonzero == 0.0
            got3 = _run_bp(st, coef, xn=st['xn'] * 50 + 3)
            assert torch.equal(got3[0], got[0])
    _report(f'bp {name} K={K}', rows)
    print(f'bp {name} K={K}: {near} changed rows within 2^-14 of a probability tie')


@pytest.mark.gpu
@pytest.mark.parametrize('K', KS)
def test_bp_type_rule_edges(K):
    """Crafted rows of the type rule (u < prob) & gen & (v_t == 0): u at prob and one fp32 step below it, prob = 1 at
    t = 0, atoms off the absorbing state, all-zero c_t rows, equal logits."""
    model = _bp_model()
    m = 60                                                              # rows per crafted group
    graphs = [(20, 8 * m), (0, 0), (5, 7)]
    j = K - 1                                                           # the predicted class of the crafted rows
    for i, t in enumerate(T_STEPS):
        coef = model.step_coef(t)
        prob = np.float32(coef.change_prob)
        st = _inputs(graphs, K, seed=3000 * K + i)
        lg, ct, u, gen = st['logits'], st['c_onehot'], st['u'], st['gen']
        lg[: 8 * m] = torch.from_numpy(np.random.RandomState(i).normal(0, 1, size=(8 * m, K)).astype(np.float32))
        lg[: 8 * m, j] += 12.0
        ct[: 8 * m] = F.one_hot(torch.zeros(8 * m, dtype=torch.long), K).float()
        gen[: 8 * m] = True
        g = [slice(k * m, (k + 1) * m) for k in range(8)]
        u[g[0]] = float(prob)                                           # u = prob: no change
        u[g[1]] = float(np.nextafter(prob, np.float32(0)))               # one step below: change
        u[g[2]] = 0.0
        if K > 1:                                                       # off the absorbing state: never changes
            lg[g[2]] = 0.0
            lg[g[2], 0] = 12.0
            ct[g[2]] = F.one_hot(torch.from_numpy(np.random.RandomState(5).randint(1, K, size=m)), K).float()
        ct[g[3]] = 0.0                                                  # all-zero c_t = state 0: changes
        u[g[3]] = 0.0
        ct[g[4]] = 0.0                                                  # ... and stays 0 when not generated
        gen[g[4]] = False
        u[g[4]] = 0.0
        lg[g[5]] = 2.5                                                  # equal logits: the lowest of the tied classes
        lg[g[5], : min(2, K - 1)] = -4.0
        u[g[5]] = 0.0
        u[g[6]] = torch.from_numpy(np.random.RandomState(6).random_sample(m).astype(np.float32))
        u[g[7]] = float(np.float32(1 - 2 ** -24))
        _, c, v, _, _ = _run_bp(st, coef)
        assert torch.equal(c, F.one_hot(v, K).float())
        assert bool((v[g[0]] == 0).all()) and bool((v[g[1]] == j).all()), t
        if K > 1:
            assert torch.equal(v[g[2]], ct[g[2]].argmax(-1)), t
        assert bool((v[g[3]] == j).all()) and bool((v[g[4]] == 0).all()), t
        assert bool((v[g[5]] == min(2, K - 1)).all()), t
        if t == 0:                                                      # prob = 1: every u in [0, 1) changes
            assert coef.change_prob == 1.0
            assert bool((v[g[6]] == j).all()) and bool((v[g[7]] == j).all())
        _bp_types_check(st, coef, v, c)


# ---- invariants: repeat calls, a graph alone vs inside a batch ------------------------------------------------------

def _subgraph(st, g):
    """Graph g of ``st`` as a one-graph input (its rows sliced, indices rebased)."""
    p0, p1 = int(st['ptr'][g]), int(st['ptr'][g + 1])
    lm = (st['bl'] == g).numpy()
    out = dict(st, ptr=np.array([0, p1 - p0], np.int32), lig_node=(st['lig_node'][lm] - p0).astype(np.int32),
               is_lig=st['is_lig'][p0:p1], bl=torch.zeros(int(lm.sum()), dtype=torch.long),
               bn=torch.zeros(p1 - p0, dtype=torch.long), B=1, N=p1 - p0, n=int(lm.sum()), x4=st['x4'][p0:p1])
    for k in ('x_t', 'x_com', 'x_pred', 'c_t', 'c_onehot', 'logits', 'xn', 'cn', 'gen', 'u'):
        out[k] = st[k][torch.from_numpy(lm)]
    return out, p0, p1, torch.from_numpy(lm)


@pytest.mark.gpu
@pytest.mark.parametrize('K', [13, 16])
def test_per_graph_kernels_repeatable_and_batch_independent(K):
    graphs = [gr for _, gs in _cases() for gr in gs]
    st = _inputs(graphs, K, seed=K)
    rs = np.random.RandomState(K)
    big = [g for g, (_, nl) in enumerate(graphs) if nl > 3]
    picks = big + list(rs.choice(len(graphs), size=30, replace=False))
    sb = dict(_sbdd_coefs())['t500']
    bpc = _bp_model().step_coef(T_SCHED // 2)
    a, b = _run_sbdd(st, sb), _run_sbdd(st, sb)
    for u_, w_ in zip(a, b):
        assert torch.equal(u_.nan_to_num(7.0), w_.nan_to_num(7.0))
    p, q = _run_bp(st, bpc), _run_bp(st, bpc)
    for u_, w_ in zip(p, q):
        assert torch.equal(u_.nan_to_num(7.0), w_.nan_to_num(7.0))
    for g in picks:
        sub, p0, p1, lm = _subgraph(st, int(g))
        xs, cs, x4s = _run_sbdd(sub, sb)
        assert torch.equal(xs, a[0][lm]) and torch.equal(cs, a[1][lm]) and torch.equal(x4s[: p1 - p0], a[2][p0:p1]), g
        xb, cb, vb, eb, _ = _run_bp(sub, bpc)
        assert torch.equal(xb, p[0][lm]) and torch.equal(cb, p[1][lm]) and torch.equal(vb, p[2][lm]), g
        assert torch.equal(eb, p[3][lm]), g


# ---- TargetDiff (reverse_kernel, one thread per atom) ---------------------------------------------------------------

def _run_td(coef, st):
    n, K = st['x0'].shape[0], st['c'].shape[1]
    keep = [_d(st[k]) for k in ('x0', 'logits', 'x_t', 'c')] + [_d(st['gen'], torch.uint8, fill=0), _d(st['pn']),
                                                                _d(st['u'])]
    xo, co, vo = _out(n, 3), _out(n, K), _out(n, 1, torch.int64)
    with torch.cuda.device(DEV):
        _lib.check(_lib.lib().cbg_reverse_step_f32(C.byref(coef), *[t.data_ptr() for t in keep], n, K, xo.data_ptr(),
                                                   co.data_ptr(), vo.data_ptr(), _lib.stream_ptr(torch.device(DEV))))
    torch.cuda.synchronize()
    for t, w in ((xo, 'x_next'), (co, 'c_next'), (vo, 'v_next')):
        _check_pad(t, n, w)
    return xo[:n].cpu(), co[:n].cpu(), vo[:n].cpu()


def _td_scalars(coef):
    return (coef.log_alphas_cumprod_prev, coef.log_one_minus_alphas_cumprod_prev, coef.log_alpha,
            coef.log_one_minus_alpha)


def _td_gap_rows(coef, K, m):
    """Rows (c_t one-hot at class 0, logits 0 / g / -200, u = 0 except u = 0.9999 at class 1) whose class flips
    between the 1e-8 of log(c_t + 1e-8) and a negligible constant: g sits midway between the two logit gaps where
    class 1 starts to win.  -> (logits, u)."""
    lac, l1mac, la, l1ma = (torch.tensor(v, dtype=F64) for v in _td_scalars(coef))
    lk = math.log(K)
    u = torch.zeros(K)
    u[1] = float(np.float32(0.9999))
    gum = -torch.log(-torch.log(u.double() + 1e-30) + 1e-30)
    ct = torch.zeros(K, dtype=F64)
    ct[0] = 1.0

    def diff(g, const):
        lg = torch.full((g.shape[0], K), -200.0, dtype=F64)
        lg[:, 0], lg[:, 1] = 0.0, g
        un = torch.logaddexp(F.log_softmax(lg, -1) + lac, l1mac - lk) + torch.logaddexp(torch.log(ct + const) + la,
                                                                                        l1ma - lk)
        sc = un + gum
        return sc[:, 1] - sc[:, 0]
    grid = torch.linspace(-40, 40, 800001, dtype=F64)
    g8 = grid[int((diff(grid, 1e-8) > 0).nonzero()[0])]
    g30 = grid[int((diff(grid, 1e-30) > 0).nonzero()[0])]
    assert abs(float(g8 - g30)) > 4e-4, (float(g8), float(g30))
    lg = torch.full((m, K), -200.0)
    lg[:, 0], lg[:, 1] = 0.0, float((g8 + g30) / 2)
    return lg, u.expand(m, K).clone()


def _td_state(rs, n, K, t, coef):
    f = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))
    st = dict(x0=f(OFFSET + rs.normal(0, 40, size=(n, 3))), x_t=f(OFFSET + rs.normal(0, 40, size=(n, 3))),
              logits=f(rs.normal(0, 3, size=(n, K))), c=f(np.eye(K)[rs.randint(0, K, size=n)]),
              gen=torch.from_numpy(rs.random_sample(n) < 0.85), pn=f(rs.normal(size=(n, 3))),
              u=f(rs.random_sample(size=(n, K))))
    q = n // 16
    lg, c, u = st['logits'], st['c'], st['u']
    lg[:q] = 1.25                                                        # equal logits
    lg[q:2 * q] = f(rs.uniform(-80, 80, size=(q, K)))                    # logits over +-80
    c[2 * q:3 * q] = 0.0                                                 # all-zero c_t
    c[3 * q:4 * q] = f(rs.dirichlet(np.ones(K), size=q))                 # soft c_t
    u[4 * q:5 * q, rs.randint(K)] = 0.0                                  # u = 0 (gumbel -log(-log(1e-30)))
    u[5 * q:6 * q, rs.randint(K)] = float(np.float32(1 - 2 ** -24))      # the largest fp32 below 1
    u[6 * q:6 * q + q // 2] = 0.0
    u[6 * q + q // 2:7 * q] = float(np.float32(1 - 2 ** -24))
    # non-generated rows with ties in c_t: argmax keeps the lowest index
    c[7 * q:7 * q + 40] = 0.0
    if K > 2:
        c[7 * q + 20:7 * q + 40, 1] = 0.5
        c[7 * q + 20:7 * q + 40, K - 1] = 0.5
    st['gen'][7 * q:7 * q + 40] = False
    n_gap = 0
    if t <= 1 and K > 1:                                                 # the 1e-8 constant decides these rows
        n_gap = q
        lg[8 * q:9 * q], u[8 * q:9 * q] = _td_gap_rows(coef, K, q)
        c[8 * q:9 * q] = F.one_hot(torch.zeros(q, dtype=torch.long), K).float()
        st['gen'][8 * q:9 * q] = True
    return st, slice(8 * q, 8 * q + n_gap)


@pytest.mark.gpu
@pytest.mark.parametrize('K', KS)
def test_targetdiff_reverse_float64(K):
    model = _td_model()
    rs = np.random.RandomState(40 + K)
    n = 4000
    near, total, worst, absmax = 0, 0, 0.0, 0.0
    for t in T_STEPS:
        coef = model.step_coef(t)
        st, gap = _td_state(rs, n, K, t, coef)
        x, c, v = _run_td(coef, st)
        gen = st['gen']
        # positions
        want = OD.pos_reverse_update(st['x0'].double(), st['x_t'].double(), coef.pos_c0, coef.pos_ct, coef.pos_logvar,
                                     coef.pos_nonzero, gen, st['pn'].double())
        sig = math.exp(0.5 * coef.pos_logvar) * coef.pos_nonzero
        term = torch.maximum(torch.maximum((coef.pos_c0 * st['x0'].double()).abs(), (coef.pos_ct * st['x_t'].double()).abs()),
                             (sig * st['pn'].double()).abs())
        bar = ULPS * _sp(term) + _sp(want)
        err = (x.double() - want).abs()
        assert bool((err[gen] <= bar[gen]).all()), (t, float((err / bar)[gen].max()))
        worst, absmax = max(worst, float((err / bar)[gen].max())), max(absmax, float(err[gen].max()))
        assert torch.equal(x[~gen], st['x_t'][~gen]), t
        if t == 0:                                                       # no noise at t = 0
            assert coef.pos_nonzero == 0.0
            assert torch.equal(_run_td(coef, dict(st, pn=st['pn'] * 100 + 1))[0], x)
        # types
        assert torch.equal(c, F.one_hot(v, K).float())
        assert torch.equal(v[~gen], st['c'][~gen].argmax(-1)), t        # torch.argmax: the lowest index on ties
        if K > 2:
            assert bool((v[7 * (n // 16) + 20:7 * (n // 16) + 40] == 1).all())
        _, _, score = OD.type_reverse_update(st['logits'].double(), st['c'], *_td_scalars(coef), gen, st['u'], K)
        top = score.topk(min(2, K), dim=-1).values
        margin = (top[:, 0] - top[:, 1]) if K > 1 else torch.full((n,), float('inf'), dtype=F64)
        clear = gen & (margin > 1e-4)
        wv = score.argmax(-1)
        assert torch.equal(v[clear], wv[clear]), (t, int((v[clear] != wv[clear]).sum()))
        if gap.stop > gap.start:                                         # 1e-8 decides: class 1 everywhere
            assert bool(clear[gap].all()) and bool((v[gap] == 1).all()), t
        near += int((gen & ~clear).sum())
        total += int(gen.sum())
    print(f'targetdiff K={K}: positions largest error / bar {worst:.3f}, largest |error| {absmax:.3e}; '
          f'{near} of {total} generated rows within 1e-4 of a Gumbel-max tie')
    assert near <= 1e-3 * total


# ---- production entry points --------------------------------------------------------------------------------------

PROD_BATCH = dict(n_prot=[60, 40, 30], n_lig=[150, 12, 7])            # the first graph: 150 ligand atoms


def _prod_model(cls, cfg_fn):
    model = cls(cfg_fn(num_steps=T_SCHED, num_layers=2))
    sd = synthetic.seeded_state_dict(model, seed=WEIGHT_SEED)
    model.load_state_dict(sd, strict=True)
    return model.eval().to(DEV)


@pytest.mark.gpu
def test_sbdd_step_matches_float64():
    model = _prod_model(DiffSBDDB200, synthetic.diffsbdd_config)
    batch = synthetic.make_batch(PROD_BATCH['n_prot'], PROD_BATCH['n_lig'], seed=8)
    state = model.begin(batch)
    K, n, plan = model.num_classes, state['n_lig'], state['plan']
    bl = batch['ligand_element_batch'].long()
    L = _lib.lib()
    rs = np.random.RandomState(3)
    for label, coef in _sbdd_coefs():
        x_t, c_t = state['X'][T_SCHED].clone(), state['C'][T_SCHED].clone()
        nx = torch.from_numpy(rs.normal(size=(n, 3)).astype(np.float32)).to(DEV)
        nc = torch.from_numpy(rs.normal(size=(n, K)).astype(np.float32)).to(DEV)
        xo, co, xp, lg = (torch.full((n, w), float('nan'), device=DEV) for w in (3, K, 3, K))
        with torch.cuda.device(DEV):
            _lib.check(L.cbg_sbdd_step_f32(C.byref(plan), C.byref(coef), x_t.data_ptr(), c_t.data_ptr(), nx.data_ptr(),
                                           nc.data_ptr(), xo.data_ptr(), co.data_ptr(), xp.data_ptr(), lg.data_ptr(),
                                           _lib.stream_ptr(torch.device(DEV))))
        torch.cuda.synchronize()
        x_t, c_t, nx, nc, xo, co, xp, lg = (v.cpu() for v in (x_t, c_t, nx, nc, xo, co, xp, lg))
        B = 3
        zs = OS.reverse_update(x_t.double(), xp.double(), coef.a, coef.b, coef.s, nx.double(), coef.mode)
        want = zs - _seg(zs, bl, B)[bl]
        a64 = torch.tensor(coef.a, dtype=F64)
        term = torch.maximum(torch.maximum(x_t.double().abs() * (1 / a64 if coef.mode == 0 else a64),
                                           (coef.b * xp.double()).abs() * (1 if coef.mode == 0 else a64)),
                             (coef.s * nx.double()).abs())
        e_zs = ULPS * _sp(term)
        bar = e_zs + (_depth(bl, B)[:, None] * U32 * _seg(zs.abs(), bl, B) + _seg(e_zs, bl, B, 'amax'))[bl] + _sp(want)
        err = (xo.double() - want).abs()
        assert bool((err <= bar).all()), (label, float((err / bar).max()))
        if coef.mode == 1:
            assert torch.equal(co, c_t * 4.0)
        else:
            cw = OS.reverse_update(c_t.double(), lg.double(), coef.a, coef.b, coef.s, nc.double(), 0)
            cterm = torch.maximum(torch.maximum((c_t.double() / a64).abs(), (coef.b * lg.double()).abs()),
                                  (coef.s * nc.double()).abs())
            assert bool(((co.double() - cw).abs() <= ULPS * _sp(cterm) + _sp(cw)).all()), label


@pytest.mark.gpu
def test_bp_step_matches_float64():
    model = _prod_model(DiffBPB200, synthetic.diffbp_config)
    batch = synthetic.make_batch(PROD_BATCH['n_prot'], PROD_BATCH['n_lig'], seed=9)
    state = model.prepare(batch)
    K, n, plan = model.num_classes, state['n_lig'], state['plan']
    com_blob = model.com_head.packed_blob(torch.device(DEV))
    gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag']).bool()
    L = _lib.lib()
    rs = np.random.RandomState(4)
    for t in T_STEPS:
        coef = model.step_coef(t)
        x_t, c_t = state['x_lig'].clone(), state['c_lig'].clone()
        pn = torch.from_numpy(rs.normal(size=(n, 3)).astype(np.float32)).to(DEV)
        u = torch.from_numpy(rs.random_sample(n).astype(np.float32)).to(DEV)
        xo, co, eo, lg = (torch.full((n, w), float('nan'), device=DEV) for w in (3, K, 3, K))
        vo = torch.full((n,), -7, dtype=torch.int64, device=DEV)
        with torch.cuda.device(DEV):
            _lib.check(L.cbg_bp_step_f32(C.byref(plan), com_blob.data_ptr(), model.com_head.num_layers, C.byref(coef),
                                         x_t.data_ptr(), c_t.data_ptr(), pn.data_ptr(), u.data_ptr(), xo.data_ptr(),
                                         co.data_ptr(), vo.data_ptr(), eo.data_ptr(), lg.data_ptr(),
                                         _lib.stream_ptr(torch.device(DEV))))
        torch.cuda.synchronize()
        x_t, c_t, pn, u, xo, co, eo, lg, vo = (v.cpu() for v in (x_t, c_t, pn, u, xo, co, eo, lg, vo))
        assert bool(torch.isfinite(eo).all())
        want = OB.pos_score_update(eo.double(), x_t.double(), coef.alpha_cumprod, coef.beta, coef.nonzero, gen,
                                   pn.double())
        be, sig = coef.beta, math.sqrt(1 - coef.alpha_cumprod)
        den = math.sqrt(1 - be)
        term = torch.maximum(torch.maximum(x_t.double().abs() / den, (be * eo.double() / sig).abs() / den),
                             (coef.nonzero * math.sqrt(be) * pn.double()).abs())
        err = (xo.double() - want).abs()
        assert bool((err <= ULPS * _sp(term) + _sp(want)).all()), (t, float(err.max()))
        st = dict(K=K, logits=lg, c_onehot=c_t, gen=gen, u=u)
        _bp_types_check(st, coef, vo, co)


@pytest.mark.gpu
def test_targetdiff_step_matches_float64():
    model = _prod_model(type(_td_model()), synthetic.targetdiff_config)
    batch = synthetic.make_batch(PROD_BATCH['n_prot'], PROD_BATCH['n_lig'], seed=10)
    state = model.prepare(batch)
    K, n, plan = model.num_classes, state['n_lig'], state['plan']
    gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag']).bool()
    L = _lib.lib()
    rs = np.random.RandomState(5)
    for t in (T_SCHED - 1, 1):
        coef = model.step_coef(t)
        x_t, c_t = state['x_lig'].clone(), state['c_lig'].clone()
        pn = torch.from_numpy(rs.normal(size=(n, 3)).astype(np.float32)).to(DEV)
        u = torch.from_numpy(rs.random_sample((n, K)).astype(np.float32)).to(DEV)
        xo, co, x0, lg = (torch.full((n, w), float('nan'), device=DEV) for w in (3, K, 3, K))
        vo = torch.full((n,), -7, dtype=torch.int64, device=DEV)
        with torch.cuda.device(DEV):
            _lib.check(L.cbg_sample_step_f32(C.byref(plan), C.byref(coef), x_t.data_ptr(), c_t.data_ptr(), pn.data_ptr(),
                                             u.data_ptr(), xo.data_ptr(), co.data_ptr(), vo.data_ptr(), x0.data_ptr(),
                                             lg.data_ptr(), _lib.stream_ptr(torch.device(DEV))))
        torch.cuda.synchronize()
        x_t, c_t, pn, u, xo, co, x0, lg, vo = (v.cpu() for v in (x_t, c_t, pn, u, xo, co, x0, lg, vo))
        want = OD.pos_reverse_update(x0.double(), x_t.double(), coef.pos_c0, coef.pos_ct, coef.pos_logvar,
                                     coef.pos_nonzero, gen, pn.double())
        sig = math.exp(0.5 * coef.pos_logvar) * coef.pos_nonzero
        term = torch.maximum(torch.maximum((coef.pos_c0 * x0.double()).abs(), (coef.pos_ct * x_t.double()).abs()),
                             (sig * pn.double()).abs())
        err = (xo.double() - want).abs()
        assert bool((err <= ULPS * _sp(term) + _sp(want)).all()), (t, float(err.max()))
        _, vw, score = OD.type_reverse_update(lg.double(), c_t, *_td_scalars(coef), gen, u, K)
        top = score.topk(2, dim=-1).values
        clear = ~gen | (top[:, 0] - top[:, 1] > 1e-4)
        assert int((~clear).sum()) <= 1
        assert torch.equal(vo[clear], vw[clear]), t
        assert torch.equal(co, F.one_hot(vo, K).float())


# ---- argument refusals (no device needed) -------------------------------------------------------------------------

P = 1 << 20          # aligned non-NULL pointer value, never dereferenced: the checks fail first


def _err():
    return _lib.lib().cbg_last_error().decode()


def test_sbdd_reverse_refusals():
    L = _lib.lib()
    coef = _lib.SbddCoef(a=1.0, b=0.5, s=0.1, mode=0)

    def rc(n_graphs=2, n_lig=4, K=13, c=coef, ptrs=None):
        p = ptrs if ptrs is not None else [P] * 10
        return L.cbg_sbdd_reverse_f32(p[0], p[1], n_graphs, p[2], n_lig, K, C.byref(c) if c is not None else None,
                                      *p[3:], None)
    for i in range(10):
        ptrs = [P] * 10
        ptrs[i] = None
        assert rc(ptrs=ptrs) != 0 and 'null argument' in _err(), i
    assert rc(c=None) != 0 and 'null argument' in _err()
    for kw, msg in (({'K': 0}, 'num_classes=0'), ({'K': 17}, 'num_classes=17'), ({'n_graphs': -1}, 'n_graphs=-1'),
                    ({'n_lig': -1}, 'n_lig=-1')):
        assert rc(**kw) != 0 and msg in _err(), kw
    for mode in (-1, 2):
        assert rc(c=_lib.SbddCoef(a=1.0, b=0.5, s=0.1, mode=mode)) != 0 and f'mode={mode}' in _err()


def test_bp_reverse_refusals():
    L = _lib.lib()
    coef = _lib.BpCoef(alpha_cumprod=0.5, beta=0.01, nonzero=1.0, change_prob=0.5)

    def rc(n_graphs=2, n_lig=4, K=13, c=coef, ptrs=None):
        p = ptrs if ptrs is not None else [P] * 13
        return L.cbg_bp_reverse_f32(p[0], p[1], n_graphs, p[2], n_lig, K, C.byref(c) if c is not None else None,
                                    *p[3:], None, None)
    for i in range(13):                                                 # eps_out (optional) follows these
        ptrs = [P] * 13
        ptrs[i] = None
        assert rc(ptrs=ptrs) != 0 and 'null argument' in _err(), i
    assert rc(c=None) != 0 and 'null argument' in _err()
    for kw, msg in (({'K': 0}, 'num_classes=0'), ({'K': 17}, 'num_classes=17'), ({'n_graphs': -1}, 'n_graphs=-1'),
                    ({'n_lig': -1}, 'n_lig=-1')):
        assert rc(**kw) != 0 and msg in _err(), kw


def test_reverse_step_refusals():
    L = _lib.lib()
    coef = _lib.StepCoef()

    def rc(n=4, K=13, c=coef, ptrs=None):
        p = ptrs if ptrs is not None else [P] * 10
        return L.cbg_reverse_step_f32(C.byref(c) if c is not None else None, *p[:7], n, K, *p[7:], None)
    for i in range(10):
        ptrs = [P] * 10
        ptrs[i] = None
        assert rc(ptrs=ptrs) != 0 and 'null argument' in _err(), i
    assert rc(c=None) != 0 and 'null argument' in _err()
    assert rc(n=-1) != 0 and 'n=-1' in _err()
    for K in (0, 17):
        assert rc(K=K) != 0 and f'num_classes={K}' in _err()
