"""The D3FG kernels one by one against plain references (DESIGN.md section 16, "Checks").

- fg_reverse_kernel through the cbg_fg_reverse_f32 hook: positions and the drawn angle bit for bit against the fp32
  expressions of tests/fg_sample_oracle.reverse_step, the histogram bin against the float64 searchsorted one, the
  orientation against the float64 product exp(e) exp(o_pred) (including composed angles at and near 0 and pi), the FG
  type against the float64 Gumbel-max class.
- ipa_heads_kernel through cbg_ipa_forward_f32 with num_sublayers = 0 and crafted head weights that pass chosen per-row
  values through exactly: R_next, eps_pos, exp(o_next) and the logits against float64.
- the encoder body (ipa_linear_kernel, ipa_ln_relu_kernel, ipa_x2h_kernel) against a float64 oracle pass on the same
  neighbour table, with a bar calibrated by the fp32 oracle's own error.
CPU: the argument checks of both entry points."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from cbgbench_b200 import _lib, synthetic
from cbgbench_b200.difffg import D3FGB200, multinomial_bin
from cbgbench_b200.ipatransformer import IPATransformerB200
from oracle import graph_ops as G
from oracle import ipa as OI

import fg_sample_oracle as OF

torch.set_grad_enabled(False)
DEV = 'cuda:0'
T_SCHED = 50                 # steps of the schedule the reverse-step tests draw their coefficients from
T_STEPS = (0, 1, T_SCHED // 2, T_SCHED - 1)
ROT_BAR = 2e-6               # per matrix element: about ten fp32 ulps of a unit entry
PI32 = float(np.float32(np.pi))
PI_MAX = PI32 * (1 + 2 ** -22)     # |o_next| <= pi up to the rounding of fp32 pi and of the product theta n
F32 = np.float32


def _exp64(w):
    return OI.so3vec_to_rotation(torch.as_tensor(w).double())


def _log64(R):
    """float64 so3 vector of rotation matrices R (the project's exp(w) is scipy's exp(w) transposed)."""
    R = torch.as_tensor(R).double()
    return torch.from_numpy(Rotation.from_matrix(R.transpose(-1, -2).numpy()).as_rotvec())


def _angle64(R):
    return torch.linalg.norm(_log64(R), dim=-1)


def _unit(rs, n):
    a = rs.normal(size=(n, 3))
    return a / np.linalg.norm(a, axis=1, keepdims=True)


_MODELS = {}


def _model(K):
    if K not in _MODELS:
        _MODELS[K] = D3FGB200(synthetic.difffg_config(num_steps=T_SCHED, num_layers=1, num_fgtype=K)).eval()
    return _MODELS[K]


def _coef(model, t):
    inv = model.rot_scheduler.angular_distrib_inv
    return model.step_coef(t, inv.stddevs.cpu(), inv.approx_flag.cpu())


def _gauss_t(model):
    inv = model.rot_scheduler.angular_distrib_inv
    return max(t for t in range(2, T_SCHED) if bool(inv.approx_flag[t]))


def _hist_ts(model):
    inv = model.rot_scheduler.angular_distrib_inv
    return [t for t in (T_SCHED // 2, T_SCHED - 1) if not bool(inv.approx_flag[t])]


def _run_reverse(model, t, st, Y=None, coef=None, extra_rows=7, seed=0):
    """cbg_fg_reverse_f32 on the ligand rows ``st`` (dict of CPU tensors: x, c, o, eps, o_pred, logits, gen, pn, rd, tu).
    The encoder rows are scattered into a composed array with ``extra_rows`` foreign rows at shuffled positions, so the
    kernel must read them at lig_node.  ``Y``: angular histograms to use instead of the model's.  -> (x, c, o, theta)."""
    n, K = st['c'].shape
    N = n + extra_rows
    g = torch.Generator().manual_seed(seed)
    lig_node = torch.randperm(N, generator=g)[:n].to(torch.int32)
    comp = lambda v, w: torch.full((N, w), 1e3).index_copy_(0, lig_node.long(), v.float())
    inv = model.rot_scheduler.angular_distrib_inv
    Yt = inv.Y if Y is None else Y
    X = inv.X.float().contiguous()
    cdf = Yt.detach().cpu()[:, :-1].double().cumsum(-1)
    d = lambda v, dt=torch.float32: v.to(DEV, dt).contiguous()
    keep = dict(lig_node=d(lig_node, torch.int32), gen=d(st['gen'], torch.uint8), X=d(X), cdf=d(cdf, torch.float64),
                eps=d(comp(st['eps'], 3)), o_pred=d(comp(st['o_pred'], 3)), logits=d(comp(st['logits'], K)),
                x=d(st['x']), c=d(st['c']), o=d(st['o']), pn=d(st['pn']), rd=d(st['rd']), tu=d(st['tu']))
    out = [torch.full((n, w), float('nan'), device=DEV) for w in (3, K, 3, 1)]
    plan = _lib.FgPlan(num_classes=K, n_lig=n, lig_node=keep['lig_node'].data_ptr(), gen_lig=keep['gen'].data_ptr(),
                       angle_x=keep['X'].data_ptr(), angle_cdf=keep['cdf'].data_ptr(), n_bins=X.shape[1])
    L = _lib.lib()
    with torch.cuda.device(DEV):
        _lib.check(L.cbg_fg_reverse_f32(C.byref(plan), coef if coef is not None else _coef(model, t),
                                        *[keep[k].data_ptr() for k in ('eps', 'o_pred', 'logits', 'x', 'c', 'o', 'pn', 'rd', 'tu')],
                                        *[o.data_ptr() for o in out], _lib.stream_ptr(torch.device(DEV))))
    torch.cuda.synchronize()
    x, c, o, th = (v.cpu() for v in out)
    return x, c, o, th[:, 0]


def _oracle(model, t, st, dtype=torch.float32, theta=None, Y=None):
    sd = dict(model.state_dict())
    if Y is not None:
        sd['rot_scheduler.angular_distrib_inv.Y'] = Y
    n = st['x'].shape[0]
    return OF.reverse_step(sd, t, torch.zeros(n, dtype=torch.long), st['x'].to(dtype), st['c'], st['o'].to(dtype),
                           st['eps'], st['o_pred'], st['logits'], st['gen'], st['pn'], st['rd'], st['tu'], theta=theta)


def _state(rs, n, K, gen_frac=0.8):
    f = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))
    rd = np.concatenate([rs.normal(size=(n, 3)), rs.random_sample(size=(n, 2)), rs.normal(size=(n, 1))], axis=1)
    return dict(x=f(rs.normal(0, 5, size=(n, 3))), c=f(np.eye(K)[rs.randint(0, K, size=n)]),
                o=f(rs.normal(0, 1.2, size=(n, 3))), eps=f(rs.normal(size=(n, 3))), o_pred=f(rs.normal(0, 1.2, size=(n, 3))),
                logits=f(rs.normal(0, 3, size=(n, K))), gen=torch.from_numpy(rs.random_sample(n) < gen_frac),
                pn=f(rs.normal(size=(n, 3))), rd=f(rd), tu=f(rs.random_sample(size=(n, K))))


# ---- reverse step: positions ----------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('K', [1, 17, 28, 32])
def test_reverse_positions_bit_exact(K):
    model = _model(K)
    rs = np.random.RandomState(K)
    n = 800
    for t in T_STEPS:
        st = _state(rs, n, K)
        mag = np.exp2(rs.uniform(-20, 20, size=(n, 3))) * np.sign(rs.normal(size=(n, 3)))
        mag[:9] = np.exp2(np.arange(-20, 21, 5))[:, None]          # the ends of the range, exactly
        st['eps'] = torch.from_numpy(mag.astype(np.float32))
        x, _, _, _ = _run_reverse(model, t, st, seed=t)
        want = _oracle(model, t, st)[0]
        gen = st['gen']
        assert torch.equal(x[gen], want[gen]), (t, (x - want).abs().max())
        assert torch.equal(x[~gen], st['x'][~gen]), t                          # non-generated rows are not touched
        if t == 0:                                                             # no noise at t = 0
            st['pn'] = torch.randn(n, 3) * 100
            assert torch.equal(_run_reverse(model, t, st)[0], x)


# ---- reverse step: the angle draw -----------------------------------------------------------------------------------------

def _theta_definition(model, t, rd, Y=None):
    """fp32 theta of so3.py:111-138 for draws rd [n,6] (the bin by multinomial_bin) and the bin itself."""
    inv = model.rot_scheduler.angular_distrib_inv
    Yt = (inv.Y if Y is None else Y)[t]
    X, std = inv.X[t], inv.stddevs[t]
    b = multinomial_bin(Yt[:-1].expand(rd.shape[0], -1), rd[:, 3])
    hist = X[b] + rd[:, 4] * (X[b + 1] - X[b])
    gauss = (std * 2 + rd[:, 5] * std).abs() % math.pi
    return (gauss if bool(inv.approx_flag[t]) else hist), b


def _edge_draws(rs, Yt, n_edges=300):
    """Bin uniforms at the edges of the histogram's CDF: 0, 1 - 2^-24, and one fp32 ulp either side of (and at) each of
    ``n_edges`` ratios C[i] / C[last]."""
    cdf = Yt[:-1].double().cumsum(0)
    idx = rs.choice(len(cdf) - 1, size=min(n_edges, len(cdf) - 1), replace=False)
    r = (cdf[idx] / cdf[-1]).numpy().astype(np.float32)
    u = np.concatenate([[0.0, 1 - 2 ** -24], np.nextafter(r, F32(0)), r, np.nextafter(r, F32(1))]).astype(np.float32)
    return np.clip(u, 0, np.float32(1 - 2 ** -24))


def _zero_bin_histogram(model, rs):
    """The model's histograms with a third of the bins and a tail set to zero weight."""
    Y = model.rot_scheduler.angular_distrib_inv.Y.clone()
    nb = Y.shape[1]
    Y[:, rs.choice(nb, size=nb // 3, replace=False)] = 0
    Y[:, nb - 400:] = 0
    Y[:, 100:140] = 0
    return Y


@pytest.mark.gpu
def test_reverse_angle_draw_bit_exact():
    model = _model(28)
    rs = np.random.RandomState(11)
    inv = model.rot_scheduler.angular_distrib_inv
    cases = [(t, None) for t in _hist_ts(model)] + [(_hist_ts(model)[0], _zero_bin_histogram(model, rs))]
    assert cases
    for t, Y in cases:
        Yt = (inv.Y if Y is None else Y)[t]
        u = _edge_draws(rs, Yt)
        n = len(u) + 200
        st = _state(rs, n, 28)
        st['rd'][:len(u), 3] = torch.from_numpy(u)
        st['rd'][: n // 2, 4] = 0.0                        # in-bin offset 0: theta is the bin's left edge
        _, _, _, th = _run_reverse(model, t, st, Y=Y)
        want, b = _theta_definition(model, t, st['rd'], Y=Y)
        assert torch.equal(th, want), (t, int((th != want).sum()))
        # the bin: the float64 searchsorted one (read back exactly where the offset is 0), never a zero-weight bin
        kb = torch.searchsorted(inv.X[t], th[: n // 2].contiguous())
        assert torch.equal(kb, b[: n // 2]), t
        assert bool((Yt[b] > 0).all()) and bool((Yt[kb] > 0).all()), t
        if Y is not None:
            assert int((Yt[:-1] == 0).sum()) > 1000
    # Gaussian branch: |2 sigma + sigma n| just below, at and above fp32 pi (the fmod wrap), and n = -2 (theta = 0)
    t = _gauss_t(model)
    s = F32(inv.stddevs[t])
    val = lambda nn: F32(abs(F32(F32(s * F32(2)) + F32(nn * s))))
    lo = hi = F32((np.pi - 2 * float(s)) / float(s))
    cand = [lo]
    for _ in range(200):
        lo, hi = np.nextafter(lo, F32(0)), np.nextafter(hi, F32(100))
        cand += [lo, hi]
    cand = sorted(cand)
    pick = [c for c in cand if val(c) < F32(np.pi)][-3:] + [c for c in cand if val(c) == F32(np.pi)][:3] + \
           [c for c in cand if val(c) > F32(np.pi)][:3]
    assert any(val(c) == F32(np.pi) for c in pick) and any(val(c) > F32(np.pi) for c in pick)
    gd = np.array(pick + [-2.0, -2.0, 0.0, 3.0, -30.0], dtype=np.float32)
    st = _state(rs, len(gd), 28)
    st['rd'][:, 5] = torch.from_numpy(gd)
    _, _, _, th = _run_reverse(model, t, st)
    want, _ = _theta_definition(model, t, st['rd'])
    assert torch.equal(th, want), (th, want)
    assert float(th[len(pick)]) == 0.0
    # t <= 1: no rotation noise
    for t in (0, 1):
        st = _state(rs, 64, 28)
        _, _, o, th = _run_reverse(model, t, st)
        assert not th.any()
        st2 = dict(st, rd=torch.randn(64, 6))
        assert torch.equal(_run_reverse(model, t, st2)[2], o)


# ---- reverse step: the orientation --------------------------------------------------------------------------------------

def _targeted_o_pred(rs, e, n_per):
    """o_pred rows whose composition exp(e) exp(o_pred) (float64) has the angle 0, pi, and delta / pi - delta for delta
    in 1e-7 ... 1e-2, along random axes; e [m,3] float64 noise vectors, one per row."""
    deltas = [1e-7, 3e-7, 1e-6, 1e-5, 1e-4, 1e-3, 1e-2]
    angles = [0.0, np.pi] + deltas + [np.pi - d for d in deltas]
    ang = np.repeat(np.array(angles), n_per)
    w = _unit(rs, len(ang)) * ang[:, None]
    E = _exp64(e[: len(ang)])
    Rt = _exp64(torch.from_numpy(w))
    return _log64(E.transpose(-1, -2) @ Rt).float()


def _noise64(t, rd, th):
    """float64 e = normalize(axis) theta with the kernel's own fp32 angle theta (zero at t <= 1)."""
    u = torch.nn.functional.normalize(rd[:, 0:3].double(), dim=-1)
    return u * th.double()[:, None] if t > 1 else torch.zeros(rd.shape[0], 3, dtype=torch.float64)


def _orientation_errors(t, st, o_k, th):
    """max |exp(o_next) - exp(e) exp(o_pred)| per row (float64) and the angle of the float64 composition."""
    R = _exp64(_noise64(t, st['rd'], th)) @ _exp64(st['o_pred'])
    return (_exp64(o_k) - R).abs().amax(dim=(-2, -1)), _angle64(R)


@pytest.mark.gpu
def test_reverse_orientation_float64():
    model = _model(28)
    rs = np.random.RandomState(5)
    report, bad = [], []
    worst_well, worst_edge = 0.0, 0.0
    for t in (_hist_ts(model)[0], _gauss_t(model), 1):
        n_rand, n_per = 400, 24
        st = _state(rs, n_rand + 16 * n_per + 6, 28)
        n = st['x'].shape[0]
        # axes: zero, subnormal and of norm 1e30 (F.normalize: a / max(|a|, 1e-12))
        st['rd'][-6:, 0:3] = torch.tensor([[0.0, 0.0, 0.0], [1e-40, -2e-40, 0.0], [1e30, -1e30, 5e29],
                                           [-3e29, 0.0, 1e30], [0.0, 0.0, 0.0], [1e-44, 0.0, 0.0]])
        st['gen'][n_rand:] = True
        _, _, _, th = _run_reverse(model, t, st)
        e = _noise64(t, st['rd'], th)
        st['o_pred'][n_rand: n_rand + 16 * n_per] = _targeted_o_pred(rs, e[n_rand:], n_per)
        if t <= 1:     # no noise: o_pred itself at exactly 0 and at fp32 pi along an axis
            st['o_pred'][n_rand] = 0.0
            st['o_pred'][n_rand + 1] = torch.tensor([PI32, 0.0, 0.0])
            st['o_pred'][n_rand + 2] = torch.from_numpy((_unit(rs, 1)[0] * np.pi).astype(np.float32))
        x, _, o, th2 = _run_reverse(model, t, st)
        assert torch.equal(th2, th)
        gen = st['gen']
        assert torch.equal(o[~gen], st['o'][~gen]), t
        og = o[gen]
        if not bool(torch.isfinite(og).all()):
            bad.append((t, 'non-finite rows', int((~torch.isfinite(og)).any(-1).sum())))
        if float(torch.linalg.norm(og.double(), dim=-1).nan_to_num(0).max()) > PI_MAX:
            bad.append((t, '|o_next| > pi'))
        err, ang = _orientation_errors(t, st, o, th)
        err, ang = err[gen].nan_to_num(float('inf')), ang[gen]
        well = (ang >= 0.1) & (ang <= np.pi - 0.1)
        worst_well = max(worst_well, float(err[well].max()))
        worst_edge = max(worst_edge, float(err[~well].max()))
        report.append((t, float(err[well].max()), float(err[ang < 1e-2].max()), float(err[ang > np.pi - 1e-2].max()),
                       int((err[ang < 1e-2] > ROT_BAR).sum()), int((err[ang > np.pi - 1e-2] > ROT_BAR).sum())))
    print('orientation: (t, worst well-conditioned, worst near 0, worst near pi, rows over the bar near 0, near pi):',
          report)
    assert not bad, bad
    bar = max(ROT_BAR, 2 * worst_well)
    assert worst_well <= ROT_BAR, report
    assert worst_edge <= bar, report


# ---- reverse step: the FG type ------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('K', [1, 17, 28, 32])
def test_reverse_type_gumbel_max(K):
    model = _model(K)
    rs = np.random.RandomState(100 + K)
    n = 1200
    near, total = 0, 0
    for t in T_STEPS:
        st = _state(rs, n, K, gen_frac=0.85)
        lg = st['logits']
        q = n // 8
        lg[:q] = 1.25                                                       # all-equal logits
        lg[q:2 * q] = torch.from_numpy(rs.uniform(-80, 80, size=(q, K)).astype(np.float32))
        lg[2 * q:3 * q, rs.randint(K)] = -1e30                              # one class at -1e30
        lg[3 * q:4 * q, K - 1] += 40.0                                      # the last lane (31 at K = 32) wins
        st['c'][4 * q:5 * q] = torch.from_numpy(rs.dirichlet(np.ones(K), size=q).astype(np.float32))   # soft c_t
        # non-generated rows with ties in c_t: argmax keeps the lowest index
        st['c'][5 * q:5 * q + 40] = 0.0
        if K > 2:
            st['c'][5 * q + 20:5 * q + 40, 1] = 0.5
            st['c'][5 * q + 20:5 * q + 40, K - 1] = 0.5
        st['gen'][5 * q:5 * q + 40] = False
        _, c, _, _ = _run_reverse(model, t, st)
        assert bool(((c == 0) | (c == 1)).all()) and bool((c.sum(-1) == 1).all()), t
        v = c.argmax(-1)
        gen = st['gen']
        assert torch.equal(v[~gen], st['c'][~gen].argmax(-1)), t            # torch.argmax: lowest index on ties
        if K > 2:
            assert bool((v[5 * q + 20:5 * q + 40] == 1).all())
        score = _oracle(model, t, st, dtype=torch.float64)[3][2][gen]
        top = score.topk(min(2, K), dim=-1).values
        margin = (top[:, 0] - top[:, 1]) if K > 1 else torch.full((int(gen.sum()),), float('inf'), dtype=torch.float64)
        clear = margin > 1e-4
        want = score.argmax(-1)
        assert torch.equal(v[gen][clear], want[clear]), (t, int((v[gen][clear] != want[clear]).sum()))
        near += int((~clear).sum())
        total += int(gen.sum())
    print(f'K={K}: {near} of {total} generated rows within 1e-4 of a tie')
    assert near <= 1e-3 * total


# ---- encoder heads --------------------------------------------------------------------------------------------------------

def _pass_through_heads(sd, H, K):
    """Head weights that pass h[:, 0:3] to eps_rot and h[:, 3:6] to eps_crd exactly ([I; -I; 0], the ReLU halves kept,
    then subtracted), the classifier's first Linear = I (pre-activations = h) and its second = h[:, 6 + k] -> logit k."""
    sd = dict(sd)
    for net, c0 in (('eps_rot_net.', 0), ('eps_crd_net.', 3)):
        w0 = torch.zeros(2 * H, H)
        w1 = torch.zeros(H, 2 * H)
        w2 = torch.zeros(3, H)
        for j in range(3):
            w0[j, c0 + j], w0[3 + j, c0 + j] = 1.0, -1.0
            w2[j, j], w2[j, 3 + j] = 1.0, -1.0
        for j in range(6):
            w1[j, j] = 1.0
        sd.update({net + '0.weight': w0, net + '0.bias': torch.zeros(2 * H), net + '2.weight': w1,
                   net + '2.bias': torch.zeros(H), net + '4.weight': w2, net + '4.bias': torch.zeros(3)})
    w = torch.zeros(K, H)
    for k in range(K):
        w[k, 6 + k] = 1.0
    sd.update({'classifier.0.weight': torch.eye(H), 'classifier.0.bias': torch.zeros(H), 'classifier.2.weight': w,
               'classifier.2.bias': torch.zeros(K)})
    return sd


def _quat_from_rotation(R):
    """eps_rot (b, c, d) with quaternion_1ijk_to_rotation_matrix(eps_rot) = R (float64): n tan(theta / 2)."""
    w = -_log64(R)          # the quaternion map is the active (transposed) convention of exp_skewsym
    th = torch.linalg.norm(w, dim=-1, keepdim=True)
    n = torch.where(th > 0, w / th.clamp_min(1e-300), torch.zeros_like(w))
    return n * torch.tan(th / 2)


def _head_rows(rs, H, K):
    """Per-row (o, h): eps_rot = h[:, 0:3] and o near 0, near pi and mixed, |eps_rot| up to 1e18, and softplus
    pre-activations at 20, 20 +- 1 ulp, 88, 89 and -100."""
    deltas = [0.0, 1e-7, 1e-6, 1e-5, 1e-4, 1e-3, 1e-2]
    o, er = [], []
    for d in deltas:
        for _ in range(6):
            a = _unit(rs, 2)
            o.append(a[0] * d); er.append(a[1] * math.tan(d / 2))                       # both near 0
            o.append(a[0] * (np.pi - d)); er.append(a[1] * 1e-9 * rs.random_sample())   # o near pi, tiny update
            o.append(a[0] * 1e-7); er.append(a[1] * (1 / max(d, 1e-18)))               # update at angle pi - 2 d
            # mixed: o random, the composition R_o U at angle d or pi - d
            oa = a[0] * rs.uniform(0.3, 3.0)
            for ang in (d, np.pi - d):
                Rt = _exp64(torch.from_numpy(_unit(rs, 1) * ang))[0]
                U = _exp64(torch.from_numpy(oa))[None].transpose(-1, -2)[0] @ Rt
                o.append(oa); er.append(_quat_from_rotation(U[None])[0].numpy())
    for mag in (1e6, 1e12, 1e18):
        a = _unit(rs, 2)
        o.append(a[0] * rs.uniform(0, 3)); er.append(a[1] * mag)
    n_edge = len(o)
    n = n_edge + 300
    o = np.concatenate([np.array(o), rs.normal(0, 1.5, size=(n - n_edge, 3))])
    er = np.concatenate([np.array(er), rs.normal(0, 2.0, size=(n - n_edge, 3))])
    h = rs.normal(0, 1.0, size=(n, H))
    h[:, 0:3] = er
    h[:, 3:6] = rs.normal(0, 3.0, size=(n, 3)) * np.exp2(rs.randint(-10, 11, size=(n, 1)))
    probes = np.array([20.0, np.nextafter(F32(20), F32(0)), np.nextafter(F32(20), F32(30)), 88.0, 89.0, -100.0],
                      dtype=np.float32)
    for j in range(min(K, len(probes))):
        h[: len(probes), 6 + j] = np.roll(probes, j)
    return torch.from_numpy(o.astype(np.float32)), torch.from_numpy(h.astype(np.float32))


def _heads64(o, h, K):
    er, ec = h[:, 0:3].double(), h[:, 3:6].double()
    U = OI.quaternion_1ijk_to_rotation_matrix(er)
    Ro = _exp64(o)
    R = Ro @ U
    eps = (Ro @ ec.unsqueeze(-1)).squeeze(-1)
    a = h[:, 6:6 + K].double()
    sp = torch.where(a > 20, a, torch.log1p(torch.exp(a)))
    return R, eps, sp - math.log(2.0)


@pytest.mark.gpu
@pytest.mark.parametrize('H,K', [(256, 28), (128, 32), (128, 6)])
def test_heads_float64(H, K):
    rs = np.random.RandomState(H + K)
    model = IPATransformerB200(synthetic.ipa_config(H, 0, K))
    sd = synthetic.seeded_state_dict(model, seed=1, skip_prefixes=())
    model.load_state_dict(_pass_through_heads(sd, H, K), strict=True)
    model = model.to(DEV)
    o, h = _head_rows(rs, H, K)
    n = o.shape[0]
    x = torch.from_numpy(rs.normal(0, 4, size=(n, 3)).astype(np.float32))
    b = torch.from_numpy(np.repeat(np.arange(3), [n // 3, n // 3, n - 2 * (n // 3)]))
    lig = torch.ones(n, dtype=torch.bool)
    gen = torch.from_numpy(rs.random_sample(n) < 0.9)
    gen[:-300] = True                                          # every crafted edge row is generated
    eps_pos, h_out, o_next, R_next, c = (t.cpu() for t in model(*[t.to(DEV) for t in (x, o, h, b, lig, gen)]))
    assert torch.equal(h_out, h)
    R64, eps64, c64 = _heads64(o, h, K)
    errR = (R_next.double() - R64).abs().amax(dim=(-2, -1))
    ang = _angle64(R64)
    well = (ang >= 0.1) & (ang <= np.pi - 0.1)
    bar = max(ROT_BAR, 2 * float(errR[well].max()))
    print(f'heads H={H}: R_next worst {float(errR[well].max()):.2e} well-conditioned, {float(errR[~well].max()):.2e} '
          f'near 0 / pi')
    assert float(errR[well].max()) <= ROT_BAR and float(errR.max()) <= bar
    g = gen
    errO = (_exp64(o_next[g]) - R64[g]).abs().amax(dim=(-2, -1))
    print(f'heads H={H}: exp(o_next) worst {float(errO[well[g]].max()):.2e} well-conditioned, '
          f'{float(errO[~well[g]].max()):.2e} near 0 / pi')
    assert bool(torch.isfinite(o_next).all())
    assert float(torch.linalg.norm(o_next[g].double(), dim=-1).max()) <= PI_MAX
    assert float(errO.max()) <= bar, (float(errO.max()), int(errO.argmax()))
    assert torch.equal(o_next[~g], o[~g]) and not eps_pos[~g].any()
    scale = h[:, 3:6].double().abs().amax(-1)
    assert bool(((eps_pos[g].double() - eps64[g]).abs().amax(-1) <= ROT_BAR * scale[g]).all())
    assert bool(((c.double() - c64).abs() <= 2e-6 * c64.abs().clamp_min(1.0)).all()), (c.double() - c64).abs().max()


# ---- encoder body ---------------------------------------------------------------------------------------------------------

# (H, k, nodes per graph, FG nodes per graph, num_sublayers, num_blocks, log2 of the h scale)
BODY_CASES = [
    (128, 32, [1, 2, 32, 33, 34, 200], [1, 1, 4, 5, 6, 20], 1, 1, 0),     # 1, 2, k, k + 1, k + 2 and 200 nodes
    (256, 32, [1, 2, 32, 33, 34], [1, 2, 32, 0, 10], 1, 1, 0),
    (128, 1, [1, 2, 3, 57], [0, 1, 3, 10], 1, 3, 0),                       # N = 63
    (256, 8, [8, 9, 10, 1, 37], [2, 9, 0, 1, 5], 4, 1, 0),                 # N = 65
    (128, 31, [31, 32, 33, 33], [31, 0, 5, 4], 1, 1, 20),                  # N = 129
    (256, 31, [65], [65], 0, 1, -20),                                      # all-ligand
    (128, 8, [63], [0], 1, 3, -20),                                        # all-protein
    (256, 32, [200, 7], [30, 7], 1, 1, 20),
    (128, 1, [1], [1], 4, 1, 0),                                           # N = 1
    (256, 1, [2, 1], [1, 0], 1, 3, 0),
]


def _body_inputs(case, seed):
    H, k, nodes, lig, nsub, nblk, c = case
    x, o, h, b, l, gen = synthetic.make_ipa_inputs(H, nodes, lig, seed, 'partial' if seed % 2 else 'denovo')
    return x, o, h * float(2.0 ** c), b, l, gen


def _body_model(case, K=12):
    H, k, nodes, lig, nsub, nblk, c = case
    model = IPATransformerB200(synthetic.ipa_config(H, nsub, K, num_blocks=nblk, k=k))
    sd = synthetic.seeded_state_dict(model, seed=7, skip_prefixes=())
    model.load_state_dict(sd, strict=True)
    return model.to(DEV), sd


@pytest.mark.gpu
@pytest.mark.parametrize('case', BODY_CASES, ids=[f'H{c[0]}_k{c[1]}_N{sum(c[2])}_s{c[4]}_b{c[5]}_c{c[6]}' for c in BODY_CASES])
def test_encoder_body_float64(case):
    """Per output and per row: |kernel - float64| <= 4 x the fp32 oracle's |oracle - float64| + one fp32 ulp of the row's
    largest value.  The fp32 oracle's row error is floored at its median relative error over the rows of that output
    times the row's scale, so a row where fp32 torch happens to land on the float64 value does not set a zero bar."""
    H, k, nodes, lig, nsub, nblk, c = case
    model, sd = _body_model(case)
    inp = _body_inputs(case, seed=sum(nodes) + k)
    x, o, h, b, l, gen = inp
    got = [t.cpu() for t in model(*[t.to(DEV) for t in inp])]
    nbr = G.neighbor_table(x, G.graph_ptr_from_batch(b), k=k, r_max=None)
    f32 = OI.ipatransformer_forward(sd, *inp, k=k, num_blocks=nblk, nbr=nbr)
    sd64 = {kk: (v.double() if v.is_floating_point() else v) for kk, v in sd.items()}
    f64 = OI.ipatransformer_forward(sd64, x.double(), o.double(), h.double(), b, l, gen, k=k, num_blocks=nblk, nbr=nbr)
    for j, nm in ((0, 'eps_pos'), (1, 'h'), (3, 'R_next'), (4, 'logits')):
        ref = f64[j].reshape(len(x), -1)
        ek = (got[j].double().reshape(len(x), -1) - ref).abs().amax(-1)
        eo = (f32[j].double().reshape(len(x), -1) - ref).abs().amax(-1)
        scale = ref.abs().amax(-1)
        rel = eo / scale.clamp_min(1e-300)
        floor = float(rel[scale > 0].median()) * scale if bool((scale > 0).any()) else torch.zeros_like(scale)
        ulp = torch.from_numpy(np.spacing(scale.numpy().astype(np.float32)).astype(np.float64))
        bar = 4 * torch.maximum(eo, floor) + ulp
        bad = ek > bar
        assert not bool(bad.any()), (nm, int(bad.sum()), float((ek / bar).max()), int((ek / bar).argmax()))
    assert torch.equal(got[2][~gen], o[~gen])
    # a graph's rows do not depend on the other graphs of the batch
    for g in range(len(nodes)):
        m = b == g
        sub = [t[m] for t in inp]
        sub[3] = torch.zeros(int(m.sum()), dtype=torch.long)
        alone = [t.cpu() for t in model(*[t.to(DEV) for t in sub])]
        for a, full in zip(alone, got):
            assert torch.equal(a, full[m]), g


# ---- argument checks (no device needed) -----------------------------------------------------------------------------------

def _fake_ws():
    return 1 << 20, 1 << 40          # aligned non-NULL pointer value, never dereferenced: the checks fail first


@pytest.mark.parametrize('k', [0, -1, 33, 64])
def test_ipa_forward_refuses_k_outside_1_32(k):
    L = _lib.lib()
    ws, nb = _fake_ws()
    rc = L.cbg_ipa_forward_f32(None, 128, 1, 1, 8, None, None, None, None, 1, 4, None, None, 4, k, None, None, None,
                               None, None, ws, nb, None)
    assert rc != 0 and f'k={k}' in L.cbg_last_error().decode()


def test_fg_workspace_bytes_cover_the_carve():
    """cbg_fg_workspace_bytes = the IPATransformer scratch + the five encoder row arrays (eps_pos, o_pred, h, R_next,
    logits), each rounded up to 256 bytes: the size fg_rows carves for cbg_fg_step_f32 and cbg_fg_eval_loss_f32."""
    L = _lib.lib()
    al = lambda b: (b + 255) // 256 * 256
    for n in (1, 2, 5, 63, 64, 65, 1000, 4097, 100_003, 1 << 20):
        for H in (128, 256):
            for K in (1, 28, 32):
                want = L.cbg_ipa_workspace_bytes(n, H) + 2 * al(n * 3 * 4) + al(n * H * 4) + al(n * 9 * 4) + al(n * K * 4)
                got = L.cbg_fg_workspace_bytes(n, H, K)
                assert got == want and got % 256 == 0, (n, H, K, got, want)


def test_fg_reverse_refusals():
    L = _lib.lib()
    nil = [None] * 12
    coef = _lib.FgCoef(t=3)
    good = dict(num_classes=28, n_lig=4, lig_node=1 << 20, gen_lig=1 << 20, angle_x=1 << 20, angle_cdf=1 << 20, n_bins=16)

    def rc(plan=None, coef=coef, ptrs=None):
        p = C.byref(_lib.FgPlan(**plan)) if plan is not None else None
        return L.cbg_fg_reverse_f32(p, coef, *(ptrs if ptrs is not None else [1 << 20] * 12), None, None)

    assert rc(None) != 0 and 'plan is NULL' in L.cbg_last_error().decode()
    for over, msg in (({'num_classes': 0}, 'num_classes=0'), ({'num_classes': 33}, 'num_classes=33'),
                      ({'n_bins': 1}, 'n_bins=1'), ({'n_lig': -1}, 'n_lig=-1'), ({'lig_node': None}, 'lig_node'),
                      ({'angle_cdf': None}, 'angle_cdf')):
        assert rc(dict(good, **over)) != 0 and msg in L.cbg_last_error().decode(), over
    assert rc(good, coef=_lib.FgCoef(t=-1)) != 0 and 't=-1' in L.cbg_last_error().decode()
    assert rc(good, ptrs=[1 << 20] * 11 + [None]) != 0 and 'NULL row' in L.cbg_last_error().decode()
    assert rc(dict(good, n_lig=0), ptrs=nil) == 0              # nothing to do: no launch, no pointer read
