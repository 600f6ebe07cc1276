"""D3FG sampler (`difffg`, DESIGN.md section 16).

CPU: the state-dict contract and angular buffers against the live-reference fixtures (tests/golden/make_golden_f8.py),
the oracle restatement (tests/fg_sample_oracle.py) against the reference trajectory, constructor refusals, the 28-class
IPA pack.  GPU: csrc/fg.cu through D3FGB200.sample against the golden trajectory and the oracle, step invariants and
the angle sampler's distribution."""
import json
import os

import numpy as np
import pytest
import torch

from cbgbench_b200 import _lib, synthetic
from cbgbench_b200.difffg import D3FGB200
from cbgbench_b200.ipatransformer import IPATransformerB200, pack_ipa_blob
from cbgbench_b200.targetdiff import get_model
from helpers import GOLDEN as GOLDEN_DIR, assert_close

import fg_sample_oracle as OF

torch.set_grad_enabled(False)
HERE = os.path.dirname(os.path.abspath(__file__))


def _maker():
    import importlib.util
    spec = importlib.util.spec_from_file_location('make_golden_f8', os.path.join(GOLDEN_DIR, 'make_golden_f8.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


MK = _maker()
CASE = MK.CASE


@pytest.fixture(scope='module')
def golden_model():
    model = D3FGB200(synthetic.difffg_config(num_steps=CASE['T'], num_layers=CASE['num_layers'], hidden=CASE['hidden']))
    sd, batch, draws = MK.build_inputs(model)
    model.load_state_dict(sd, strict=True)
    return model.eval(), sd, batch, draws


def _gold():
    return np.load(os.path.join(GOLDEN_DIR, 'fg_trajectory.npz'))


def test_state_dict_and_angular_buffers_match_reference(golden_model):
    model = golden_model[0]
    with open(os.path.join(GOLDEN_DIR, 'fg_state_keys.json')) as f:
        want = json.load(f)
    got = {k: list(v.shape) for k, v in model.state_dict().items()}
    assert list(got) == list(want) and got == want
    fresh = D3FGB200(synthetic.difffg_config(num_steps=CASE['T'], num_layers=CASE['num_layers'], hidden=CASE['hidden']))
    g = _gold()
    for r in MK.Y_ROWS:
        assert torch.equal(fresh.rot_scheduler.angular_distrib_inv.Y[r], torch.from_numpy(g[f'Y{r}']))
    for name in ('difffg', 'difffg_v2'):
        cfg = synthetic.difffg_config(num_steps=4, num_layers=1)
        cfg['type'] = name
        assert isinstance(get_model(cfg), D3FGB200)


def test_oracle_matches_reference_trajectory(golden_model):
    _, sd, batch, draws = golden_model
    want = OF.sample(sd, batch, CASE['T'], *draws)
    g = _gold()
    for t in range(-1, CASE['T']):
        for j, nm in enumerate(('xc', 'c', 'o')):
            ref = torch.from_numpy(g[f't{t}/{nm}'])
            assert float((want[t][j] - ref).abs().max() / (ref.abs().max() + 1e-12)) < 1e-5, (t, nm)


def test_constructor_refusals_and_cpu_model():
    def cfg(**over):
        c = synthetic.difffg_config(num_steps=4, num_layers=1)
        for k, v in over.items():
            c['embedder'][k] = v
        return c
    with pytest.raises(NotImplementedError):
        D3FGB200(cfg(time={'type': 'sin'}))
    with pytest.raises(NotImplementedError):
        D3FGB200(cfg(vec={'type': 'x', 'vec_emb_dim': 8}))
    with pytest.raises(NotImplementedError):
        D3FGB200(cfg(residue={'type': 'linear'}))
    with pytest.raises(NotImplementedError):
        D3FGB200(synthetic.difffg_config(num_steps=4, num_layers=1, num_fgtype=40))    # 40 > the IPA class cap
    m = D3FGB200(synthetic.difffg_config(num_steps=4, num_layers=1))
    with pytest.raises(NotImplementedError):
        m.eval()(synthetic.make_fg_batch([10], [2]))
    with pytest.raises(NotImplementedError):
        m.train()(synthetic.make_fg_batch([10], [2]))
    with pytest.raises(RuntimeError):
        m.eval().sample(synthetic.make_fg_batch([10], [2]))


def test_ipa_pack_28_classes():
    H = 256
    model = IPATransformerB200(synthetic.ipa_config(H, 1, 28))
    sd = synthetic.seeded_state_dict(model, seed=1, skip_prefixes=())
    blob = pack_ipa_blob(sd, H, 1, 1, 28)
    L = _lib.lib()
    g0 = _lib.blob_layout()['global_floats']
    names = {L.cbg_ipa_head_field_name(f).decode(): f for f in range(L.cbg_ipa_head_fields())}
    off, size = L.cbg_ipa_head_field_offset(H, names['CLS_W1']), L.cbg_ipa_head_field_size(H, names['CLS_W1'])
    assert size == 32 * H
    w = blob[g0 + off: g0 + off + size].view(32, H)
    assert torch.equal(w[:28], sd['classifier.2.weight']) and not w[28:].any()
    off = L.cbg_ipa_head_field_offset(H, names['CLS_B1'])
    assert torch.equal(blob[g0 + off: g0 + off + 28], sd['classifier.2.bias'])


# ---- GPU -----------------------------------------------------------------------------------------------------------------

def _on_gpu(golden_model):
    model, sd, batch, draws = golden_model
    return model.to('cuda:0'), sd, batch, draws


def _rot(o):
    return OF.so3vec_to_rotation(o.double())


def _rot_agree(a, b, tol):
    """Fraction of rows whose rotation matrices exp(a), exp(b) agree to ``tol`` element-wise."""
    return float(((_rot(a) - _rot(b)).abs().amax(dim=(-2, -1)) < tol).double().mean()) if a.numel() else 1.0


def _near_pi(o, tol=1e-2):
    """Rows whose rotation angle is within ``tol`` of pi: there the reference's fp32 log map (so3.py:10-22), which the
    golden trajectory and the oracle use, is ill-conditioned, so its rounding errors grow by orders of magnitude and
    carry into later steps (the kernels' log map is exact there: tests/test_fg_kernels.py)."""
    return torch.linalg.norm(o.double(), dim=-1) > np.pi - tol


@pytest.mark.gpu
def test_cuda_golden_trajectory(golden_model):
    model, sd, batch, draws = _on_gpu(golden_model)
    T = CASE['T']
    traj = model.sample(batch, *draws)
    g = _gold()
    ok = torch.ones(sum(CASE['n_fg']), dtype=torch.bool)     # FGs that have not passed near pi so far
    for t in range(T - 1, -2, -1):
        xc, c, o, _ = (a.cpu() if torch.is_tensor(a) else a for a in traj[t])
        ref = torch.from_numpy(g[f't{t}/xc'])
        # 1e-4 relative to the state's magnitude: the encoder's fp32 sums (1e-4 parity, tests/test_ipa.py) reach the
        # positions through b / sqrt(1 - abar) at every step and accumulate over the trajectory
        assert_close(xc, ref, rtol=1e-4, atol=1e-4 * float(ref.abs().max()), what=f'xc at {t}')
        assert torch.equal(c, torch.from_numpy(g[f't{t}/c'])), f'FG types at {t}'
        og = torch.from_numpy(g[f't{t}/o'])
        ok &= ~_near_pi(og)
        # rotations compose over the trajectory: the encoder's 1e-4 parity in the rotation head (tests/test_ipa.py)
        # accumulates step after step, and the log map that stores o (and o_pred) is ill-conditioned near pi
        assert _rot_agree(o[ok], og[ok], 1e-2) > 0.9, f'rotation at {t}'
        assert ok.float().mean() > 0.8
    assert model.last_launches > 0


@pytest.mark.gpu
def test_cuda_matches_oracle_shipped_depth():
    rs = np.random.RandomState(5)
    n_res = rs.randint(40, 151, size=16).tolist()
    n_fg = rs.randint(2, 21, size=16).tolist()
    T, steps = 20, 10
    model = D3FGB200(synthetic.difffg_config(num_steps=T, num_layers=9))
    sd = synthetic.seeded_state_dict(model, seed=4)
    model.load_state_dict(sd, strict=True)
    model = model.eval().to('cuda:0')
    batch = synthetic.make_fg_batch(n_res, n_fg, seed=21, partial_graphs=(3, 7))
    draws = synthetic.make_fg_draws(T, sum(n_fg), seed=22)
    got = model.sample(batch, *draws, num_steps=steps)
    want = OF.sample(sd, batch, T, *draws, num_steps=steps)
    same = torch.ones(sum(n_fg), dtype=torch.bool)       # FGs whose sampled types have agreed so far
    for t in range(T - 2, T - 2 - steps, -1):
        xc, c, o, _ = (a.cpu() if torch.is_tensor(a) else a for a in got[t])
        w = want[t][0]
        assert_close(xc[same], w[same], rtol=1e-3, atol=2e-3 * float(w.abs().max()), what=f'xc at {t}')
        same &= ~_near_pi(want[t][2])
        assert _rot_agree(o[same], want[t][2][same], 5e-2) > 0.9, f'rotation at {t}'
        same &= c.argmax(-1) == want[t][1].argmax(-1)
        # random weights leave near-ties in the type posterior: a few FGs take another type and leave the comparison
        assert same.float().mean() > 0.9, f'FG types at {t}: {same.float().mean()}'


@pytest.mark.gpu
def test_cuda_step_invariants(golden_model):
    model, sd, batch, draws = _on_gpu(golden_model)
    T = CASE['T']
    a = model.sample(batch, *draws)
    b = model.sample(batch, *draws)
    for t in a:
        for x, y in zip(a[t][:3], b[t][:3]):
            assert torch.equal(x.cpu(), y.cpu())                                  # repeat runs are bit-identical
    gen = batch['ligand_gen_flag']
    for t in range(-1, T - 1):
        for j in range(3):
            assert torch.equal(a[t][j].cpu()[~gen], a[T - 1][j][~gen])          # non-generated FGs never move
    # no rotation noise at t <= 1: with the axis draws of those steps replaced, t = 1 and 0 do not change
    pos, rot, typ = draws
    rot2 = rot.clone()
    rot2[:2] = torch.randn_like(rot2[:2])
    c2 = model.sample(batch, pos, rot2, typ)
    for t in (0, -1):
        assert torch.equal(c2[t][2].cpu(), a[t][2].cpu())
    # a graph alone == the same graph inside the batch
    g = 1
    ml, mr = batch['ligand_type_fg_batch'] == g, batch['protein_type_fg_batch'] == g
    sub = {k: (v[ml] if k.startswith('ligand_') else v[mr]) for k, v in batch.items() if k != 'protein_num_chains'}
    sub['protein_num_chains'] = batch['protein_num_chains'][g:g + 1]
    sub['ligand_type_fg_batch'] = torch.zeros(int(ml.sum()), dtype=torch.long)
    sub['protein_type_fg_batch'] = torch.zeros(int(mr.sum()), dtype=torch.long)
    alone = model.sample(sub, pos[:, ml], rot[:, ml], typ[:, ml])
    for t in range(-1, T - 1):
        # to rounding, not bit for bit: the once-per-batch protein MLP runs through cuBLAS, whose kernel choice depends
        # on the number of residue rows
        assert torch.equal(alone[t][1].cpu(), a[t][1].cpu()[ml])
        w = a[t][0].cpu()[ml]
        assert_close(alone[t][0].cpu(), w, rtol=1e-3, atol=1e-3 * float(w.abs().max()), what=f'graph alone, xc at {t}')
        ow = a[t][2].cpu()[ml]
        far = ~_near_pi(ow)
        assert _rot_agree(alone[t][2].cpu()[far], ow[far], 1e-2) > 0.8


@pytest.mark.gpu
def test_cuda_default_draws_equal_injected_draws(golden_model):
    model, sd, batch, draws = _on_gpu(golden_model)
    T, n, K = CASE['T'], sum(CASE['n_fg']), 28
    dev = torch.device('cuda:0')
    torch.manual_seed(123)
    a = model.sample(batch)
    torch.manual_seed(123)
    pos, rot, typ = [torch.empty(T, n, d) for d in (3, 6, K)]
    for t in reversed(range(T)):
        pos[t] = torch.randn(n, 3, device=dev).cpu()
        rot[t, :, 0:3] = torch.randn(n, 3, device=dev).cpu()
        rot[t, :, 3] = torch.rand(n, device=dev).cpu()
        rot[t, :, 4] = torch.rand(n, device=dev).cpu()
        rot[t, :, 5] = torch.randn(n, device=dev).cpu()
        typ[t] = torch.rand(n, K, device=dev).cpu()
    b = model.sample(batch, pos, rot, typ)
    for t in a:
        for x, y in zip(a[t][:3], b[t][:3]):
            assert torch.equal(x.cpu(), y.cpu())


@pytest.mark.gpu
def test_cuda_angle_sampler_distribution():
    """Rotation angles drawn by the kernel (read back as the angle of R' R_pred^T) follow the histogram CDF of
    angular_distrib_inv.Y[t] where the histogram branch is used and |N(2 sigma, sigma)| where the Gaussian one is
    (Kolmogorov-Smirnov, 10^5 samples per t), and equal the angles of the definition draw for draw."""
    from scipy import stats
    T = 20
    model = D3FGB200(synthetic.difffg_config(num_steps=T, num_layers=1))
    model.load_state_dict(synthetic.seeded_state_dict(model, seed=2), strict=True)
    model = model.eval().to('cuda:0')
    batch = synthetic.make_fg_batch([8] * 1000, [100] * 1000, seed=4)
    n = 100000
    inv = model.rot_scheduler.angular_distrib_inv
    flags, X, Y, std = inv.approx_flag.cpu(), inv.X.cpu().double(), inv.Y.cpu().double(), inv.stddevs.cpu().double()
    ts = [t for t in range(2, T) if flags[t]][-1:] + [t for t in range(2, T) if not flags[t]][::6]
    assert any(flags[t] for t in ts) and any(not flags[t] for t in ts)
    rs = np.random.RandomState(3)
    for t in ts:
        pos, rot, typ = synthetic.make_fg_draws(T, n, seed=int(rs.randint(1 << 30)))
        got, well = _angles_kernel(model, batch, t, pos, rot, typ)
        ref = _angles_reference(inv, t, rot[t])
        assert (np.abs(got - ref)[well] < 2e-3).mean() > 0.99, t
        if flags[t]:
            s = float(std[t])
            cdf = lambda x: stats.norm.cdf((x - 2 * s) / s) - stats.norm.cdf((-x - 2 * s) / s)
        else:
            w = torch.cat([torch.zeros(1, dtype=torch.float64), Y[t, :-1].cumsum(0)])
            edges, w = X[t].numpy(), (w / w[-1]).numpy()
            cdf = lambda x: np.interp(x, edges, w)
        assert stats.kstest(got, cdf).pvalue > 1e-4, t


def _angles_reference(inv, t, rd):
    """theta of so3.py:111-138 for the draws rd [n,6] (CPU, definition of the bin draw)."""
    import math
    from cbgbench_b200.difffg import multinomial_bin
    X, Y, std = inv.X.cpu(), inv.Y.cpu(), inv.stddevs.cpu()
    n = rd.shape[0]
    tt = torch.full((n,), t, dtype=torch.long)
    b = multinomial_bin(Y[tt][:, :-1], rd[:, 3])
    hist = X[tt, b] + rd[:, 4] * (X[tt, b + 1] - X[tt, b])
    gauss = (std[tt] * 2 + rd[:, 5] * std[tt]).abs() % math.pi
    return torch.where(inv.approx_flag.cpu()[tt], gauss, hist).numpy()


def _angles_kernel(model, batch, t, pos, rot, typ):
    """Angle of R_next R_pred^T per FG after the step at t, read from two runs that differ only in the rotation noise."""
    T = model.num_diffusion_timesteps
    a = model.sample(batch, pos, rot, typ, num_steps=T - t)
    rot0 = rot.clone()
    rot0[t, :, 0:3] = 0.0            # zero axis: normalize(0) = 0, so e = 0 and R' = R_pred
    b = model.sample(batch, pos, rot0, typ, num_steps=T - t)
    oa, ob = a[t - 1][2].cpu(), b[t - 1][2].cpu()
    E = _rot(oa) @ _rot(ob).transpose(-1, -2)
    cos = ((E.diagonal(dim1=-2, dim2=-1).sum(-1) - 1) / 2).clamp(-1, 1)
    return torch.acos(cos).numpy(), (~_near_pi(oa, 0.05) & ~_near_pi(ob, 0.05)).numpy()
