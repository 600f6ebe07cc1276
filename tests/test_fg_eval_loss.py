"""D3FG validation losses: eval-mode D3FGB200.forward / eval_losses (csrc/fg_eval.cu, DESIGN.md section 17) against the
reference's eval-mode D3FG.forward of ``difffg`` and ``difffg_v2`` (fixtures of tests/golden/make_golden_f9.py) and the
CPU restatement tests/fg_eval_loss_oracle.py."""
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

import fg_eval_loss_oracle as OE
from eval_loss_oracle import auroc as ref_auroc
from helpers import GOLDEN as GOLDEN_DIR, assert_close, loss_close
from cbgbench_b200 import _lib, synthetic
from cbgbench_b200.difffg import D3FGB200
from cbgbench_b200.targetdiff import eval_t_values, get_model

torch.set_grad_enabled(False)


def _maker():
    spec = importlib.util.spec_from_file_location('make_golden_f9', os.path.join(GOLDEN_DIR, 'make_golden_f9.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


MK = _maker()
CASE_MODELS = [(c, m) for c in MK.CASES for m in MK.MODELS]
IDS = [f'{c}-{m}' for c, m in CASE_MODELS]
LOSS_KEYS = ('pos', 'rot', 'fg')
# The t = 0 type loss is the decoder NLL -log p with p within a few ulps of 1, which fp32 holds only to about one ulp of
# 1 (6e-8): the losses get an absolute 5e-7 beside the relative 1e-4 (as the TargetDiff validation loss, section 13).
LOSS_RTOL, LOSS_ATOL = 1e-4, 5e-7
DEV = 'cuda:0'


def _gold():
    return np.load(os.path.join(GOLDEN_DIR, 'fg_eval_loss.npz'))


def _model(name, model_name, device=None, num_layers=MK.NUM_LAYERS, hidden=MK.HIDDEN, T=None, interval=None):
    T = MK.CASES[name][0] if T is None else T
    cfg = synthetic.difffg_config(num_steps=T, num_layers=num_layers, hidden=hidden)
    cfg['type'] = model_name
    cfg['eval_interval'] = MK.CASES[name][1] if interval is None else interval
    model = get_model(cfg)
    sd = synthetic.seeded_state_dict(model, seed=MK.WEIGHT_SEED)
    model.load_state_dict(sd, strict=True)
    model.eval()
    return (model.to(device) if device else model), sd


def _inputs(name):
    batch = MK.case_batch(name)
    t_values = MK.case_t_values(name)
    return batch, t_values, MK.case_draws(name, len(t_values))


# ---- CPU ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('case,model_name', CASE_MODELS, ids=IDS)
def test_oracle_matches_fixtures(case, model_name):
    g = _gold()
    _, sd = _model(case, model_name)
    batch, t_values, draws = _inputs(case)
    form = 'score' if model_name == 'difffg' else 'denoise'
    loss, res, per_t, _ = OE.eval_losses(sd, batch, t_values, *draws, form=form)
    key = f'{case}/{model_name}'
    for k in LOSS_KEYS:
        want = float(g[f'{key}/{k}'])
        assert abs(float(loss[k]) - want) <= 1e-6 * abs(want), (k, float(loss[k]), want)
    assert np.allclose(per_t.numpy(), g[f'{key}/per_t'], rtol=1e-6, atol=0)
    for k in res[0]:
        if f'{key}/{k}' in g.files:
            want = torch.from_numpy(g[f'{key}/{k}'])
            got = torch.stack([r[k] for r in res])
            if want.dtype == torch.int64:
                assert torch.equal(got, want), k
            else:
                assert float((got - want).abs().max()) <= 1e-6 * float(want.abs().max()), k


def test_eval_coef_matches_torch_expressions():
    model, _ = _model('ragged', 'difffg')
    ps, rs, ts = model.pos_scheduler, model.rot_scheduler, model.type_scheduler
    fwd = rs.angular_distrib_fwd
    f32 = lambda v: np.float32(v).tobytes()
    for t in (0, 1, 7, 19):
        c = model.eval_coef(t)
        a, ar = ps.alphas_cumprod[t].float(), rs.alphas_cumprod[t].float()
        assert c.t == t and c.t_is_zero == (t == 0)
        assert f32(c.pos_sqrt_alphas_cumprod) == f32(float(a.sqrt()))
        assert f32(c.pos_sqrt_one_minus_alphas_cumprod) == f32(float((1. - a).sqrt()))
        assert f32(c.rot_sqrt_alphas_cumprod) == f32(float(torch.sqrt(ar)))
        assert f32(c.rot_std) == f32(float(fwd.stddevs[t])) and c.rot_gaussian == int(fwd.approx_flag[t])
        assert f32(c.rot_std) == f32(float(torch.sqrt(1 - rs.alphas_cumprod[t])))
        tm1 = max(t - 1, 0)
        for field, name, idx in (('log_alphas_cumprod', 'log_alphas_cumprod_v', t),
                                 ('log_one_minus_alphas_cumprod', 'log_one_minus_alphas_cumprod_v', t),
                                 ('log_alphas_cumprod_prev', 'log_alphas_cumprod_v', tm1),
                                 ('log_one_minus_alphas_cumprod_prev', 'log_one_minus_alphas_cumprod_v', tm1),
                                 ('log_alpha', 'log_alphas_v', t), ('log_one_minus_alpha', 'log_one_minus_alphas_v', t)):
            assert f32(getattr(c, field)) == f32(float(getattr(ts, name)[idx])), (t, field)


def test_forward_angle_prefix_sums():
    model, _ = _model('ragged', 'difffg')
    rs = model.rot_scheduler
    fwd = rs.fwd_cdf('cpu')
    assert fwd.dtype == torch.float64 and fwd.shape == (20, rs.angular_distrib_fwd.num_bins - 1)
    assert torch.equal(fwd, rs.angular_distrib_fwd.Y[:, :-1].double().cumsum(-1))
    inv = rs.bin_cdf('cpu')
    assert torch.equal(inv, rs.angular_distrib_inv.Y[:, :-1].double().cumsum(-1))
    assert not torch.equal(fwd, inv)
    assert rs.fwd_cdf('cpu') is fwd and rs.bin_cdf('cpu') is inv          # cached, separately
    # the bin search over the prefix sums is the definition of the multinomial draw
    from cbgbench_b200.difffg import multinomial_bin
    u = torch.rand(500, generator=torch.Generator().manual_seed(0))
    for t in (1, 10, 19):
        b = multinomial_bin(rs.angular_distrib_fwd.Y[t, :-1].expand(500, -1), u)
        assert torch.equal(b, torch.searchsorted(fwd[t], (u.double() * fwd[t, -1]).contiguous(), right=True))


def test_refusals():
    model, _ = _model('ragged', 'difffg')
    batch, t_values, draws = _inputs('ragged')
    with pytest.raises(NotImplementedError):
        model.train()(batch)
    model.eval()
    with pytest.raises(NotImplementedError):
        model(batch)                              # the batch has no ligand_mask_heavyatom: refused before it is read
    with pytest.raises(NotImplementedError):
        model(None)
    for bad in ([20], [-1], []):
        with pytest.raises(ValueError):
            model.eval_losses(batch, bad)
    with pytest.raises(ValueError):
        model.eval_losses(batch, [0], pos_noise=draws[0][:1])
    trailing = synthetic.make_fg_batch([20, 30], [4, 0], seed=5)    # the last graph has residues but no FG
    with pytest.raises(ValueError, match='no functional group'):
        model.eval_losses(trailing, [0, 5])
    v2 = _model('ragged', 'difffg_v2')[0]
    assert isinstance(v2, D3FGB200) and v2.pos_loss_form == _lib.FG_LOSS_DENOISE
    assert type(model).pos_loss_form == _lib.FG_LOSS_SCORE


# ---- GPU ------------------------------------------------------------------------------------------------------------------

def _run(model, batch, t_values, draws, **kw):
    return model.eval_losses(batch, t_values, *draws, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize('case,model_name', CASE_MODELS, ids=IDS)
def test_cuda_matches_fixtures(case, model_name):
    g = _gold()
    model, _ = _model(case, model_name, DEV)
    batch, t_values, draws = _inputs(case)
    loss, res = model(batch, *draws)
    key = f'{case}/{model_name}'
    for k in LOSS_KEYS:
        assert loss[k].dtype == torch.float32 and loss[k].dim() == 0 and loss[k].device.type == 'cpu'
        assert loss_close(float(loss[k]), float(g[f'{key}/{k}']), LOSS_RTOL, LOSS_ATOL, nan_equal=True), \
            (k, float(loss[k]), float(g[f'{key}/{k}']))
    pos_keys = ['eps_0', 'eps_pred', 'score_0', 'score_pred'] if model_name == 'difffg' else ['x0', 'xt', 'x_pred']
    assert len(res) == len(t_values)
    gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag'])
    for r, rr in enumerate(res):
        assert list(rr) == pos_keys + ['mask_gen', 'v0', 'vt', 'c_pred', 'R0', 'R_pred']
        for k, v in rr.items():
            assert v.device == torch.device(DEV), k
            assert v.dtype == (torch.bool if k == 'mask_gen' else torch.int64 if k in ('v0', 'vt') else torch.float32), k
        assert torch.equal(rr['mask_gen'].cpu(), gen)
        assert torch.equal(rr['v0'].cpu(), batch['ligand_type_fg'])
        assert torch.equal(rr['vt'].cpu(), torch.from_numpy(g[f'{key}/vt'][r])), f'vt at t={t_values[r]}'
    stack = lambda k: torch.stack([rr[k] for rr in res]).cpu()
    # the encoder's outputs carry its 1e-4 parity (tests/test_ipa.py); what the kernels compute from the draws alone is
    # held to fp32 rounding
    for k, rtol, atol_scale in (('eps_pred', 1e-4, 1e-4), ('score_pred', 1e-4, 1e-4), ('x_pred', 1e-4, 1e-4),
                                ('c_pred', 1e-4, 1e-5), ('R_pred', 1e-4, 1e-4), ('score_0', 1e-6, 1e-7),
                                ('xt', 1e-6, 1e-7)):
        if k in rr:
            want = torch.from_numpy(g[f'{key}/{k}'])
            assert_close(stack(k), want, rtol=rtol, atol=atol_scale * max(float(want.abs().max()), 1.0), what=k)
    if 'eps_0' in rr:
        assert torch.equal(stack('eps_0'), draws[0])
    assert_close(res[0]['R0'].cpu(), torch.from_numpy(g[f'{key}/R0']), rtol=1e-6, atol=1e-6, what='R0')
    if not math.isnan(float(g[f'{key}/auroc'])):
        assert abs(ref_auroc(res) - float(g[f'{key}/auroc'])) < 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize('model_name', ['difffg', 'difffg_v2'])
def test_cuda_matches_oracle_shipped_depth(model_name):
    """16 ragged pockets, 9 layers, H = 256, partial generation, against the oracle.  The encoder reads a FG's o_t only
    in its own row's heads, and the oracle's o_t is the reference's fp32 log map, which is inexact within ~0.05 of pi:
    the rows and per-graph position / rotation terms of FGs noised that close to pi are left out (the kernel's log map is
    checked there against float64 in test_cuda_noised_orientation_matches_float64)."""
    rs = np.random.RandomState(6)
    n_res = rs.randint(40, 151, size=16).tolist()
    n_fg = rs.randint(2, 21, size=16).tolist()
    T = 20
    model, sd = _model('ragged', model_name, DEV, num_layers=9, T=T, interval=10)
    batch = synthetic.make_fg_batch(n_res, n_fg, seed=23, partial_graphs=(2, 9))
    t_values = eval_t_values(T, 10)
    draws = synthetic.make_fg_draws(len(t_values), sum(n_fg), seed=24)
    loss, res = _run(model, batch, t_values, draws)
    form = 'score' if model_name == 'difffg' else 'denoise'
    o_loss, o_res, per_t, o_ot = OE.eval_losses(sd, batch, t_values, *draws, form=form)
    gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag'])
    far = (math.pi - OE.noised_angles_f64(sd, batch, t_values, draws[1])) > MK.NEAR_PI     # [R,n]
    far |= ~gen
    assert far.float().mean() > 0.9
    bl = batch['ligand_type_fg_batch']
    B = int(bl.max()) + 1
    gl = model.last_graph_loss.cpu().view(len(t_values), B, 4)
    for r, t in enumerate(t_values):
        got, want = res[r], o_res[r]
        assert torch.equal(got['vt'].cpu(), want['vt']), f'vt at t={t}'
        f = far[r]
        pk = 'eps_pred' if form == 'score' else 'x_pred'
        for k in (pk, 'R_pred'):
            w = want[k][f]
            assert_close(got[k].cpu()[f], w, rtol=1e-3, atol=1e-3 * float(w.abs().max()), what=f'{k} at t={t}')
        assert_close(got['c_pred'].cpu(), want['c_pred'], rtol=1e-3, atol=1e-5, what=f'c_pred at t={t}')
        # per-graph terms of graphs whose generated FGs are all far from pi
        tgt = draws[0][r] if form == 'score' else want['x0']
        mse = ((want[pk] - tgt) ** 2).sum(-1)
        cos = OE.rotation_cosine_loss(want['R_pred'], want['R0'])
        for g in range(B):
            rows = (bl == g) & gen
            if not bool(rows.any()) or not bool(f[rows].all()):
                continue
            for c, term in ((0, mse[rows].mean()), (1, cos[rows].mean())):
                assert abs(float(gl[r, g, c]) - float(term)) <= 1e-3 * abs(float(term)) + 1e-5, (t, g, c)
        # the type loss does not read o_t: the per-t value, by the sizing rule over the graphs' means
        last = int((gl[r, :, 3] > 0).nonzero().max())
        assert abs(float(gl[r, :last + 1, 2].mean()) - float(per_t[r, 2])) <= 1e-3 * abs(float(per_t[r, 2])) + 1e-6, t
    assert abs(float(loss['fg']) - float(o_loss['fg'])) <= 1e-3 * abs(float(o_loss['fg']))


def _special_orientations(batch):
    """o0 rows with angles at 0, near 0, near pi and at pi (rows 0 .. 7 of the batch)."""
    o = batch['ligand_o_fg'].clone()
    ax = torch.tensor([[1., 0., 0.], [0.6, -0.8, 0.], [0., 0., 1.], [0.48, 0.6, 0.64]])
    o[0] = 0.
    o[1] = ax[1] * 1e-7
    o[2] = ax[2] * 3e-4
    o[3] = ax[3] * (math.pi - 1e-3)
    o[4] = ax[0] * math.pi
    o[5] = ax[1] * (math.pi - 1e-6)
    o[6] = ax[3] * (math.pi / math.sqrt(0.9999))     # beyond pi: the same rotation as the short way round
    o[7] = -ax[2] * (math.pi - 0.02)
    batch['ligand_o_fg'] = o
    return batch


@pytest.mark.gpu
def test_cuda_noised_orientation_matches_float64():
    """exp(o_t) of the noise kernel against float64 exp(e) exp(sqrt(abar_rot) o0) with the same angle draw, to 2e-6 per
    matrix element, at every timestep (t = 0: Gaussian branch; the rest: histogram branch) and for o0 near 0 and pi."""
    T = 20
    model, sd = _model('ragged', 'difffg', DEV, num_layers=1, T=T)
    batch = _special_orientations(synthetic.make_fg_batch([30, 40, 25], [12, 20, 9], seed=31, partial_graphs=(1,)))
    t_values = list(range(T))
    draws = synthetic.make_fg_draws(T, 41, seed=32)
    draws[1][3, 5, 0:3] = 0.0                                          # a zero axis: e = 0
    _run(model, batch, t_values, draws)
    ot = model.last_ot.cpu()
    gen = batch['ligand_gen_flag']
    o0 = batch['ligand_o_fg'].double()
    assert torch.equal(ot[:, ~gen], batch['ligand_o_fg'][~gen].expand(T, -1, -1))
    for r, t in enumerate(t_values):
        rd = draws[1][r]
        theta = OE.forward_angle(sd, t, rd).double()
        e = torch.nn.functional.normalize(rd[:, 0:3].double(), dim=-1) * theta[:, None]
        c0 = float(torch.sqrt(sd['rot_scheduler.alphas_cumprod'][t]))      # the fp32 coefficient the reference uses
        want = _exp64(e) @ _exp64(c0 * o0)
        got = _exp64(ot[r].double())
        err = (got - want).abs().amax(dim=(-2, -1))[gen]
        assert float(err.max()) < 2e-6, (t, float(err.max()), int(err.argmax()))


def _exp64(w):
    """Rodrigues' formula in float64 (exact at small angles, unlike the 1e-8-regularised reference expression)."""
    n = torch.linalg.norm(w, dim=-1)
    x, y, z = w.unbind(-1)
    o = torch.zeros_like(x)
    S = torch.stack([o, z, -y, -z, o, x, y, -x, o], dim=-1).reshape(w.shape[:-1] + (3, 3))
    small = n < 1e-4
    nn_ = torch.where(small, torch.ones_like(n), n)
    b = torch.where(small, 1 - n ** 2 / 6, torch.sin(nn_) / nn_)
    c = torch.where(small, 0.5 - n ** 2 / 24, (1 - torch.cos(nn_)) / nn_ ** 2)
    return torch.eye(3, dtype=w.dtype) + b[..., None, None] * S + c[..., None, None] * (S @ S)


@pytest.mark.gpu
@pytest.mark.parametrize('model_name', ['difffg', 'difffg_v2'])
def test_cuda_launch_splits_are_bit_identical(model_name):
    """One launch == R single-t calls == a launch split by the node budget == a repeat, bit for bit."""
    model, _ = _model('partial_mid_empty', model_name, DEV)
    batch, t_values, draws = _inputs('partial_mid_empty')
    n_nodes = sum(MK.CASES['partial_mid_empty'][2]) + sum(MK.CASES['partial_mid_empty'][3])

    def flat(out):
        loss, res = out
        return [loss[k] for k in LOSS_KEYS] + [v for rr in res for v in rr.values()] + [model.last_ot.clone(),
                                                                                         model.last_graph_loss.clone()]
    one = flat(_run(model, batch, t_values, draws))
    launches = model.last_launches
    again = flat(_run(model, batch, t_values, draws))
    split = flat(_run(model, batch, t_values, draws, max_nodes=3 * n_nodes))
    assert model.last_launches > launches
    singles = [model.eval_losses(batch, [t], draws[0][r:r + 1], draws[1][r:r + 1], draws[2][r:r + 1])
               for r, t in enumerate(t_values)]
    for a, b in zip(one, again):
        assert torch.equal(a.cpu(), b.cpu()) or (a.isnan().all() and b.isnan().all())
    for a, b in zip(one, split):
        assert torch.equal(a.cpu(), b.cpu()) or (a.isnan().all() and b.isnan().all())
    loss, res = one[:3], _run(model, batch, t_values, draws)[1]
    for r, (sl, sr) in enumerate(singles):
        for k, v in sr[0].items():
            assert torch.equal(v.cpu(), res[r][k].cpu()), (r, k)
    # get_dict_mean of the single-t losses: a float32 mean over t of each loss
    for i, k in enumerate(LOSS_KEYS):
        assert torch.equal(torch.mean(torch.tensor([float(sl[k]) for sl, _ in singles])), loss[i]), k


@pytest.mark.gpu
def test_cuda_default_draws_equal_injected_draws():
    model, _ = _model('ragged', 'difffg', DEV)
    batch, t_values, _ = _inputs('ragged')
    n, K, R = sum(MK.CASES['ragged'][3]), 28, len(t_values)
    dev = torch.device(DEV)
    torch.manual_seed(321)
    a_loss, a_res = model(batch)
    torch.manual_seed(321)
    pos, rot, typ = [torch.empty(R, n, d) for d in (3, 6, K)]
    for r in range(R):
        pos[r] = torch.randn(n, 3, device=dev).cpu()
        rot[r, :, 0:3] = torch.randn(n, 3, device=dev).cpu()
        rot[r, :, 3] = torch.rand(n, device=dev).cpu()
        rot[r, :, 4] = torch.rand(n, device=dev).cpu()
        rot[r, :, 5] = torch.randn(n, device=dev).cpu()
        typ[r] = torch.rand(n, K, device=dev).cpu()
    b_loss, b_res = model(batch, pos, rot, typ)
    for k in LOSS_KEYS:
        assert torch.equal(a_loss[k], b_loss[k])
    for ra, rb in zip(a_res, b_res):
        for k in ra:
            assert torch.equal(ra[k].cpu(), rb[k].cpu()), k
