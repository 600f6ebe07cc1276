"""Validation losses: eval-mode TargetDiffB200.forward / eval_losses against the reference's eval-mode
TargetDiff.forward (fixtures of tests/golden/make_golden_f5.py) and the CPU restatement tests/eval_loss_oracle.py."""
import math

import numpy as np
import pytest
import torch

import eval_loss_oracle as EO
from helpers import assert_bitwise, assert_close, case_batch, golden, loss_close, stack, to_dev, make_model
from cbgbench_b200 import synthetic
from cbgbench_b200.targetdiff import eval_t_values

# must match tests/golden/make_golden_f5.py
EVAL_CASES = [
    ('ragged_denovo', 1000, 10, [120, 60, 40], [20, 12, 7], 41, 'denovo', [], 51),
    ('partial_mid_empty', 1000, 10, [80, 60, 50], [15, 10, 12], 42, 'partial', [1], 52),
    ('t50_interval7', 50, 7, [90, 70], [14, 9], 43, 'denovo', [], 53),
    ('interval1', 1000, 1, [100, 50], [16, 8], 44, 'denovo', [], 54),
]


# Losses agree to 1e-4 relative, plus an absolute 5e-7 (four fp32 ulps of 1): at t == 0 the type loss is the decoder
# NLL -log p(v0), with p within ~1e-5 of 1.  That p comes out of a sum of exponentials near 1, so both the reference
# and this path hold it only to about one ulp of 1 (1.2e-7), which is 1e-3 of a 2.6e-5 loss.
LOSS_RTOL, LOSS_ATOL = 1e-4, 5e-7


def per_graph_means(values, gen, batch_idx, n_graphs):
    """Per-graph mean over generated atoms (0 for a graph without any), in float64."""
    out = []
    for g in range(n_graphs):
        sel = gen & (batch_idx == g)
        out.append(float(values[sel].double().mean()) if bool(sel.any()) else 0.0)
    return out


# ---- CPU --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('T,n', [(1000, 10), (50, 10), (50, 7), (1000, 1), (7, 3), (2, 10)])
def test_eval_t_values_match_numpy(T, n):
    want = [int(v) for v in np.trunc(np.linspace(0, T - 1, n))]
    assert eval_t_values(T, n) == want == EO.eval_t_values(T, n)
    if (T, n) == (50, 10):
        assert want == [0, 5, 10, 16, 21, 27, 32, 38, 43, 49]


@pytest.mark.parametrize('case', EVAL_CASES, ids=[c[0] for c in EVAL_CASES])
def test_oracle_matches_fixtures(case):
    name, T, interval, n_prot, n_lig, seed, gen_mode, empty, noise_seed = case
    gd = golden('eval_loss.npz')
    _, sd = make_model(num_steps=T)
    batch = case_batch(n_prot, n_lig, seed, gen_mode, empty)
    t_values = EO.eval_t_values(T, interval)
    assert t_values == gd[f'{name}/t_values'].tolist()
    pn, tu = synthetic.make_noise(len(t_values), batch['ligand_pos'].shape[0], 13, seed=noise_seed)
    loss, res, _ = EO.eval_losses(sd, batch, t_values, pn, tu)
    for key in ('pos', 'atom'):
        assert abs(float(loss[key]) - float(gd[f'{name}/{key}'])) <= 1e-6 * abs(float(gd[f'{name}/{key}']))
    for key in ('xt', 'x_pred', 'c_pred'):
        assert_close(torch.stack([r[key] for r in res]), torch.from_numpy(gd[f'{name}/{key}']), what=key)
    assert torch.equal(torch.stack([r['vt'] for r in res]), torch.from_numpy(gd[f'{name}/vt']))


def test_oracle_scatter_mean_quirks():
    """A graph without generated atoms counts as 0 below the last generated graph id and is dropped above it; no
    generated atom at all gives NaN (mean of an empty tensor)."""
    _, sd = make_model(num_steps=100)
    t_values = [0, 40, 99]
    for empty, n_counted in (([1], 3), ([2], 2), ([0, 1, 2], 0)):
        batch = case_batch([30, 25, 20], [6, 5, 4], seed=61, empty_graphs=empty)
        n = batch['ligand_pos'].shape[0]
        pn, tu = synthetic.make_noise(len(t_values), n, 13, seed=62)
        _, res, per_t = EO.eval_losses(sd, batch, t_values, pn, tu)
        for r, (lp, _) in enumerate(per_t):
            if n_counted == 0:
                assert math.isnan(float(lp))
                continue
            mse = ((res[r]['x_pred'] - res[r]['x0']) ** 2).sum(-1)
            means = per_graph_means(mse, res[r]['mask_gen'], batch['ligand_element_batch'], n_counted)
            assert abs(float(lp) - sum(means) / n_counted) <= 1e-6 * abs(float(lp))


def test_training_mode_forward_raises():
    model, _ = make_model(num_steps=10)
    model.train()
    with pytest.raises(NotImplementedError, match='autograd'):
        model(synthetic.make_batch([20], [5], seed=1))


def test_diffsbdd_forward_is_a_sampling_build():
    from cbgbench_b200.targetdiff import get_model
    model = get_model(synthetic.diffsbdd_config(num_steps=10)).eval()
    with pytest.raises(NotImplementedError, match='sampling build'):
        model(synthetic.make_batch([20], [5], seed=1))


def test_diffbp_forward_on_a_cpu_model_raises():
    from cbgbench_b200.targetdiff import get_model
    model = get_model(synthetic.diffbp_config(num_steps=10)).eval()
    with pytest.raises(NotImplementedError, match='CUDA device'):
        model(synthetic.make_batch([20], [5], seed=1))


# ---- GPU --------------------------------------------------------------------------------------------------------------
def gpu_model(T, interval=None):
    model, sd = make_model(num_steps=T, device='cuda')
    if interval is not None:
        model.cfg['eval_interval'] = interval
    return model, sd


@pytest.mark.gpu
@pytest.mark.parametrize('case', EVAL_CASES, ids=[c[0] for c in EVAL_CASES])
def test_gpu_forward_matches_reference_fixtures(case):
    name, T, interval, n_prot, n_lig, seed, gen_mode, empty, noise_seed = case
    gd = golden('eval_loss.npz')
    model, _ = gpu_model(T, interval)
    batch = case_batch(n_prot, n_lig, seed, gen_mode, empty)
    R = len(gd[f'{name}/t_values'])
    pn, tu = synthetic.make_noise(R, batch['ligand_pos'].shape[0], 13, seed=noise_seed)
    dbatch = to_dev(batch)
    loss, res = model(dbatch, pos_noise=pn, type_uniform=tu)
    for key in ('pos', 'atom'):
        assert loss[key].device.type == 'cpu' and loss[key].dtype == torch.float32 and loss[key].dim() == 0
        want = float(gd[f'{name}/{key}'])
        assert loss_close(float(loss[key]), want, LOSS_RTOL, LOSS_ATOL), (key, float(loss[key]), want)
    assert len(res) == R
    assert torch.equal(stack(res, 'vt'), torch.from_numpy(gd[f'{name}/vt']))
    for key in ('xt', 'x_pred', 'c_pred'):
        assert_close(stack(res, key), torch.from_numpy(gd[f'{name}/{key}']), what=key)
    gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag'])
    for r in res:
        assert set(r) == {'x0', 'xt', 'x_pred', 'mask_gen', 'v0', 'vt', 'c_pred'}
        assert all(v.device.type == 'cuda' for v in r.values())
        assert r['vt'].dtype == torch.int64 and r['mask_gen'].dtype == torch.bool
        assert torch.equal(r['x0'].cpu(), batch['ligand_pos'])
        assert torch.equal(r['v0'].cpu(), batch['ligand_atom_type'])
        assert torch.equal(r['mask_gen'].cpu(), gen)
    # the reference's evaluator (AUROC over v0 vs c_pred, masked by mask_gen) on these results
    assert abs(EO.auroc(res) - float(gd[f'{name}/auroc'])) < 1e-3


def check_against_oracle(model, sd, batch, t_values, noise_seed):
    n = batch['ligand_pos'].shape[0]
    pn, tu = synthetic.make_noise(len(t_values), n, 13, seed=noise_seed)
    loss, res = model.eval_losses(to_dev(batch), t_values, pos_noise=pn, type_uniform=tu)
    o_loss, o_res, _ = EO.eval_losses(sd, batch, t_values, pn, tu)
    for key in ('pos', 'atom'):
        want = float(o_loss[key])
        if math.isnan(want):
            assert math.isnan(float(loss[key]))
        else:
            assert loss_close(float(loss[key]), want, LOSS_RTOL, LOSS_ATOL), (key, float(loss[key]), want)
    assert torch.equal(stack(res, 'vt'), torch.stack([r['vt'] for r in o_res]))
    for key in ('xt', 'x_pred', 'c_pred'):
        assert_close(stack(res, key), torch.stack([r[key] for r in o_res]), what=key)


@pytest.mark.gpu
def test_gpu_matches_oracle_config2_shape():
    """The shipped sampling shape: 64 pockets of 300 atoms with 24-atom ligands (at the two end timesteps: the CPU
    oracle takes ~35 s per timestep at this size)."""
    model, sd = gpu_model(1000)
    batch = synthetic.make_batch([300] * 64, [24] * 64, seed=71)
    check_against_oracle(model, sd, batch, [0, 999], noise_seed=72)


@pytest.mark.gpu
def test_gpu_matches_oracle_ragged_pockets():
    model, sd = gpu_model(1000)
    batch = case_batch([100, 350, 800, 520], [12, 30, 45, 22], seed=73, gen_mode='partial')
    check_against_oracle(model, sd, batch, [0, 1, 300, 999], noise_seed=74)


@pytest.mark.gpu
def test_gpu_scatter_mean_quirks_match_oracle():
    model, sd = gpu_model(100)
    for empty in ([2], [0, 1, 2]):      # trailing graph dropped; nothing generated -> NaN
        batch = case_batch([30, 25, 20], [6, 5, 4], seed=61, empty_graphs=empty)
        check_against_oracle(model, sd, batch, [0, 40, 99], noise_seed=62)


def run_eval(model, batch, t_values, pn, tu, **kw):
    loss, res = model.eval_losses(batch, t_values, pos_noise=pn, type_uniform=tu, **kw)
    return loss, {k: stack(res, k) for k in ('xt', 'vt', 'x_pred', 'c_pred')}


@pytest.mark.gpu
def test_gpu_replica_batching_is_exact():
    """R replicas in one launch == R single-timestep calls == a forced split over several launches, bit for bit;
    repeated runs are bit-identical."""
    model, _ = gpu_model(1000)
    batch = to_dev(case_batch([150, 90, 60], [20, 14, 9], seed=81, gen_mode='partial'))
    t_values = eval_t_values(1000, 10)
    n = batch['ligand_pos'].shape[0]
    pn, tu = synthetic.make_noise(len(t_values), n, 13, seed=82)
    one = run_eval(model, batch, t_values, pn, tu)
    assert_bitwise(one, run_eval(model, batch, t_values, pn, tu), ('pos', 'atom'))
    n_nodes = n + batch['protein_pos'].shape[0]
    # launches of 3, 3, 3, 1
    assert_bitwise(one, run_eval(model, batch, t_values, pn, tu, max_nodes=3 * n_nodes), ('pos', 'atom'))
    singles = [run_eval(model, batch, [t], pn[r:r + 1], tu[r:r + 1]) for r, t in enumerate(t_values)]
    for k in one[1]:
        assert torch.equal(one[1][k], torch.cat([s[1][k] for s in singles])), k
    for k in ('pos', 'atom'):
        assert torch.equal(one[0][k], torch.mean(torch.tensor([float(s[0][k]) for s in singles]))), k


@pytest.mark.gpu
def test_gpu_default_noise_is_the_seeded_draws():
    """Without injected noise the draws are torch's on the model device, per t: randn [n_lig,3] then rand [n_lig,K]."""
    model, _ = gpu_model(1000)
    batch = to_dev(case_batch([80, 40], [12, 7], seed=91))
    n, K, R = batch['ligand_pos'].shape[0], 13, 10
    torch.manual_seed(1234)
    default = model(batch)
    torch.manual_seed(1234)
    draws = [(torch.randn(n, 3, device='cuda'), torch.rand(n, K, device='cuda')) for _ in range(R)]
    injected = model(batch, pos_noise=torch.stack([d[0] for d in draws]), type_uniform=torch.stack([d[1] for d in draws]))
    for k in ('pos', 'atom'):
        assert torch.equal(default[0][k], injected[0][k])
    for a, b in zip(default[1], injected[1]):
        for k in a:
            assert torch.equal(a[k], b[k]), k
