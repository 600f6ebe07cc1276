"""DiffSBDD validation losses: eval-mode DiffSBDDB200.forward / eval_losses against the reference's eval-mode
DiffSBDD.forward (fixtures of tests/golden/make_golden_f7.py) and the CPU restatement tests/sbdd_eval_loss_oracle.py."""
import math

import numpy as np
import pytest
import torch

import sbdd_eval_loss_oracle as SO
from helpers import assert_bitwise, assert_close, case_batch, golden, loss_close, stack, to_dev
from cbgbench_b200 import synthetic
from cbgbench_b200.diffsbdd import DiffSBDDB200, eval_t_values

# must match tests/golden/make_golden_f7.py
SBDD_EVAL_CASES = [
    ('ragged_denovo', 1000, 10, [120, 60, 90], [20, 12, 30], 241, 'denovo', [], 251),
    ('partial_empty', 1000, 10, [80, 60, 50, 40], [15, 10, 12, 9], 242, 'partial', [1], 252),
    ('middle_empty_one_atom', 1000, 10, [70, 50, 40], [14, 0, 1], 243, 'denovo', [], 253),
    ('t50_interval7', 50, 7, [90, 70], [14, 9], 244, 'denovo', [], 254),
    ('interval1', 1000, 1, [100, 50], [16, 8], 245, 'denovo', [], 255),
]
K = 13
WEIGHT_SEED = 0
LOSS_KEYS = ('pos', 'atom')
VEC_KEYS = ('eps_0_pos', 'eps_pred_pos', 'score_0_pos', 'score_pred_pos',
            'eps_0_atom', 'eps_pred_atom', 'score_0_atom', 'score_pred_atom')
# The losses are means of per-graph terms of order 1 - 1e4, so a relative bar alone suffices for them.  A per-graph term
# can be a small difference of large summands: pos_kl = d log(1/sigma_T) + 0.5 (d sigma_T^2 + |alpha_T x0|^2) - 0.5 d with
# d = 3 (n_g - 1) up to ~200 and sigma_T^2 = 1 - 5e-4 ends near 0.5 |alpha_T x0|^2 ~ 1e-2.  Its summands are the same fp32
# values here and in the reference except the fixed-order sum |alpha_T x0|^2, so the two results differ by a few ulps of
# the summands (ulp(128) = 1.5e-5): the terms get an absolute 5e-5 beside the relative 1e-4.
LOSS_RTOL, TERM_ATOL = 1e-4, 5e-5


def sbdd_model(T, device=None, interval=None, **kw):
    model = DiffSBDDB200(synthetic.diffsbdd_config(num_steps=T, **kw))
    sd = synthetic.seeded_state_dict(model, seed=WEIGHT_SEED)
    model.load_state_dict(sd, strict=True)
    model.eval()
    if interval is not None:
        model.cfg['eval_interval'] = interval
    return (model.to(device) if device is not None else model), sd


# ---- CPU --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', SBDD_EVAL_CASES, ids=[c[0] for c in SBDD_EVAL_CASES])
def test_oracle_matches_fixtures(case):
    name, T, interval, n_prot, n_lig, seed, gen_mode, empty, noise_seed = case
    gd = golden('sbdd_eval_loss.npz')
    _, sd = sbdd_model(T)
    batch = case_batch(n_prot, n_lig, seed, gen_mode, empty)
    t_values = SO.eval_t_values(T, interval)
    assert t_values == gd[f'{name}/t_values'].tolist()
    noise = synthetic.make_sbdd_eval_noise(len(t_values), batch['ligand_pos'].shape[0], K, seed=noise_seed)
    loss, res, per_t, terms = SO.eval_losses(sd, batch, t_values, noise, T, K)
    for key in LOSS_KEYS:
        want = float(gd[f'{name}/{key}'])
        assert abs(float(loss[key]) - want) <= 1e-6 * abs(want), key
    assert_close(terms, torch.from_numpy(gd[f'{name}/terms']), rtol=1e-6, atol=1e-6, what='terms')
    for key in VEC_KEYS:
        assert_close(torch.stack([r[key] for r in res]), torch.from_numpy(gd[f'{name}/{key}']), what=key)
    assert torch.equal(torch.stack([r['mask_gen_pos'] for r in res]), torch.from_numpy(gd[f'{name}/mask_gen_pos']))


@pytest.mark.parametrize('T,n', [(1000, 10), (1000, 1), (50, 7), (10, 10), (1000, 3), (7, 4)])
def test_t_values_are_the_truncated_linspace_from_1_to_T(T, n):
    want = np.trunc(np.linspace(1, T, n)).astype(np.int64).tolist()
    assert eval_t_values(T, n) == want == SO.eval_t_values(T, n)
    assert want[0] == 1 and (want[-1] == T or n == 1)


def test_host_scalars_are_the_references_fp32_expressions():
    model, sd = sbdd_model(1000, num_layers=1)
    for t in (1, 112, 999, 1000):
        c = model.eval_coef(t)
        for pre, key in (('pos', 'pos_scheduler.gamma.gamma'), ('type', 'type_scheduler.gamma.gamma')):
            g_s, g_t, g_0, g_T = SO.schedule(sd[key], t, 1000)
            a_t, s_t = SO.alpha_sigma(g_t)
            a_0, s_0 = SO.alpha_sigma(g_0)
            a_T, s_T = SO.alpha_sigma(g_T)
            want = {'alpha_t': a_t, 'sigma_t': s_t, 'alpha_0': a_0, 'sigma_0': s_0, 'alpha_T': a_T,
                    't_weight': -1000 * 0.5 * (1 - torch.exp(-(g_s - g_t))),
                    'log_const': -(0.5 * g_0) - SO.LOG_2PI_HALF, 'log_inv_sigma_T': torch.log(1 / s_T),
                    'sigma2_T': s_T ** 2}
            for k, v in want.items():
                assert getattr(c, f'{pre}_{k}') == float(v[0]), (t, pre, k)


def test_forward_raises_without_a_gpu_path():
    batch = synthetic.make_batch([20], [5], seed=1)
    model, _ = sbdd_model(10, num_layers=1)
    model.train()
    with pytest.raises(NotImplementedError, match='autograd'):
        model(batch)
    model.eval()
    with pytest.raises(NotImplementedError, match='CUDA device'):
        model(batch)                                      # CPU model: no CPU implementation, no fallback
    with pytest.raises(ValueError, match=r'\[1, 10\]'):
        model.eval_losses(batch, [0])                     # DiffSBDD's timesteps run from 1 to T


# ---- GPU --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('case', SBDD_EVAL_CASES, ids=[c[0] for c in SBDD_EVAL_CASES])
def test_gpu_forward_matches_reference_fixtures(case):
    name, T, interval, n_prot, n_lig, seed, gen_mode, empty, noise_seed = case
    gd = golden('sbdd_eval_loss.npz')
    model, _ = sbdd_model(T, 'cuda', interval)
    batch = case_batch(n_prot, n_lig, seed, gen_mode, empty)
    R, n = len(gd[f'{name}/t_values']), batch['ligand_pos'].shape[0]
    noise = synthetic.make_sbdd_eval_noise(R, n, K, seed=noise_seed)
    loss, res = model(to_dev(batch), noise=noise)
    assert list(loss) == list(LOSS_KEYS)
    for key in LOSS_KEYS:
        assert loss[key].device.type == 'cpu' and loss[key].dtype == torch.float32 and loss[key].dim() == 0
        want = float(gd[f'{name}/{key}'])
        assert loss_close(float(loss[key]), want, LOSS_RTOL), (key, float(loss[key]), want)
    assert_close(model.last_terms.cpu(), torch.from_numpy(gd[f'{name}/terms']), rtol=LOSS_RTOL, atol=TERM_ATOL, what='terms')
    assert len(res) == R
    for key in VEC_KEYS:
        assert_close(stack(res, key), torch.from_numpy(gd[f'{name}/{key}']), what=key)
    gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag'])
    for r in res:
        assert list(r) == list(SO.RESULT_KEYS)
        assert all(v.device.type == 'cuda' for v in r.values())
        for key in VEC_KEYS:
            assert r[key].dtype == torch.float32 and r[key].shape == (n, 3 if key.endswith('_pos') else K)
        for key in ('mask_gen_pos', 'mask_gen_atom'):
            assert r[key].dtype == torch.bool and torch.equal(r[key].cpu(), gen)
    assert torch.equal(stack(res, 'mask_gen_pos'), torch.from_numpy(gd[f'{name}/mask_gen_pos']))


def check_against_oracle(model, sd, batch, t_values, noise_seed):
    T = model.num_diffusion_timesteps
    noise = synthetic.make_sbdd_eval_noise(len(t_values), batch['ligand_pos'].shape[0], K, seed=noise_seed)
    loss, res = model.eval_losses(to_dev(batch), t_values, noise=noise)
    o_loss, o_res, _, o_terms = SO.eval_losses(sd, batch, t_values, noise, T, K)
    for key in LOSS_KEYS:
        assert loss_close(float(loss[key]), float(o_loss[key]), LOSS_RTOL), (key, float(loss[key]), float(o_loss[key]))
    assert_close(model.last_terms.cpu(), o_terms, rtol=LOSS_RTOL, atol=TERM_ATOL, what='terms')
    for key in ('mask_gen_pos', 'mask_gen_atom'):
        assert torch.equal(stack(res, key), torch.stack([r[key] for r in o_res])), key
    for key in VEC_KEYS:
        assert_close(stack(res, key), torch.stack([r[key] for r in o_res]), what=key)


@pytest.mark.gpu
def test_gpu_matches_oracle_config2_shape():
    """The shipped sampling shape: 64 pockets of 300 atoms with 24-atom ligands, at the two end timesteps."""
    model, sd = sbdd_model(1000, 'cuda')
    batch = synthetic.make_batch([300] * 64, [24] * 64, seed=271)
    check_against_oracle(model, sd, batch, [1, 1000], noise_seed=272)


@pytest.mark.gpu
def test_gpu_matches_oracle_ragged_pockets():
    """100 - 800-atom pockets with partial generation."""
    model, sd = sbdd_model(1000, 'cuda')
    batch = case_batch([100, 350, 800, 520], [12, 30, 64, 22], seed=273, gen_mode='partial')
    check_against_oracle(model, sd, batch, [1, 2, 300, 1000], noise_seed=274)


@pytest.mark.gpu
@pytest.mark.parametrize('n_prot,n_lig', [([80], [1]), ([60, 50, 40], [10, 0, 6]), ([0, 90], [5, 20]),
                                          ([60, 40], [10, 0]), ([70, 30], [1, 12])],
                         ids=['one_atom', 'middle_without_ligand', 'no_pocket', 'trailing_pocket_only', 'one_atom_first'])
def test_gpu_edges(n_prot, n_lig):
    """t = T, a one-atom ligand (d = 0), a graph without ligand atoms in the middle (its n_g = 0 terms count) and at the
    end (dropped; its pocket keeps its coordinates), a graph without a pocket."""
    model, sd = sbdd_model(100, 'cuda', num_layers=3)
    batch = case_batch(n_prot, n_lig, 275, gen_mode='partial')
    check_against_oracle(model, sd, batch, [1, 50, 100], noise_seed=276)


def run_eval(model, batch, t_values, noise, **kw):
    loss, res = model.eval_losses(batch, t_values, noise=noise, **kw)
    return loss, {k: stack(res, k) for k in res[0]}, model.last_terms.cpu()


@pytest.mark.gpu
def test_gpu_replica_batching_is_exact():
    """2R copies in one launch == R single-timestep calls == a forced split over several launches == a repeat == the
    unpruned denoiser, bit for bit."""
    model, _ = sbdd_model(1000, 'cuda')
    batch = to_dev(case_batch([150, 90, 60], [20, 14, 55], seed=281, gen_mode='partial'))
    t_values = eval_t_values(1000, 10)
    n = batch['ligand_pos'].shape[0]
    noise = synthetic.make_sbdd_eval_noise(len(t_values), n, K, seed=282)
    one = run_eval(model, batch, t_values, noise)
    assert model.last_launches > 0
    assert_bitwise(one, run_eval(model, batch, t_values, noise), LOSS_KEYS)
    n_nodes = n + batch['protein_pos'].shape[0]
    assert_bitwise(one, run_eval(model, batch, t_values, noise, max_nodes=6 * n_nodes), LOSS_KEYS)    # 3, 3, 3, 1 timesteps
    singles = [run_eval(model, batch, [t], {k: v[r:r + 1] for k, v in noise.items()}) for r, t in enumerate(t_values)]
    for k in one[1]:
        if k.startswith('mask_gen'):
            continue
        assert torch.equal(one[1][k], torch.cat([s[1][k] for s in singles])), k
    assert torch.equal(one[2], torch.cat([s[2] for s in singles]))
    for k in LOSS_KEYS:
        assert torch.equal(one[0][k], torch.mean(torch.tensor([float(s[0][k]) for s in singles]))), k
    model.use_prune = False
    assert_bitwise(one, run_eval(model, batch, t_values, noise), LOSS_KEYS)


@pytest.mark.gpu
def test_gpu_default_noise_is_the_seeded_draws():
    """Without injected noise the draws are torch's on the model device, per t: randn [n_lig,3], [n_lig,K] at t, then
    the same two at 0."""
    model, _ = sbdd_model(1000, 'cuda')
    batch = to_dev(case_batch([80, 40], [12, 7], seed=291))
    n, R = batch['ligand_pos'].shape[0], 10
    torch.manual_seed(1234)
    default = model(batch)
    torch.manual_seed(1234)
    draws = [[torch.randn(n, d, device='cuda') for d in (3, K, 3, K)] for _ in range(R)]
    noise = {k: torch.stack([d[i] for d in draws]) for i, k in enumerate(('x_t', 'c_t', 'x_0', 'c_0'))}
    injected = model(batch, noise=noise)
    for k in LOSS_KEYS:
        assert torch.equal(default[0][k], injected[0][k])
    for a, b in zip(default[1], injected[1]):
        for k in a:
            assert torch.equal(a[k], b[k]), k
    assert not math.isnan(float(default[0]['pos']))
