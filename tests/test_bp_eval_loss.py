"""DiffBP validation losses: eval-mode DiffBPB200.forward / eval_losses against the reference's eval-mode DiffBP.forward
(fixtures of tests/golden/make_golden_f6.py) and the CPU restatement tests/bp_eval_loss_oracle.py."""
import math

import pytest
import torch

import bp_eval_loss_oracle as BO
from helpers import assert_bitwise, assert_close, case_batch, golden, loss_close, stack, to_dev
from cbgbench_b200 import synthetic
from cbgbench_b200.diffbp import DiffBPB200
from cbgbench_b200.targetdiff import eval_t_values

# must match tests/golden/make_golden_f6.py
BP_EVAL_CASES = [
    ('ragged_denovo', 1000, 10, [120, 60, 90], [20, 12, 60], 141, 'denovo', [], 151),
    ('partial_empty', 1000, 10, [80, 60, 50, 40], [15, 10, 12, 9], 142, 'partial', [1, 3], 152),
    ('t50_interval7', 50, 7, [90, 70], [14, 9], 143, 'denovo', [], 153),
    ('interval1', 1000, 1, [100, 50], [16, 8], 144, 'denovo', [], 154),
]
LOSS_KEYS = ('pos', 'atom', 'com', 'inter')
VEC_KEYS = ('eps_0', 'eps_pred', 'score_0', 'score_pred', 'eps_0_com', 'eps_pred_com', 'score_0_com', 'score_pred_com')
WEIGHT_SEED = 0
# All four losses are means of terms of order 0.1 - 10 (or exactly 0: the atom loss without masked atoms, and the
# position loss of a one-atom ligand, whose zero-centred noise and prediction are both exactly 0), so a relative bar
# alone suffices.
LOSS_RTOL = 1e-4


def bp_model(T, device=None, interval=None, **kw):
    model = DiffBPB200(synthetic.diffbp_config(num_steps=T, **kw))
    sd = synthetic.seeded_state_dict(model, seed=WEIGHT_SEED)
    model.load_state_dict(sd, strict=True)
    model.eval()
    if interval is not None:
        model.cfg['eval_interval'] = interval
    return (model.to(device) if device is not None else model), sd


# ---- CPU --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', BP_EVAL_CASES, ids=[c[0] for c in BP_EVAL_CASES])
def test_oracle_matches_fixtures(case):
    name, T, interval, n_prot, n_lig, seed, gen_mode, empty, noise_seed = case
    gd = golden('bp_eval_loss.npz')
    _, sd = bp_model(T)
    batch = case_batch(n_prot, n_lig, seed, gen_mode, empty)
    t_values = BO.eval_t_values(T, interval)
    assert t_values == gd[f'{name}/t_values'].tolist()
    pn, tu = synthetic.make_bp_noise(len(t_values), batch['ligand_pos'].shape[0], seed=noise_seed)
    loss, res, _ = BO.eval_losses(sd, batch, t_values, pn, tu, T)
    for key in LOSS_KEYS:
        want = float(gd[f'{name}/{key}'])
        assert abs(float(loss[key]) - want) <= 1e-6 * abs(want), key
    for key in VEC_KEYS + ('c_pred',):
        assert_close(torch.stack([r[key] for r in res]), torch.from_numpy(gd[f'{name}/{key}']), what=key)
    for key in ('vt', 'mask_gen'):
        assert torch.equal(torch.stack([r[key] for r in res]), torch.from_numpy(gd[f'{name}/{key}'])), key


def test_knn_all_pairs_and_ties():
    """graph_ops-style knn: each y gets its min(k, n_x_g) nearest x of the same graph, nearest first, ties to the
    lower x index; with n_x_g <= k every pair of the graph is an edge."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(30, 3, generator=g)
    y = torch.randn(7, 3, generator=g)
    bx = torch.tensor([0] * 20 + [1] * 10)
    by = torch.tensor([0] * 4 + [1] * 3)
    e = BO.knn(x, y, 48, bx, by)
    assert e.shape[1] == 4 * 20 + 3 * 10
    for j in range(7):
        cols = e[1][e[0] == j]
        assert sorted(cols.tolist()) == torch.nonzero(bx == by[j]).flatten().tolist()
        d = ((x[cols] - y[j]) ** 2).sum(-1)
        assert bool((d[1:] >= d[:-1]).all())
    # ties: three copies of one point at the cut of k = 2 -> the two lowest indices
    x = torch.tensor([[5., 0., 0.], [1., 0., 0.], [0., 1., 0.], [0., 0., 1.], [3., 0., 0.]])
    e = BO.knn(x, torch.zeros(1, 3), 2)
    assert e[1].tolist() == [1, 2]
    e = BO.knn(x, torch.zeros(1, 3), 3)
    assert e[1].tolist() == [1, 2, 3]


def test_oracle_sizing_quirks():
    """pos / com: no generated atom gives NaN, a trailing graph without generated atoms is dropped and one in the
    middle counts as 0; atom: no masked atom (every t = 0) gives 0."""
    T = 100
    _, sd = bp_model(T, num_layers=2, num_layers_com=1)
    t_values = [0, 60]
    for empty, n_counted in (([1], 3), ([2], 2), ([0, 1, 2], 0)):
        batch = case_batch([30, 25, 20], [6, 5, 4], seed=61, empty_graphs=empty)
        pn, tu = synthetic.make_bp_noise(len(t_values), batch['ligand_pos'].shape[0], seed=62)
        _, res, per_t = BO.eval_losses(sd, batch, t_values, pn, tu, T)
        assert float(per_t[0][1]) == 0.0                  # t = 0: nothing is masked
        for r, (lp, la, lc, li) in enumerate(per_t):
            assert math.isfinite(float(li))
            if n_counted == 0:
                assert math.isnan(float(lp)) and math.isnan(float(lc))
                assert float(la) == 0.0                   # the type mask is gen-masked too
                continue
            bl, gen = batch['ligand_element_batch'], res[r]['mask_gen_com']
            mse = ((res[r]['eps_pred'] - res[r]['eps_0']) ** 2).sum(-1)
            means = [float(mse[gen & (bl == g)].double().mean()) if bool((gen & (bl == g)).any()) else 0.0
                     for g in range(n_counted)]
            assert abs(float(lp) - sum(means) / n_counted) <= 1e-6 * abs(float(lp))


def test_forward_raises_without_a_gpu_path():
    batch = synthetic.make_batch([20], [5], seed=1)
    model, _ = bp_model(10, num_layers=1, num_layers_com=1)
    model.train()
    with pytest.raises(NotImplementedError, match='autograd'):
        model(batch)
    model.eval()
    with pytest.raises(NotImplementedError, match='CUDA device'):
        model(batch)                                      # CPU model: no CPU implementation, no fallback
    cfg = synthetic.diffbp_config(num_steps=10, num_layers=1, num_layers_com=1)
    cfg['intersect_reg'] = False
    model = DiffBPB200(cfg).eval()
    with pytest.raises(NotImplementedError, match='intersect_reg'):
        model(batch)


# ---- GPU --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('case', BP_EVAL_CASES, ids=[c[0] for c in BP_EVAL_CASES])
def test_gpu_forward_matches_reference_fixtures(case):
    name, T, interval, n_prot, n_lig, seed, gen_mode, empty, noise_seed = case
    gd = golden('bp_eval_loss.npz')
    model, _ = bp_model(T, 'cuda', interval)
    batch = case_batch(n_prot, n_lig, seed, gen_mode, empty)
    R = len(gd[f'{name}/t_values'])
    pn, tu = synthetic.make_bp_noise(R, batch['ligand_pos'].shape[0], seed=noise_seed)
    loss, res = model(to_dev(batch), pos_noise=pn, type_uniform=tu)
    assert set(loss) == set(LOSS_KEYS)
    for key in LOSS_KEYS:
        assert loss[key].device.type == 'cpu' and loss[key].dtype == torch.float32 and loss[key].dim() == 0
        want = float(gd[f'{name}/{key}'])
        assert loss_close(float(loss[key]), want, LOSS_RTOL, nan_equal=True), (key, float(loss[key]), want)
    assert len(res) == R
    assert torch.equal(stack(res, 'vt'), torch.from_numpy(gd[f'{name}/vt']))
    assert torch.equal(stack(res, 'mask_gen'), torch.from_numpy(gd[f'{name}/mask_gen']))
    for key in VEC_KEYS + ('c_pred',):
        assert_close(stack(res, key), torch.from_numpy(gd[f'{name}/{key}']), what=key)
    gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag'])
    for r in res:
        assert list(r) == list(BO.RESULT_KEYS)
        assert all(v.device.type == 'cuda' for v in r.values())
        assert r['vt'].dtype == torch.float32 and r['c_pred'].dtype == torch.float32
        assert r['mask_gen'].dtype == torch.bool and r['v0'].dtype == torch.int64
        assert all(r[k].dtype == torch.float32 and r[k].shape == (batch['ligand_pos'].shape[0], 3) for k in VEC_KEYS)
        assert torch.equal(r['v0'].cpu(), batch['ligand_atom_type'])
        assert torch.equal(r['mask_gen_com'].cpu(), gen)
    want = float(gd[f'{name}/auroc'])
    got = BO.auroc(res)
    assert (math.isnan(want) and math.isnan(got)) or abs(got - want) < 1e-3


def check_against_oracle(model, sd, batch, t_values, noise_seed):
    T = model.num_diffusion_timesteps
    pn, tu = synthetic.make_bp_noise(len(t_values), batch['ligand_pos'].shape[0], seed=noise_seed)
    loss, res = model.eval_losses(to_dev(batch), t_values, pos_noise=pn, type_uniform=tu)
    o_loss, o_res, _ = BO.eval_losses(sd, batch, t_values, pn, tu, T)
    for key in LOSS_KEYS:
        assert loss_close(float(loss[key]), float(o_loss[key]), LOSS_RTOL, nan_equal=True), \
            (key, float(loss[key]), float(o_loss[key]))
    for key in ('vt', 'mask_gen', 'mask_gen_com'):
        assert torch.equal(stack(res, key), torch.stack([r[key] for r in o_res])), key
    for key in VEC_KEYS + ('c_pred',):
        assert_close(stack(res, key), torch.stack([r[key] for r in o_res]), what=key)


@pytest.mark.gpu
def test_gpu_matches_oracle_config2_shape():
    """The shipped sampling shape: 64 pockets of 300 atoms with 24-atom ligands, at the two end timesteps."""
    model, sd = bp_model(1000, 'cuda')
    batch = synthetic.make_batch([300] * 64, [24] * 64, seed=171)
    check_against_oracle(model, sd, batch, [0, 999], noise_seed=172)


@pytest.mark.gpu
def test_gpu_matches_oracle_ragged_pockets():
    """100 - 800-atom pockets, partial generation, one ligand above the kNN's k = 48."""
    model, sd = bp_model(1000, 'cuda')
    batch = case_batch([100, 350, 800, 520], [12, 30, 64, 22], seed=173, gen_mode='partial')
    check_against_oracle(model, sd, batch, [0, 1, 300, 999], noise_seed=174)


def duplicate_batch(n_prot, n_lig, seed):
    """Partial generation (the fixed first two thirds keep x_t = x0 = xs_mean) with ligand atoms 1 .. 9 placed on atom 0:
    exact ties in the protein -> ligand kNN."""
    batch = case_batch(n_prot, n_lig, seed, gen_mode='partial')
    pos = batch['ligand_pos'].clone()
    pos[1:10] = pos[0]
    batch['ligand_pos'] = pos
    return batch


@pytest.mark.gpu
@pytest.mark.parametrize('n_prot,n_lig,dup', [([300], [48], False), ([300], [49], False), ([400], [200], False),
                                              ([120], [60], True), ([80], [1], False), ([0, 90], [5, 50], True)],
                         ids=['n48', 'n49', 'n200', 'duplicates', 'one_atom', 'no_pocket_then_dup'])
def test_gpu_interior_loss_edges(n_prot, n_lig, dup):
    model, sd = bp_model(100, 'cuda', num_layers=3, num_layers_com=2)
    batch = (duplicate_batch if dup else lambda p, l, s: case_batch(p, l, s, gen_mode='partial'))(n_prot, n_lig, 175)
    check_against_oracle(model, sd, batch, [0, 50, 99], noise_seed=176)


def run_eval(model, batch, t_values, pn, tu, **kw):
    loss, res = model.eval_losses(batch, t_values, pos_noise=pn, type_uniform=tu, **kw)
    return loss, {k: stack(res, k) for k in res[0]}


@pytest.mark.gpu
def test_gpu_replica_batching_is_exact():
    """R replicas in one launch == R single-timestep calls == a forced split over several launches == a repeat == the
    unpruned denoiser without static lists, bit for bit."""
    model, _ = bp_model(1000, 'cuda')
    batch = to_dev(case_batch([150, 90, 60], [20, 14, 55], seed=181, gen_mode='partial'))
    t_values = eval_t_values(1000, 10)
    n = batch['ligand_pos'].shape[0]
    pn, tu = synthetic.make_bp_noise(len(t_values), n, seed=182)
    one = run_eval(model, batch, t_values, pn, tu)
    assert model.last_launches > 0
    assert_bitwise(one, run_eval(model, batch, t_values, pn, tu), LOSS_KEYS, nan_equal=True)
    n_nodes = n + batch['protein_pos'].shape[0]
    # launches of 3, 3, 3, 1
    assert_bitwise(one, run_eval(model, batch, t_values, pn, tu, max_nodes=3 * n_nodes), LOSS_KEYS, nan_equal=True)
    singles = [run_eval(model, batch, [t], pn[r:r + 1], tu[r:r + 1]) for r, t in enumerate(t_values)]
    for k in one[1]:
        if k in ('v0', 'mask_gen_com'):
            continue
        assert torch.equal(one[1][k], torch.cat([s[1][k] for s in singles])), k
    for k in LOSS_KEYS:
        assert torch.equal(one[0][k], torch.mean(torch.tensor([float(s[0][k]) for s in singles]))), k
    model.use_prune = model.use_static_lists = False
    assert_bitwise(one, run_eval(model, batch, t_values, pn, tu), LOSS_KEYS, nan_equal=True)


@pytest.mark.gpu
def test_gpu_default_noise_is_the_seeded_draws():
    """Without injected noise the draws are torch's on the model device, per t: randn [n_lig,3] then rand [n_lig]."""
    model, _ = bp_model(1000, 'cuda')
    batch = to_dev(case_batch([80, 40], [12, 7], seed=191))
    n, R = batch['ligand_pos'].shape[0], 10
    torch.manual_seed(1234)
    default = model(batch)
    torch.manual_seed(1234)
    draws = [(torch.randn(n, 3, device='cuda'), torch.rand(n, device='cuda')) for _ in range(R)]
    injected = model(batch, pos_noise=torch.stack([d[0] for d in draws]), type_uniform=torch.stack([d[1] for d in draws]))
    for k in LOSS_KEYS:
        assert torch.equal(default[0][k], injected[0][k])
    for a, b in zip(default[1], injected[1]):
        for k in a:
            assert torch.equal(a[k], b[k]), k
