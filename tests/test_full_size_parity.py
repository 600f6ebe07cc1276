"""Parity AT the BASELINE.json shapes: the CUDA path against the oracle on every graph of a full-size batch (config 2:
64 x (300 + 24) atoms; config 3: 128 pockets, radius graph r = 10, partial generation; config 5: ragged 100-800-atom
pockets), config 1 against a T = 50 trajectory of the live reference, and a long free-running trajectory.

The oracle is the as-written [E, 340] formulation on the host CPU, so these tests take a few minutes
(one oracle forward of config 2 is ~10-30 s); they are what the smaller-shape tests of test_gpu_parity.py cannot show:
300-atom graphs, 128-graph batches and 800-atom graphs compared element by element.
"""
import os

import numpy as np
import pytest
import torch

from cbgbench_b200 import synthetic
from helpers import assert_close, composed_inputs, golden, make_model, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4
torch.set_grad_enabled(False)


def dev():
    return torch.device('cuda:0')


@pytest.fixture(autouse=True)
def _oracle_threads():
    old = torch.get_num_threads()
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    yield
    torch.set_num_threads(old)


def _check_sample_against_oracle(model, sd, batch, T, steps, enc=None, seed=3):
    """`steps` sampling steps of the product (R-cache / static lists / pruning as shipped) against the oracle with the
    same injected noise: atom types bit-exact, coordinates element-wise and in the max norm, for ALL graphs."""
    from oracle import diffusion as OD
    enc = enc or {}
    n_lig = int(batch['ligand_pos'].shape[0])
    pn, tu = synthetic.make_noise(T, n_lig, 13, seed=seed)
    traj = model.sample(batch, pos_noise=pn, type_uniform=tu, num_steps=steps)
    want = OD.sample(sd, batch, T, pn, tu, stop_after=steps, k=enc.get('k', 32),
                     cutoff_mode=enc.get('cutoff_mode', 'knn'), r_max=enc.get('r_max', 10.0))
    fixed = ~batch.get('ligand_gen_flag', batch['ligand_lig_flag'])
    for t in range(T - 1 - steps, T - 1):
        xg, cg = traj[t][0].cpu(), traj[t][1].cpu()
        xo, co = want[t]
        assert torch.equal(cg.argmax(-1), co.argmax(-1)), f't={t}: atom types differ'
        assert rel_err(xg, xo) < TOL, f't={t}: {rel_err(xg, xo):.2e}'
        assert_close(xg, xo, rtol=1e-4, atol=1e-5, what=f'coordinates t={t}')
        assert torch.equal(xg[fixed], batch['ligand_pos'][fixed])


def test_config2_full_batch_forward_and_sampling_vs_oracle():
    """config 2: 64 pockets x (300 protein + 24 ligand atoms), every graph: one denoiser forward (x, h, logits) and two
    sampling steps."""
    from oracle import denoiser as ODn
    T = 1000
    model, sd = make_model(T, device=dev())
    batch = synthetic.make_batch([300] * 64, [24] * 64, seed=2024)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    xo, ho, co = ODn.unitransformer_forward(sd, x, h, bidx, lig, gen)
    d = dev()
    xg, hg, cg = (t.cpu() for t in model.denoiser(x.to(d), h.to(d), bidx.to(d), lig.to(d), gen.to(d)))
    for name, a, b in (('x', xg, xo), ('h', hg, ho), ('c', cg, co)):
        assert rel_err(a, b) < TOL, f'{name}: {rel_err(a, b):.2e}'
    assert_close(xg, xo, rtol=1e-4, atol=1e-5, what='x')
    assert_close(hg, ho, rtol=1e-4, atol=1e-4, what='h')          # |h| ~ 10: atol scaled to the tensor
    assert_close(cg[lig], co[lig], rtol=1e-4, atol=1e-4, what='ligand logits')
    assert torch.equal(cg[lig].argmax(-1), co[lig].argmax(-1))
    _check_sample_against_oracle(model, sd, batch, T, steps=2)


def test_config3_radius_linker_batch_sampling_vs_oracle():
    """config 3: 128 pockets, radius graph r = 10 A (cap 32), partial generation (linker-style fixed context), sampling
    path with static lists, cached terms and pruning on."""
    T = 1000
    enc = {'cutoff_mode': 'radius', 'r_max': 10.0}
    model, sd = make_model(T, device=dev(), **enc)
    batch = synthetic.make_batch([300] * 128, [24] * 128, seed=2024, gen_mode='partial')
    _check_sample_against_oracle(model, sd, batch, T, steps=2, enc=enc)


def test_config5_ragged_scaffold_batch_all_graphs_vs_oracle():
    """config 5: ragged pockets of 100 ... 800 atoms (both extremes present), partial generation, every graph compared."""
    T = 1000
    rs = np.random.RandomState(77)
    n_prot = [int(v) for v in rs.randint(100, 801, size=16)]
    n_prot[3], n_prot[11] = 800, 100
    model, sd = make_model(T, device=dev())
    batch = synthetic.make_batch(n_prot, [24] * 16, seed=2029, gen_mode='partial')
    _check_sample_against_oracle(model, sd, batch, T, steps=2)


def test_config1_T50_trajectory_matches_live_reference_golden():
    """config 1: one pocket (200 + 24 atoms), 50 denoise steps: every state of the UNMODIFIED reference's
    TargetDiff.sample (tests/golden/make_golden_c1.py) - atom types bit-exact, coordinates within tolerance."""
    g = golden('trajectory_c1_T50.npz')
    T = 50
    model, sd = make_model(T, device=dev())
    batch = synthetic.make_batch([200], [24], seed=2024)
    pn, tu = synthetic.make_noise(T, 24, 13, seed=31)
    traj = model.sample(batch, pos_noise=pn, type_uniform=tu)
    worst = 0.0
    for t in range(-1, T):
        assert np.array_equal(traj[t][1].cpu().argmax(-1).numpy(), g[f'v{t}'].astype(np.int64)), f't={t}'
        worst = max(worst, rel_err(traj[t][0].cpu(), g[f'x{t}']))
        assert_close(traj[t][0].cpu(), g[f'x{t}'], rtol=1e-4, atol=1e-5, what=f'x t={t}')
    assert worst < TOL, worst


def test_long_free_running_trajectory_vs_oracle():
    """300 denoise steps of a T = 1000 schedule on two small pockets with the same injected noise on both sides.  Sampling
    is contractive in the coordinates (posterior mean pulls towards the prediction), so the trajectories must stay
    together: atom types equal at (almost) every (step, atom) - a Gumbel arg-max may flip on a ~1e-6 near-tie and the
    flipped atom then lives its own life - and statistics of the final state (type histogram, per-graph radius of
    gyration) must agree."""
    from oracle import diffusion as OD
    T, steps = 1000, 300
    model, sd = make_model(T, device=dev())
    batch = synthetic.make_batch([60, 45], [12, 9], seed=55)
    n_lig = 21
    pn, tu = synthetic.make_noise(T, n_lig, 13, seed=41)
    traj = model.sample(batch, pos_noise=pn, type_uniform=tu, num_steps=steps)
    want = OD.sample(sd, batch, T, pn, tu, stop_after=steps)
    same, total, first_flip = 0, 0, None
    for t in range(T - 1 - steps, T - 1):
        vg, vo = traj[t][1].cpu().argmax(-1), want[t][1].argmax(-1)
        same += int((vg == vo).sum())
        total += n_lig
        if first_flip is None and not torch.equal(vg, vo):
            first_flip = t
    t_end = T - 1 - steps
    xg, xo = traj[t_end][0].cpu(), want[t_end][0]
    assert same >= 0.98 * total, (same, total, first_flip)
    if first_flip is None:                                  # no near-tie met: the whole trajectory is comparable
        assert rel_err(xg, xo) < 1e-3, rel_err(xg, xo)
    bl = batch['ligand_element_batch']
    for gsel in (0, 1):
        m = bl == gsel
        rg = lambda x: float((x[m] - x[m].mean(0)).pow(2).sum(-1).mean().sqrt())
        assert abs(rg(xg) - rg(xo)) < 0.05 * rg(xo) + 1e-3, (gsel, rg(xg), rg(xo))
    hg = torch.bincount(traj[t_end][1].cpu().argmax(-1), minlength=13)
    ho = torch.bincount(want[t_end][1].argmax(-1), minlength=13)
    assert int((hg - ho).abs().sum()) <= 2, (hg.tolist(), ho.tolist())
