"""wgmma X2H tile kernels (csrc/x2h_tc.cu, edge impl 6): operand-convention self-test on the hardware, parity against the
reference goldens / the fp32 SIMT kernels / the oracle, on the forward and on the sampling path."""
import numpy as np
import pytest
import torch

from cbgbench_b200 import _lib, synthetic
from helpers import FORWARD_CASES, composed_inputs, golden, make_model, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4
torch.set_grad_enabled(False)


def dev():
    return torch.device('cuda:0')


@pytest.fixture
def edge_impl_reset():
    yield
    _lib.check(_lib.lib().cbg_set_edge_impl(_lib.DEFAULT_EDGE_IMPL, 0))


@pytest.mark.parametrize('a_from_smem', [1, 0], ids=['A_smem', 'A_regs'])
def test_wgmma_f16_operand_conventions(a_from_smem):
    """D = A B^T with f16 operands on wgmma: B in the canonical K-major shared-memory layout, A from shared memory or
    from registers (the accumulator-compatible fragment layout), fp32 accumulator fragment stored row by row."""
    rs = np.random.RandomState(5 + a_from_smem)
    a = rs.normal(size=(128, 32)).astype(np.float16)
    b = rs.normal(size=(128, 32)).astype(np.float16)
    ad, bd = torch.from_numpy(a).to(dev()), torch.from_numpy(b).to(dev())
    d = torch.full((128, 128), float('nan'), device=dev())
    _lib.check(_lib.lib().cbg_selftest_umma_f16(ad.data_ptr(), bd.data_ptr(), d.data_ptr(), a_from_smem, None))
    torch.cuda.synchronize()
    want = a.astype(np.float64) @ b.astype(np.float64).T
    err = np.abs(d.cpu().numpy().astype(np.float64) - want).max()
    assert err < 1e-4, f'max abs err {err:.3e}'


@pytest.mark.parametrize('case', FORWARD_CASES, ids=[c[0] for c in FORWARD_CASES])
def test_forward_tcgen05_matches_golden_and_simt(case, edge_impl_reset):
    name, n_prot, n_lig, seed, gen_mode, enc = case
    gold = golden('forward_cases.npz')
    model, sd = make_model(10, device=dev(), **enc)
    batch = synthetic.make_batch(n_prot, n_lig, seed=seed, gen_mode=gen_mode)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    args = [t.to(dev()) for t in (x, h, bidx, lig, gen)]
    L = _lib.lib()
    outs = {}
    for impl in (0, 6):
        _lib.check(L.cbg_set_edge_impl(impl, 0))
        h1 = model.denoiser(*args, stop_after_layers=1)[1].cpu()
        outs[impl] = (h1,) + tuple(t.cpu() for t in model.denoiser(*args))
    d1 = rel_err(outs[6][0], outs[0][0])
    report = f'{name}: h after 1 layer vs simt {d1:.2e}; ' + ', '.join(
        f'{k} vs golden {rel_err(outs[6][i + 1], gold[name + "/" + k]):.2e}' for i, k in enumerate(('x', 'h', 'c')))
    print(report)
    assert torch.isfinite(outs[6][3]).all(), report
    assert d1 < 1e-5, report
    for i, k in enumerate(('x', 'h', 'c')):
        assert rel_err(outs[6][i + 1], gold[f'{name}/{k}']) < TOL, report
    assert torch.equal(outs[6][1][~gen], x[~gen])


def test_forward_tcgen05_layer_by_layer_vs_oracle(edge_impl_reset):
    from oracle import denoiser as ODn
    _lib.check(_lib.lib().cbg_set_edge_impl(6, 0))
    model, sd = make_model(10, device=dev())
    batch = synthetic.make_batch([200, 40, 20, 3], [24, 10, 5, 2], seed=12)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    xo, ho, co, trace = ODn.unitransformer_forward(sd, x, h, bidx, lig, gen, return_trace=True)
    args = [t.to(dev()) for t in (x, h, bidx, lig, gen)]
    for L_ in range(1, 10):
        xg, hg, cg = model.denoiser(*args, stop_after_layers=L_)
        ex, eh = rel_err(xg.cpu(), trace['x'][L_ - 1]), rel_err(hg.cpu(), trace['h'][L_ - 1])
        assert ex < TOL and eh < TOL, f'layer {L_}: x {ex:.2e} h {eh:.2e}'


def test_sampling_path_tcgen05_matches_simt(edge_impl_reset):
    """Sampling path (static lists, pruning): atom types identical, coordinates equal to rounding, at every step."""
    T = 6
    L = _lib.lib()
    for gen_mode, sizes in (('denovo', ([140, 60, 20], [20, 9, 5])), ('partial', ([90, 70], [18, 12]))):
        model, sd = make_model(T, device=dev())
        batch = synthetic.make_batch(*sizes, seed=131, gen_mode=gen_mode)
        n_lig = int(batch['ligand_pos'].shape[0])
        pn, tu = synthetic.make_noise(T, n_lig, 13, seed=19)
        res = {}
        for impl in (0, 6):
            _lib.check(L.cbg_set_edge_impl(impl, 0))
            res[impl] = model.sample(batch, pos_noise=pn, type_uniform=tu)
        for t in range(-1, T):
            assert torch.equal(res[0][t][1].cpu().argmax(-1), res[6][t][1].cpu().argmax(-1)), (gen_mode, t)
            e = rel_err(res[6][t][0].cpu(), res[0][t][0].cpu())
            assert e < 1e-5, (gen_mode, t, e)


def test_tcgen05_many_tiles_per_cta_and_ragged_tail(edge_impl_reset):
    """More tiles than SMs (every CTA loops over several tiles) and a node count that is not a multiple of the 4-node
    tile: forward against the SIMT kernels."""
    L = _lib.lib()
    model, sd = make_model(10, device=dev(), num_layers=2)
    sizes = [300] * 9 + [37]
    batch = synthetic.make_batch(sizes, [24] * 9 + [6], seed=77)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    assert x.shape[0] % 4 != 0 and x.shape[0] // 4 > 3 * 132
    args = [t.to(dev()) for t in (x, h, bidx, lig, gen)]
    outs = {}
    for impl in (0, 6):
        _lib.check(L.cbg_set_edge_impl(impl, 0))
        outs[impl] = [t.cpu() for t in model.denoiser(*args)]
    for a, b, k in zip(outs[6], outs[0], 'xhc'):
        assert rel_err(a, b) < 1e-5, (k, rel_err(a, b))


@pytest.mark.parametrize('gen_mode', ['denovo', 'partial'])
def test_h2x_tcgen05_matches_simt(gen_mode, edge_impl_reset):
    """H2X on the tile kernel (attention weights into the compact buffer, then the 16-output value head + coordinate
    update): coordinates after 1, 2 and all layers against the fp32 SIMT h2x_kernel.  > 4 * 132 generated atoms (every
    CTA loops) and a count that is not a multiple of the 4-node tile."""
    L = _lib.lib()
    model, sd = make_model(10, device=dev(), num_layers=3)
    n_graphs = 31
    batch = synthetic.make_batch([60 + 3 * g for g in range(n_graphs)], [24 if g else 23 for g in range(n_graphs)],
                                 seed=405, gen_mode=gen_mode)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    n_gen = int(gen.sum())
    if gen_mode == 'denovo':
        assert n_gen > 4 * 132 and n_gen % 4 != 0
    args = [t.to(dev()) for t in (x, h, bidx, lig, gen)]
    outs = {}
    for impl in (0, 6):
        _lib.check(L.cbg_set_edge_impl(impl, 0))
        outs[impl] = [model.denoiser(*args, stop_after_layers=s)[0].cpu() for s in (1, 2, -1)]
    for a, b, s in zip(outs[6], outs[0], (1, 2, 3)):
        moved = (a - x).abs().max()
        assert float(moved) > 1e-3, 'H2X moved nothing'
        assert torch.equal(a[~gen], x[~gen])
        assert rel_err(a, b) < 1e-5, (s, rel_err(a, b))
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-5), s


def test_tcgen05_repeated_runs_are_bit_identical(edge_impl_reset):
    """The G rows and the per-node partial results are handed between the warps of a warpgroup through shared memory and
    named barriers, and every sum has a fixed order: a lost hand-over would show up as run-to-run differences.
    Config-2-sized forward (every CTA loops ~40 times), 8 repeats, outputs must be bit-identical."""
    model, sd = make_model(10, device=dev(), num_layers=3)
    batch = synthetic.make_batch([300] * 64, [24] * 64, seed=2024)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    args = [t.to(dev()) for t in (x, h, bidx, lig, gen)]
    first = [t.clone() for t in model.denoiser(*args)]
    for _ in range(7):
        again = model.denoiser(*args)
        for a, b in zip(first, again):
            assert torch.equal(a, b)
