"""Prologue and drain of the software-pipelined wgmma tile loop (csrc/x2h_tc.cu): every CTA issues tile 0 before its loop
and finishes its last tile without a successor, so the short loops are the edge cases.  X2H and H2X through the C ABI at
exactly 1, 2 and 3 tiles per CTA, fewer tiles than SMs, node counts that are not a multiple of the 4-node tile, and a
pruned sampling step whose device-side node list is shorter than the host count; against the fp32 SIMT kernels at the
suite's bars, and repeated runs bit-identical."""
import ctypes as C

import numpy as np
import pytest
import torch

from cbgbench_b200 import _lib, synthetic
from helpers import assert_close, composed_inputs, make_model, rel_err

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


def dev():
    return torch.device('cuda:0')


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def tiles_per_cta(n_rows):
    """Tiles of CTA 0 (the most loaded one) for a launch over n_rows listed nodes: grid = min(tiles, SMs)."""
    tiles = (n_rows + 3) // 4
    return -(-tiles // min(tiles, sms()))


def split(total, parts):
    return [total // parts + (1 if g < total % parts else 0) for g in range(parts)]


def batch_for(n_nodes, n_gen, seed):
    """De-novo batch with n_nodes atoms of which n_gen are generated (ligand), graphs of at most ~400 atoms."""
    graphs = max(1, -(-n_nodes // 400))
    return synthetic.make_batch(split(n_nodes - n_gen, graphs), split(n_gen, graphs), seed=seed, gen_mode='denovo')


@pytest.fixture
def edge_impl_reset():
    yield
    _lib.check(_lib.lib().cbg_set_edge_impl(_lib.DEFAULT_EDGE_IMPL, 0))


# (id, (n_nodes, n_gen) as a function of the SM count S, tiles of CTA 0 in the X2H launches, in the H2X launches);
# X2H runs over all n_nodes, H2X over the n_gen generated atoms
CASES = [
    ('x2h1_h2x_fewer_than_sms', lambda S: (4 * S, 30), 1, 1),
    ('x2h2_h2x1', lambda S: (8 * S, 4 * S), 2, 1),
    ('x2h3_h2x2_ragged', lambda S: (12 * S - 1, 8 * S - 3), 3, 2),
    ('x2h_fewer_than_sms_ragged', lambda S: (161, 13), 1, 1),
    ('x2h4_h2x3_ragged', lambda S: (16 * S, 12 * S - 1), 4, 3),
]


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_short_tile_loops_match_simt(case, edge_impl_reset):
    name, sizes, x2h_tiles, h2x_tiles = case
    n_nodes, n_gen = sizes(sms())
    assert (tiles_per_cta(n_nodes), tiles_per_cta(n_gen)) == (x2h_tiles, h2x_tiles)
    if 'fewer' in name:
        assert (min(n_nodes, n_gen) + 3) // 4 < sms()
    L = _lib.lib()
    model, sd = make_model(10, device=dev(), num_layers=2)
    x, h, bidx, lig, gen = composed_inputs(sd, batch_for(n_nodes, n_gen, seed=300 + n_nodes))
    assert x.shape[0] == n_nodes and int(gen.sum()) == n_gen
    args = [t.to(dev()) for t in (x, h, bidx, lig, gen)]
    outs = {}
    for impl in (0, 6):
        _lib.check(L.cbg_set_edge_impl(impl, 0))
        outs[impl] = [[t.cpu() for t in model.denoiser(*args, stop_after_layers=s)] for s in (1, -1)]
    again = [t.cpu() for t in model.denoiser(*args)]
    for stop, (tc, simt) in zip(('1 layer', 'all layers'), zip(outs[6], outs[0])):
        moved = float((tc[0] - x).abs().max())
        assert moved > 1e-3, f'{name}: H2X moved nothing'
        for a, b, k in zip(tc, simt, 'xhc'):
            assert torch.isfinite(a).all(), (name, stop, k)
            assert rel_err(a, b) < 1e-4, (name, stop, k, rel_err(a, b))
            assert_close(a, b, what=f'{name} {stop} {k}')
    for a, b in zip(again, outs[6][1]):
        assert torch.equal(a, b), name


def test_pruned_sampling_short_device_list_matches_simt(edge_impl_reset):
    """Receptive-field pruning: layer l's X2H launches are sized for the host node count but read a device-side list
    length that shrinks from layer to layer, so most CTAs of the late layers find 0, 1 or 2 tiles (or none at all) in
    a grid sized for many more.  Eager and graph-replayed sampling, against the SIMT kernels and bit-identical on repeat."""
    T = 4
    L = _lib.lib()
    model, sd = make_model(T, device=dev())
    batch = synthetic.make_batch([300] * 6 + [120], [24] * 6 + [10], seed=515, gen_mode='denovo')
    n_lig = int(batch['ligand_pos'].shape[0])
    pn, tu = synthetic.make_noise(T, n_lig, 13, seed=23)
    states = []
    prepare = model.prepare

    def keep_state(*a, **k):
        states.append(prepare(*a, **k))
        return states[-1]
    model.prepare = keep_state
    res = {}
    for impl, use_graph, tag in ((0, False, 'simt'), (6, False, 'eager'), (6, True, 'graph'), (6, True, 'graph_repeat')):
        _lib.check(L.cbg_set_edge_impl(impl, 0))
        model.use_graph = use_graph
        res[tag] = model.sample(batch, pos_noise=pn, type_uniform=tu)
    plan = states[-1]['plan']
    counts = np.zeros(plan.num_layers + 1, dtype=np.int32)
    _lib.check(L.cbg_sample_prune_counts_host(C.byref(plan), counts.ctypes.data, _lib.stream_ptr(dev())))
    n_nodes = states[-1]['n_nodes']
    # the last layers' lists are far shorter than the host count: fewer tiles than SMs for the late launches
    assert counts[plan.num_layers] < n_nodes and (counts[plan.num_layers] + 3) // 4 < sms(), (counts, n_nodes)
    for t in range(-1, T):
        for tag in ('eager', 'graph'):
            assert torch.equal(res[tag][t][1].cpu().argmax(-1), res['simt'][t][1].cpu().argmax(-1)), (tag, t)
            assert_close(res[tag][t][0].cpu(), res['simt'][t][0].cpu(), what=f'{tag} step {t}')
        for i in (0, 1):
            assert torch.equal(res['graph_repeat'][t][i], res['graph'][t][i]), t
            assert torch.equal(res['eager'][t][i], res['graph'][t][i]), t
