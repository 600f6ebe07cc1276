"""Parity of the CUDA path (through the C-ABI) against the oracle and the reference goldens.

Bars (BASELINE.json north_star): coordinates / logits within 1e-4 relative fp32
(max|a-b| / max|b|), integer outputs (neighbour lists, atom-type argmax) bit-exact.
Run on an H100:  python -m pytest tests -m gpu
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cbgbench_b200 import _lib, synthetic
from helpers import FORWARD_CASES, composed_inputs, golden, make_model, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4          # relative fp32 tolerance of the parity bar
torch.set_grad_enabled(False)


def dev():
    return torch.device('cuda:0')


def _ws(n_nodes, n_gen=0):
    L = _lib.lib()
    nbytes = L.cbg_workspace_bytes(n_nodes, n_gen)
    buf = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev())
    off = (-buf.data_ptr()) % 256
    return buf, buf.data_ptr() + off, nbytes


def _gptr(batch_idx):
    counts = torch.bincount(batch_idx)
    ptr = torch.zeros(counts.numel() + 1, dtype=torch.int32)
    ptr[1:] = torch.cumsum(counts, 0)
    return ptr.to(dev()), int(counts.numel()), int(counts.max())


def cuda_neighbors(x, batch_idx, k=32, mode=0, r_max=10.0):
    L = _lib.lib()
    N = x.shape[0]
    gptr, B, max_n = _gptr(batch_idx)
    xd = x.to(dev()).contiguous()
    nbr = torch.empty((N, 32), dtype=torch.int32, device=dev())
    buf, wsp, wsb = _ws(N)
    _lib.check(L.cbg_build_neighbors_f32(xd.data_ptr(), gptr.data_ptr(), B, N, max_n, mode, k, r_max,
                                         nbr.data_ptr(), wsp, wsb, None))
    torch.cuda.synchronize()
    return nbr.cpu().long()


# ---------------------------------------------------------------------------------------------
# stage: neighbour lists (bit-exact)
# A graph above 3 072 atoms (48 KB of float4 coordinates) needs the kNN kernel's opt-in dynamic shared memory.
LARGE_GRAPH_BATCH = [3500, 40, 7]


@pytest.mark.parametrize('sizes', [[224], [299, 25, 1, 2, 33, 32], [850, 100, 450], LARGE_GRAPH_BATCH])
@pytest.mark.parametrize('k', [32, 8])
def test_knn_bit_exact(sizes, k):
    from oracle import graph_ops as G
    rs = np.random.RandomState(sum(sizes) + k)
    x = torch.from_numpy((4.0 * rs.normal(size=(sum(sizes), 3))).astype(np.float32))
    x[5] = x[3]                                  # exact duplicate -> distance ties
    bidx = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
    ptr = [0] + list(np.cumsum(sizes))
    want = G.neighbor_table(x, ptr, k=k)
    got = cuda_neighbors(x, bidx, k=k)
    assert torch.equal(got, want)


def test_radius_graph_bit_exact():
    from oracle import graph_ops as G
    for sizes in ([300, 120], LARGE_GRAPH_BATCH):
        rs = np.random.RandomState(9)
        x = torch.from_numpy((6.0 * rs.normal(size=(sum(sizes), 3))).astype(np.float32))
        bidx = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
        want = G.neighbor_table(x, [0] + list(np.cumsum(sizes)), k=32, r_max=6.0)
        got = cuda_neighbors(x, bidx, k=32, mode=1, r_max=6.0)
        assert torch.equal(got, want), sizes
        assert (want == -1).any() and (want[:, 0] >= 0).any(), sizes


def test_knn_rejects_graph_over_shared_memory_limit():
    """The neighbour search holds one graph's coordinates in shared memory (200 KB, 12 800 atoms): a larger graph is
    refused on the host with an error, before any launch."""
    L = _lib.lib()
    sizes = [12801, 5]
    N = sum(sizes)
    x = torch.zeros((N, 3), dtype=torch.float32, device=dev())
    gptr = torch.tensor([0, sizes[0], N], dtype=torch.int32, device=dev())
    nbr = torch.full((N, 32), -7, dtype=torch.int32, device=dev())
    buf, wsp, wsb = _ws(N)
    rc = L.cbg_build_neighbors_f32(x.data_ptr(), gptr.data_ptr(), 2, N, max(sizes), 0, 32, 10.0, nbr.data_ptr(), wsp, wsb, None)
    torch.cuda.synchronize()
    assert rc != 0
    assert b'12801 atoms exceeds the 12800-atom shared-memory limit' in L.cbg_last_error()
    assert bool((nbr == -7).all())                     # nothing was written


# ---------------------------------------------------------------------------------------------
# stage: edge gate
def test_edge_gate_matches_oracle():
    from oracle import denoiser as ODn, graph_ops as G
    model, sd = make_model(10)
    batch = synthetic.make_batch([200, 40], [24, 10], seed=3)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    ptr = G.graph_ptr_from_batch(bidx)
    nbr = G.neighbor_table(x, ptr, k=32)
    ei = G.table_to_edge_index(nbr)
    # float64 reference: independent of the host CPU's fp32 GEMM code path
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    want = torch.zeros(nbr.shape, dtype=torch.float64)
    want[nbr >= 0] = ODn.edge_gate(sd64, 'denoiser.', x.double(), ei[0], ei[1]).flatten()
    L = _lib.lib()
    blob = model.denoiser.packed_blob(dev())
    N = x.shape[0]
    ew = torch.empty((N, 32), dtype=torch.float32, device=dev())
    buf, wsp, wsb = _ws(N)
    xd = x.to(dev()).contiguous()                       # keep references alive across the call
    nd = nbr.to(dev(), torch.int32).contiguous()
    _lib.check(L.cbg_edge_gate_f32(blob.data_ptr(), xd.data_ptr(), nd.data_ptr(), N, ew.data_ptr(), wsp, wsb, None))
    torch.cuda.synchronize()
    err = rel_err(ew.cpu(), want)
    assert err < 5e-6, f'edge gate rel err {err:.3e}'


# ---------------------------------------------------------------------------------------------
# full forward: per-layer trace against the oracle, then the reference goldens
def test_forward_layer_by_layer_vs_oracle():
    from oracle import denoiser as ODn
    model, sd = make_model(10, device=dev())
    batch = synthetic.make_batch([200, 40, 20], [24, 10, 5], seed=11)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    xo, ho, co, trace = ODn.unitransformer_forward(sd, x, h, bidx, lig, gen, return_trace=True)
    args = [t.to(dev()) for t in (x, h, bidx, lig, gen)]
    for L_ in range(1, 10):
        xg, hg, cg = model.denoiser(*args, stop_after_layers=L_)
        ex, eh = rel_err(xg.cpu(), trace['x'][L_ - 1]), rel_err(hg.cpu(), trace['h'][L_ - 1])
        assert ex < TOL and eh < TOL, f'layer {L_}: x {ex:.2e} h {eh:.2e}'
    xg, hg, cg = model.denoiser(*args)
    assert rel_err(xg.cpu(), xo) < TOL and rel_err(hg.cpu(), ho) < TOL and rel_err(cg.cpu(), co) < TOL
    # the inputs must not be modified (reference clones x, unitransformer.py:178)
    assert torch.equal(args[0].cpu(), x) and torch.equal(args[1].cpu(), h)


@pytest.mark.parametrize('case', FORWARD_CASES, ids=[c[0] for c in FORWARD_CASES])
def test_forward_matches_reference_golden(case):
    name, n_prot, n_lig, seed, gen_mode, enc = case
    gold = golden('forward_cases.npz')
    model, sd = make_model(10, device=dev(), **enc)
    batch = synthetic.make_batch(n_prot, n_lig, seed=seed, gen_mode=gen_mode)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    xg, hg, cg = model.denoiser(x.to(dev()), h.to(dev()), bidx.to(dev()), lig.to(dev()), gen.to(dev()))
    ex, eh, ec = (rel_err(a.cpu(), gold[f'{name}/{k}']) for a, k in ((xg, 'x'), (hg, 'h'), (cg, 'c')))
    assert ex < TOL and eh < TOL and ec < TOL, f'{name}: x {ex:.2e} h {eh:.2e} c {ec:.2e}'
    # atoms with gen_flag == False never move (unitransformer.py:182)
    assert torch.equal(xg.cpu()[~gen], x[~gen])
    # element-wise closeness of the moved coordinates as well
    assert torch.allclose(xg.cpu(), torch.from_numpy(gold[f'{name}/x']), rtol=1e-4, atol=1e-4)


def test_forward_radius_mode_vs_oracle():
    from oracle import denoiser as ODn
    model, sd = make_model(10, device=dev(), cutoff_mode='radius', r_max=9.0)
    batch = synthetic.make_batch([150, 80], [20, 12], seed=31)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    xo, ho, co = ODn.unitransformer_forward(sd, x, h, bidx, lig, gen, cutoff_mode='radius', r_max=9.0)
    xg, hg, cg = model.denoiser(x.to(dev()), h.to(dev()), bidx.to(dev()), lig.to(dev()), gen.to(dev()))
    assert rel_err(xg.cpu(), xo) < TOL and rel_err(hg.cpu(), ho) < TOL and rel_err(cg.cpu(), co) < TOL


@pytest.mark.parametrize('enc', [{}, {'cutoff_mode': 'radius', 'r_max': 9.0}], ids=['knn', 'radius9'])
def test_forward_with_large_graph_vs_oracle(enc):
    """A 2-layer forward on a batch with one 3 500-atom pocket (the neighbour search's opt-in shared-memory path)."""
    from oracle import denoiser as ODn
    model, sd = make_model(10, device=dev(), num_layers=2, **enc)
    batch = synthetic.make_batch([3476, 60], [24, 12], seed=33)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    assert int(torch.bincount(bidx).max()) == 3500
    xo, ho, co = ODn.unitransformer_forward(sd, x, h, bidx, lig, gen, cutoff_mode=enc.get('cutoff_mode', 'knn'),
                                            r_max=enc.get('r_max', 10.0))
    xg, hg, cg = model.denoiser(x.to(dev()), h.to(dev()), bidx.to(dev()), lig.to(dev()), gen.to(dev()))
    for name, a, b in (('x', xg, xo), ('h', hg, ho), ('c', cg, co)):
        err = rel_err(a.cpu(), b)
        assert err < TOL, f'{name}: rel err {err:.2e}'
    assert torch.equal(xg.cpu()[~gen], x[~gen])


def test_forward_host_buffers_equals_device_path():
    model, sd = make_model(10, device=dev())
    batch = synthetic.make_batch([120, 60], [16, 8], seed=41)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    xd, hd, cd = model.denoiser(x.to(dev()), h.to(dev()), bidx.to(dev()), lig.to(dev()), gen.to(dev()))
    xh, hh, ch = model.denoiser.forward_host(x, h, bidx, lig, gen)
    assert not xh.is_cuda
    assert torch.equal(xh, xd.cpu()) and torch.equal(hh, hd.cpu()) and torch.equal(ch, cd.cpu())


def test_cpu_tensors_are_rejected_not_silently_computed():
    model, sd = make_model(10)
    batch = synthetic.make_batch([30], [6], seed=1)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    with pytest.raises(RuntimeError):
        model.denoiser(x, h, bidx, lig, gen)


# ---------------------------------------------------------------------------------------------
# properties (size independent)
def _rand_rotation(rs):
    q, _ = np.linalg.qr(rs.normal(size=(3, 3)))
    if np.linalg.det(q) < 0:
        q[:, 0] = -q[:, 0]
    return torch.from_numpy(q.astype(np.float32))


def test_e3_equivariance_and_batch_independence():
    model, sd = make_model(10, device=dev())
    batch = synthetic.make_batch([180, 90, 60], [20, 12, 7], seed=51)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    d = dev()
    x1, h1, c1 = model.denoiser(x.to(d), h.to(d), bidx.to(d), lig.to(d), gen.to(d))
    rs = np.random.RandomState(4)
    R, tvec = _rand_rotation(rs), torch.tensor([3.0, -2.0, 5.0])
    xr = x @ R.T + tvec
    x2, h2, c2 = model.denoiser(xr.to(d), h.to(d), bidx.to(d), lig.to(d), gen.to(d))
    # rotated/translated input -> rotated/translated coordinates, invariant features/logits
    # (kNN selection may flip on near-ties after rotation, hence 1e-3 rather than 1e-4)
    assert rel_err(x2.cpu(), x1.cpu() @ R.T + tvec) < 1e-3
    assert rel_err(h2.cpu(), h1.cpu()) < 1e-3 and rel_err(c2.cpu(), c1.cpu()) < 1e-3
    # graphs are independent: running graph 1 alone reproduces its rows bit-for-bit
    m = bidx == 1
    xa, ha, ca = model.denoiser(x[m].to(d), h[m].to(d), torch.zeros(int(m.sum()), dtype=torch.long, device=d),
                                lig[m].to(d), gen[m].to(d))
    assert torch.equal(xa.cpu(), x1.cpu()[m]) and torch.equal(ha.cpu(), h1.cpu()[m]) and torch.equal(ca.cpu(), c1.cpu()[m])


def test_forward_is_deterministic():
    model, sd = make_model(10, device=dev())
    batch = synthetic.make_batch([300] * 4, [24] * 4, seed=61)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    d = dev()
    a = model.denoiser(x.to(d), h.to(d), bidx.to(d), lig.to(d), gen.to(d))
    b = model.denoiser(x.to(d), h.to(d), bidx.to(d), lig.to(d), gen.to(d))
    for u, v in zip(a, b):
        assert torch.equal(u, v)


# ---------------------------------------------------------------------------------------------
# reverse step and sampling loop
def test_reverse_step_matches_reference_golden():
    g = golden('reverse_step.npz')
    model, sd = make_model(1000, device=dev())
    L = _lib.lib()
    d = dev()
    n, K = g['x0'].shape[0], 13
    td = lambda k, dt=torch.float32: torch.from_numpy(g[k]).to(d, dt).contiguous()
    x0, xt, logits, ct, noise, uni = td('x0'), td('xt'), td('logits'), td('ct'), td('noise'), td('uni')
    gen = td('gen', torch.uint8)
    for t in (0, 1, 500, 999):
        coef = model.step_coef(t)
        xn = torch.empty((n, 3), device=d)
        cn = torch.empty((n, K), device=d)
        vn = torch.empty(n, dtype=torch.int64, device=d)
        _lib.check(L.cbg_reverse_step_f32(C.byref(coef), x0.data_ptr(), logits.data_ptr(), xt.data_ptr(), ct.data_ptr(),
                                          gen.data_ptr(), noise.data_ptr(), uni.data_ptr(), n, K,
                                          xn.data_ptr(), cn.data_ptr(), vn.data_ptr(), None))
        torch.cuda.synchronize()
        assert np.array_equal(vn.cpu().numpy(), g[f't{t}/v_next']), t        # integer: bit-exact
        assert np.array_equal(cn.cpu().numpy(), g[f't{t}/c_next']), t
        assert rel_err(xn.cpu(), g[f't{t}/x_next']) < 1e-6, t


def test_short_trajectory_matches_reference_golden():
    """TargetDiff.sample over T=10 steps with the reference's injected noise: every step's
    atom types bit-exact, coordinates within tolerance."""
    g = golden('trajectory.npz')
    T = 10
    model, sd = make_model(T, device=dev())
    batch = synthetic.make_batch([150, 60], [20, 9], seed=21)
    pn, tu = synthetic.make_noise(T, 29, 13, seed=7)
    traj = model.sample(batch, pos_noise=pn, type_uniform=tu)
    assert sorted(traj.keys()) == list(range(-1, T))
    for t in range(-1, T):
        x, c, b = traj[t]
        assert (x.is_cuda, c.is_cuda) == ((t == -1), (t == -1))          # reference contract: >=0 on CPU
        assert np.array_equal(c.cpu().argmax(-1).numpy(), g[f'v{t}']), f't={t}'
        assert rel_err(x.cpu(), g[f'x{t}']) < TOL, f't={t}'
        assert torch.equal(b.cpu(), batch['ligand_element_batch'])
    assert model.last_launches > 0


def test_sample_partial_generation_keeps_context_fixed():
    from oracle import diffusion as OD
    T = 6
    model, sd = make_model(T, device=dev())
    batch = synthetic.make_batch([100, 70], [18, 12], seed=71, gen_mode='partial')
    pn, tu = synthetic.make_noise(T, 30, 13, seed=8)
    traj = model.sample(batch, pos_noise=pn, type_uniform=tu)
    want = OD.sample(sd, batch, T, pn, tu)
    fixed = ~batch['ligand_gen_flag']
    for t in range(-1, T):
        assert torch.equal(traj[t][0].cpu()[fixed], batch['ligand_pos'][fixed])
        assert torch.equal(traj[t][1].cpu().argmax(-1)[fixed], batch['ligand_atom_type'][fixed])
        assert torch.equal(traj[t][1].cpu().argmax(-1), want[t][1].argmax(-1)), t
        assert rel_err(traj[t][0].cpu(), want[t][0]) < TOL, t


def test_sample_with_torch_rng_is_seed_reproducible():
    T = 4
    model, sd = make_model(T, device=dev())
    batch = synthetic.make_batch([80], [10], seed=81)
    torch.manual_seed(2024)
    a = model.sample(batch)
    torch.manual_seed(2024)
    b = model.sample(batch, traj_mode='final')
    assert torch.equal(a[0][0], b[0][0]) and torch.equal(a[0][1], b[0][1])
    assert torch.equal(a[-1][0], b[-1][0])
    assert set(b.keys()) == {0, -1}


# ---------------------------------------------------------------------------------------------
# BASELINE.json full-size shapes: size-independent properties
def test_full_size_config2_properties():
    """config 2 shape (64 pockets x (300 + 24) atoms): finite outputs, fixed atoms never move,
    per-graph results identical to running one of the graphs alone (bit-for-bit)."""
    model, sd = make_model(10, device=dev())
    batch = synthetic.make_batch([300] * 64, [24] * 64, seed=2024)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    d = dev()
    xg, hg, cg = model.denoiser(x.to(d), h.to(d), bidx.to(d), lig.to(d), gen.to(d))
    assert torch.isfinite(xg).all() and torch.isfinite(hg).all() and torch.isfinite(cg).all()
    assert torch.equal(xg.cpu()[~gen], x[~gen])
    for gsel in (0, 37, 63):
        m = bidx == gsel
        xa, ha, ca = model.denoiser(x[m].to(d), h[m].to(d), torch.zeros(int(m.sum()), dtype=torch.long, device=d),
                                    lig[m].to(d), gen[m].to(d))
        assert torch.equal(xa.cpu(), xg.cpu()[m]) and torch.equal(ca.cpu(), cg.cpu()[m])


def test_ragged_config5_shape_vs_oracle_subset():
    """config 5 style ragged pockets (100..800 atoms): compare two of the graphs with the oracle."""
    from oracle import denoiser as ODn
    rs = np.random.RandomState(5)
    n_prot = [int(v) for v in rs.randint(100, 801, size=12)]
    n_prot[0], n_prot[1] = 800, 100
    model, sd = make_model(10, device=dev())
    batch = synthetic.make_batch(n_prot, [24] * 12, seed=91, gen_mode='partial')
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    d = dev()
    xg, hg, cg = model.denoiser(x.to(d), h.to(d), bidx.to(d), lig.to(d), gen.to(d))
    for gsel in (0, 1):
        m = bidx == gsel
        xo, ho, co = ODn.unitransformer_forward(sd, x[m], h[m], torch.zeros(int(m.sum()), dtype=torch.long), lig[m], gen[m])
        assert rel_err(xg.cpu()[m], xo) < TOL and rel_err(hg.cpu()[m], ho) < TOL and rel_err(cg.cpu()[m], co) < TOL


# ---------------------------------------------------------------------------------------------
# node projections: fp32 SIMT kernel and the wgmma (3xTF32, f16 split) kernels against a float64 reference
# (n_nodes, which rows): 'all' = rows 0..n-1 (row_idx NULL), 'sorted' / 'unsorted' = 150 listed rows, 'none' = n_rows 0.
# The wgmma kernels work in 64-row warpgroups of 128-row CTAs, so 64 / 65 / 128 / 129 rows sit on either side of a
# warpgroup and a CTA edge; 257 rows fill three CTAs, which leaves the last cluster of 2 or 4 CTAs partly padded.
NODE_PROJ_ROWS = {'n1': (1, 'all'), 'n64': (64, 'all'), 'n65': (65, 'all'), 'n128': (128, 'all'), 'n129': (129, 'all'),
                  'n257': (257, 'all'), 'n333': (333, 'all'), 'n333-sorted': (333, 'sorted'),
                  'n333-unsorted': (333, 'unsorted'), 'none': (64, 'none')}


@pytest.mark.parametrize('impl', [0, 1, 2, 11, 12, 14],
                         ids=['simt', 'wgmma-tf32', 'wgmma-f16', 'wgmma-tf32-cluster1', 'wgmma-tf32-cluster2',
                              'wgmma-tf32-cluster4'])
@pytest.mark.parametrize('sublayer', [0, 1], ids=['x2h', 'h2x'])
@pytest.mark.parametrize('rows', list(NODE_PROJ_ROWS))
def test_node_projections_match_float64(impl, sublayer, rows):
    model, sd = make_model(10, device=dev())
    L = _lib.lib()
    lay = _lib.blob_layout()
    blob = model.denoiser.packed_blob(dev())
    layer = 3
    rs = np.random.RandomState(17)
    N, kind = NODE_PROJ_ROWS[rows]
    h = torch.from_numpy((1.5 * rs.normal(size=(N, 128))).astype(np.float32))
    subset = rs.choice(N, size=150, replace=False) if kind in ('sorted', 'unsorted') else None
    row_idx = None
    if kind == 'sorted':
        row_idx = torch.from_numpy(np.sort(subset).astype(np.int32))
    elif kind == 'unsorted':
        row_idx = torch.from_numpy(subset.astype(np.int32))
        assert not bool((row_idx[1:] > row_idx[:-1]).all())
    hd = h.to(dev())
    base_ptr = blob.data_ptr() + 4 * (lay['global_floats'] + layer * lay['layer_floats'])
    pre = f'denoiser.blocks.{layer}.' + ('x2h_layers.0.' if sublayer == 0 else 'h2x_layers.0.')
    kn, vn, qn = ('hk_func', 'hv_func', 'hq_func') if sublayer == 0 else ('xk_func', 'xv_func', 'xq_func')
    d = lambda k: sd[pre + k].double()
    h64 = h.double()
    w0k, w0v = d(kn + '.net.0.weight'), d(vn + '.net.0.weight')
    want = [h64 @ w0k[:, 212:340].T, h64 @ w0v[:, 212:340].T,
            h64 @ w0k[:, 84:212].T + d(kn + '.net.0.bias'), h64 @ w0v[:, 84:212].T + d(vn + '.net.0.bias')]
    # the packer centres the first Linear of the edge MLPs (X2H and H2X) over the feature axis (exact: LayerNorm follows
    # it directly), so every plane comes out minus its row mean
    want = [w - w.mean(-1, keepdim=True) for w in want]
    qh = F.layer_norm(h64 @ d(qn + '.net.0.weight').T + d(qn + '.net.0.bias'), (128,), d(qn + '.net.1.weight'),
                      d(qn + '.net.1.bias'), 1e-5).relu()
    want.append((qh @ d(qn + '.net.3.weight').T + d(qn + '.net.3.bias')) / np.sqrt(8.0))
    planes = torch.full((5, N, 128), float('nan'), device=dev())
    ridx = row_idx.to(dev()) if row_idx is not None else None
    n_rows = 0 if kind == 'none' else (N if row_idx is None else int(row_idx.numel()))
    assert L.cbg_node_proj_f32(base_ptr, sublayer, impl, hd.data_ptr(), ridx.data_ptr() if ridx is not None else None,
                               n_rows, N, planes.data_ptr(), None) == 0, L.cbg_last_error()
    torch.cuda.synchronize()
    if kind == 'none':                                            # nothing to do: every plane stays untouched
        assert torch.isnan(planes.cpu()).all()
        return
    sel = slice(None) if row_idx is None else row_idx.long()
    for p in range(5):
        err = rel_err(planes[p].cpu()[sel], want[p][sel])
        assert err < 2e-6, f'impl {impl} sublayer {sublayer} plane {p}: rel err {err:.2e}'
    if row_idx is not None:                                       # rows not listed stay untouched
        mask = torch.ones(N, dtype=torch.bool)
        mask[row_idx.long()] = False
        assert torch.isnan(planes.cpu()[:, mask]).all()


def test_rcache_matches_uncached_path(edge_impl_reset):
    """SIMT kernels: streaming the cached first-Linear terms of static edges (R-cache) must not change results:
    same atom types, coordinates equal to summation-order rounding."""
    T = 5
    _lib.check(_lib.lib().cbg_set_edge_impl(0, 0))
    for gen_mode, sizes in (('denovo', ([140, 60, 20], [20, 9, 5])), ('partial', ([90, 70], [18, 12]))):
        model, sd = make_model(T, device=dev())
        batch = synthetic.make_batch(*sizes, seed=101, gen_mode=gen_mode)
        n_lig = int(batch['ligand_pos'].shape[0])
        pn, tu = synthetic.make_noise(T, n_lig, 13, seed=9)
        model.use_rcache = True
        a = model.sample(batch, pos_noise=pn, type_uniform=tu)
        model.use_rcache = False
        b = model.sample(batch, pos_noise=pn, type_uniform=tu)
        for t in range(-1, T):
            assert torch.equal(a[t][1].cpu().argmax(-1), b[t][1].cpu().argmax(-1)), (gen_mode, t)
            assert rel_err(a[t][0].cpu(), b[t][0].cpu()) < 1e-5, (gen_mode, t)


def test_receptive_field_pruning_is_exact():
    """Skipping the per-layer work of nodes that cannot reach a generated / ligand atom any more must
    leave every sampled coordinate and atom type bit-identical."""
    T = 4
    for gen_mode, sizes in (('denovo', ([300, 120, 40], [24, 10, 6])), ('partial', ([200, 150], [18, 12]))):
        model, sd = make_model(T, device=dev())
        batch = synthetic.make_batch(*sizes, seed=111, gen_mode=gen_mode)
        n_lig = int(batch['ligand_pos'].shape[0])
        pn, tu = synthetic.make_noise(T, n_lig, 13, seed=10)
        model.use_prune = True
        a = model.sample(batch, pos_noise=pn, type_uniform=tu)
        model.use_prune = False
        b = model.sample(batch, pos_noise=pn, type_uniform=tu)
        for t in range(-1, T):
            assert torch.equal(a[t][0].cpu(), b[t][0].cpu()), (gen_mode, t)
            assert torch.equal(a[t][1].cpu(), b[t][1].cpu()), (gen_mode, t)


@pytest.mark.parametrize('enc', [{'cutoff_mode': 'radius', 'r_max': 7.0}, {'k': 8}, {'k': 20}],
                         ids=['radius7', 'k8', 'k20'])
def test_sample_path_other_graph_modes_vs_oracle(enc):
    """The fused sampling step (R-cache + pruning on) in radius mode and with k < 32: every step's atom
    types bit-exact and coordinates within tolerance of the oracle trajectory."""
    from oracle import diffusion as OD
    T = 5
    model, sd = make_model(T, device=dev(), **enc)
    batch = synthetic.make_batch([160, 70, 33], [20, 11, 6], seed=131, gen_mode='partial')
    n_lig = int(batch['ligand_pos'].shape[0])
    pn, tu = synthetic.make_noise(T, n_lig, 13, seed=12)
    traj = model.sample(batch, pos_noise=pn, type_uniform=tu)
    want = OD.sample(sd, batch, T, pn, tu, k=enc.get('k', 32), cutoff_mode=enc.get('cutoff_mode', 'knn'),
                     r_max=enc.get('r_max', 10.0))
    for t in range(-1, T):
        assert torch.equal(traj[t][1].cpu().argmax(-1), want[t][1].argmax(-1)), t
        assert rel_err(traj[t][0].cpu(), want[t][0]) < TOL, t


def test_knn_random_ragged_batches_bit_exact():
    """Many random ragged batches (graph sizes 1..400, clustered and duplicated points)."""
    from oracle import graph_ops as G
    rs = np.random.RandomState(1234)
    for trial in range(6):
        sizes = [int(v) for v in rs.randint(1, 400, size=rs.randint(1, 9))]
        x = (rs.normal(size=(sum(sizes), 3)) * rs.choice([0.5, 3.0, 10.0])).astype(np.float32)
        if len(x) > 10:
            x[rs.randint(0, len(x), size=5)] = x[rs.randint(0, len(x), size=5)]     # exact duplicates -> ties
        x = torch.from_numpy(x)
        bidx = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
        ptr = [0] + list(np.cumsum(sizes))
        k = int(rs.choice([32, 17, 3]))
        assert torch.equal(cuda_neighbors(x, bidx, k=k), G.neighbor_table(x, ptr, k=k)), (trial, sizes, k)


@pytest.mark.parametrize('layers,classes,wseed', [(3, 8, 1), (6, 16, 2), (9, 13, 3)], ids=['L3-K8', 'L6-K16', 'L9-K13-seed3'])
def test_other_depths_class_counts_and_weights_vs_oracle(layers, classes, wseed):
    """num_layers / num_atomtype other than the de-novo defaults (the reference infers the class count from
    the featuriser mode, configuration.py:13-38) and different weight draws: forward + 3 sampling steps."""
    from cbgbench_b200.targetdiff import TargetDiffB200
    from oracle import denoiser as ODn, diffusion as OD
    T = 3
    cfg = synthetic.targetdiff_config(num_steps=T, num_layers=layers, num_atomtype=classes)
    model = TargetDiffB200(cfg)
    sd = synthetic.seeded_state_dict(model, seed=wseed)
    model.load_state_dict(sd, strict=True)
    model = model.to(dev()).eval()
    batch = synthetic.make_batch([140, 55], [17, 9], seed=141 + wseed, num_classes=classes)
    # single forward through the nn.Module seam
    c_lig = F.one_hot(batch['ligand_atom_type'], classes).float()
    h_lig, h_rec = OD.context_embed(sd, c_lig, batch['protein_atom_feature'], batch['protein_aa_type'],
                                    batch['ligand_lig_flag'], batch['protein_lig_flag'])
    sort_idx, bidx, is_lig = OD.compose(batch['ligand_element_batch'], batch['protein_element_batch'])
    x = torch.cat([batch['protein_pos'], batch['ligand_pos']], 0)[sort_idx]
    h = torch.cat([h_rec, h_lig], 0)[sort_idx]
    xo, ho, co = ODn.unitransformer_forward(sd, x, h, bidx, is_lig, is_lig)
    d = dev()
    xg, hg, cg = model.denoiser(x.to(d), h.to(d), bidx.to(d), is_lig.to(d), is_lig.to(d))
    assert cg.shape == (x.shape[0], classes)
    assert rel_err(xg.cpu(), xo) < TOL and rel_err(hg.cpu(), ho) < TOL and rel_err(cg.cpu(), co) < TOL
    # fused sampling steps
    n_lig = int(batch['ligand_pos'].shape[0])
    pn, tu = synthetic.make_noise(T, n_lig, classes, seed=13)
    traj = model.sample(batch, pos_noise=pn, type_uniform=tu)
    want = OD.sample(sd, batch, T, pn, tu, num_classes=classes)
    for t in range(-1, T):
        assert torch.equal(traj[t][1].cpu().argmax(-1), want[t][1].argmax(-1)), t
        assert rel_err(traj[t][0].cpu(), want[t][0]) < TOL, t


def test_sample_driver_single_gpu(tmp_path):
    """The sample.py-style driver (section 8 row f1): per-pocket results, reproducible from the seed."""
    from cbgbench_b200 import sample_driver
    out = str(tmp_path / 'res.pt')
    argv = ['--pockets', '5', '--batch-size', '2', '--n-prot', '40', '--n-lig', '6', '--steps', '4', '--layers', '2',
            '--out', out]
    a = sample_driver.main(argv)
    b = sample_driver.main(argv)
    saved = torch.load(out)
    assert len(a) == len(saved) == 5
    for ra, rb in zip(a, b):
        assert ra['pos'].shape == (6, 3) and ra['v'].shape == (6,)
        assert torch.equal(ra['pos'], rb['pos']) and torch.equal(ra['v'], rb['v'])
        assert torch.isfinite(ra['pos']).all() and int(ra['v'].max()) < 13


# ---------------------------------------------------------------------------------------------
# the two implementations of the fused X2H edge kernels: wgmma (default) and fp32 SIMT (independent cross-check)
EDGE_IMPLS = {0: 'simt', 6: 'wgmma'}


@pytest.fixture
def edge_impl_reset():
    yield
    _lib.check(_lib.lib().cbg_set_edge_impl(0, 12))
    _lib.check(_lib.lib().cbg_set_edge_impl(_lib.DEFAULT_EDGE_IMPL, 0))     # library default


@pytest.mark.parametrize('case', FORWARD_CASES, ids=[c[0] for c in FORWARD_CASES])
def test_edge_kernel_implementations_agree(case, edge_impl_reset):
    """Both implementations of the X2H kernels (the SIMT ones at every CTA size) must match the reference golden and
    each other.  cbg_set_edge_impl sets the CTA size of the SIMT X2H kernels only, so with impl 0 the SIMT H2X kernel
    runs at its default 12 warps; its other CTA sizes are covered by tests/test_kernel_variants.py (CBG_H2X_WARPS)."""
    name, n_prot, n_lig, seed, gen_mode, enc = case
    gold = golden('forward_cases.npz')
    model, sd = make_model(10, device=dev(), **enc)
    batch = synthetic.make_batch(n_prot, n_lig, seed=seed, gen_mode=gen_mode)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    args = [t.to(dev()) for t in (x, h, bidx, lig, gen)]
    outs, report = {}, []
    for impl, label in EDGE_IMPLS.items():
        for warps in ((8, 12, 16) if impl == 0 else (0,)):
            _lib.check(_lib.lib().cbg_set_edge_impl(impl, warps))
            h1 = model.denoiser(*args, stop_after_layers=1)[1].cpu()
            xg, hg, cg = (t.cpu() for t in model.denoiser(*args))
            outs[(impl, warps)] = (h1, xg, hg, cg)
            errs = [rel_err(a, gold[f'{name}/{k}']) for a, k in ((xg, 'x'), (hg, 'h'), (cg, 'c'))]
            report.append(f'{label}/w{warps}: x {errs[0]:.1e} h {errs[1]:.1e} c {errs[2]:.1e}')
    base = outs[(0, 12)]
    bad = []
    for key, o in outs.items():
        d1, dx, dh = rel_err(o[0], base[0]), rel_err(o[1], base[1]), rel_err(o[2], base[2])
        report.append(f'{EDGE_IMPLS[key[0]]}/w{key[1]} vs simt: h(1 layer) {d1:.1e} x {dx:.1e} h {dh:.1e}')
        if not (d1 < 1e-5 and dx < 1e-4 and dh < 1e-4) or not torch.isfinite(o[2]).all():
            bad.append(key)
    assert not bad, f'{name}: ' + ' | '.join(report)
    for (impl, warps), o in outs.items():
        for a, k in ((o[1], 'x'), (o[2], 'h'), (o[3], 'c')):
            assert rel_err(a, gold[f'{name}/{k}']) < TOL, f'{name}: ' + ' | '.join(report)


def test_edge_kernel_implementations_agree_on_the_sampling_path(edge_impl_reset):
    """Sampling path (static lists, pruning on): wgmma and SIMT kernels give the same atom types and coordinates equal
    to rounding; the SIMT kernels also with their R-cache on (streamed first-Linear terms of static edges)."""
    T = 5
    for gen_mode, sizes in (('denovo', ([140, 60, 20], [20, 9, 5])), ('partial', ([90, 70], [18, 12]))):
        model, sd = make_model(T, device=dev())
        batch = synthetic.make_batch(*sizes, seed=131, gen_mode=gen_mode)
        n_lig = int(batch['ligand_pos'].shape[0])
        pn, tu = synthetic.make_noise(T, n_lig, 13, seed=19)
        res = {}
        for key, impl, rcache in (('tc', 6, False), ('simt', 0, False), ('simt+rcache', 0, True)):
            model.use_rcache = rcache
            _lib.check(_lib.lib().cbg_set_edge_impl(impl, 0))
            res[key] = model.sample(batch, pos_noise=pn, type_uniform=tu)
        for key in ('tc', 'simt+rcache'):
            for t in range(-1, T):
                assert torch.equal(res['simt'][t][1].cpu().argmax(-1), res[key][t][1].cpu().argmax(-1)), (gen_mode, key, t)
                e = rel_err(res[key][t][0].cpu(), res['simt'][t][0].cpu())
                assert e < 1e-5, (gen_mode, key, t, e)


def test_static_fast_path_and_dynamic_scheduling_are_bit_identical(edge_impl_reset):
    """SIMT kernels with the R-cache: nodes whose 32 in-edges are all static skip the coordinate gathers / RBF set-up, and
    warps draw nodes from a work counter instead of a round-robin; neither may change a single bit of the sampled
    coordinates and types."""
    T = 4
    L = _lib.lib()
    try:
        for gen_mode, sizes in (('denovo', ([300, 120, 40], [24, 10, 6])), ('partial', ([200, 150], [18, 12]))):
            model, sd = make_model(T, device=dev())
            model.use_rcache = True
            batch = synthetic.make_batch(*sizes, seed=141, gen_mode=gen_mode)
            n_lig = int(batch['ligand_pos'].shape[0])
            pn, tu = synthetic.make_noise(T, n_lig, 13, seed=23)
            _lib.check(L.cbg_set_edge_impl(0, 0))
            res = {}
            for fast, dyn in ((1, 1), (0, 1), (1, 0), (0, 0)):
                _lib.check(L.cbg_set_option(b'static_fast', fast))
                _lib.check(L.cbg_set_option(b'dyn_sched', dyn))      # work-counter vs round-robin node scheduling
                res[(fast, dyn)] = model.sample(batch, pos_noise=pn, type_uniform=tu)
            for key in ((0, 1), (1, 0), (0, 0)):
                for t in range(-1, T):
                    assert torch.equal(res[key][t][0].cpu(), res[(1, 1)][t][0].cpu()), (gen_mode, key, t)
                    assert torch.equal(res[key][t][1].cpu(), res[(1, 1)][t][1].cpu()), (gen_mode, key, t)
    finally:
        _lib.check(L.cbg_set_option(b'static_fast', 1))
        _lib.check(L.cbg_set_option(b'dyn_sched', 1))


def test_cuda_graph_replay_is_bit_identical():
    """cbg_sample_step_graph_f32 (first step eager, second captured, the rest replayed from one CUDA graph) must give
    the trajectory of the eager per-step path bit for bit - coordinates, one-hot types - on de-novo and
    partial-generation batches, and report the graph's kernel count as launches."""
    T = 9
    for gen_mode, sizes in (('denovo', ([140, 60, 20], [20, 9, 5])), ('partial', ([90, 70], [18, 12]))):
        model, sd = make_model(T, device=dev())
        batch = synthetic.make_batch(*sizes, seed=171, gen_mode=gen_mode)
        n_lig = int(batch['ligand_pos'].shape[0])
        pn, tu = synthetic.make_noise(T, n_lig, 13, seed=37)
        model.use_graph = False
        a = model.sample(batch, pos_noise=pn, type_uniform=tu)
        eager_launches = model.last_launches
        model.use_graph = True
        b = model.sample(batch, pos_noise=pn, type_uniform=tu)
        for t in range(-1, T):
            assert torch.equal(a[t][0].cpu(), b[t][0].cpu()), (gen_mode, t)
            assert torch.equal(a[t][1].cpu(), b[t][1].cpu()), (gen_mode, t)
        assert model.last_launches == eager_launches          # graph nodes are counted like launches
