"""The kernel paths selected by the CBG_* switches, against the default configuration and the oracle.

Each switch is read once per process (getenv, cached in a static), so every configuration runs the fixed workload of
tests/variant_child.py in a child process of its own, with every CBG_* variable of this process removed and the
configuration's added.  The children run one at a time; a timeout kills the child.

Bars:
- "bit-identical": every saved output of the child equals the reference child's bit for bit.
- "tolerance": against the oracle, relative error below 1e-4, coordinates element-wise within rtol 1e-4 / atol 1e-5
  and atom types bit-exact; against the default child, relative error below 1e-5 for h after one layer and for the
  coordinates of every sampling step, and equal atom types.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import variant_child as V
from helpers import assert_close, make_model, rel_err

pytestmark = pytest.mark.gpu
CHILD = os.path.abspath(V.__file__)
CHILD_TIMEOUT = 900          # seconds: CUDA start-up plus well under a minute of work on an H100
TOL = 1e-4                   # against the oracle
TOL_VARIANT = 1e-5           # against the default child
torch.set_grad_enabled(False)


def _run_child(out_dir, env_add):
    name = '_'.join(f'{k}={v}' for k, v in sorted(env_add.items())) or 'default'
    out = os.path.join(out_dir, name + '.npz')
    env = {k: v for k, v in os.environ.items() if not k.startswith('CBG_')}
    env.update(env_add)
    cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [CHILD, out]
    # subprocess.run kills the child when the timeout expires
    res = subprocess.run(cmd, env=env, cwd=V.ROOT, capture_output=True, text=True, timeout=CHILD_TIMEOUT)
    assert res.returncode == 0, f'{name}: child exited with {res.returncode}\n{res.stdout[-4000:]}\n{res.stderr[-4000:]}'
    with np.load(out) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope='module')
def child(tmp_path_factory):
    """child(**env) -> outputs of the workload under those switches; each configuration runs once per module."""
    out_dir = str(tmp_path_factory.mktemp('variants'))
    cache = {}

    def get(**env):
        key = tuple(sorted(env.items()))
        if key not in cache:
            cache[key] = _run_child(out_dir, env)
        return cache[key]
    return get


@pytest.fixture(scope='module')
def default_out(child):
    return child()


@pytest.fixture(scope='module')
def oracle():
    """The workload on the CPU oracle, keyed like the child's outputs."""
    from oracle import denoiser as ODn, diffusion as OD, diffusion_bp as OB, diffusion_sbdd as OS
    want = {}
    for case in V.forward_cases():
        name, enc = case[0], case[5]
        _, sd = make_model(10, **enc)
        x, h, bidx, lig, gen = V.forward_inputs(case, sd)
        xo, ho, co, trace = ODn.unitransformer_forward(sd, x, h, bidx, lig, gen, k=enc.get('k', 32), return_trace=True)
        want[f'fwd/{name}/l1/x'], want[f'fwd/{name}/l1/h'] = trace['x'][0], trace['h'][0]
        want[f'fwd/{name}/all/x'], want[f'fwd/{name}/all/h'], want[f'fwd/{name}/all/c'] = xo, ho, co
    _, sd = make_model(V.SAMPLE_T)
    for case in V.SAMPLE_CASES:
        batch, pn, tu = V.sample_inputs(case)
        traj = OD.sample(sd, batch, V.SAMPLE_T, pn, tu)
        want[f'sample/{case[0]}/x'], want[f'sample/{case[0]}/c'] = V.stack_traj(traj, V.SAMPLE_T)
    _, sd = V.sbdd_model(V.F2_T)
    batch, noise = V.sbdd_inputs()
    want['sbdd/x'], want['sbdd/c'] = V.stack_traj(OS.sample(sd, batch, V.F2_T, noise)[0], V.F2_T)
    _, sd = V.bp_model(V.F2_T)
    batch, (pn, tu) = V.bp_inputs()
    want['bp/x'], want['bp/c'] = V.stack_traj(OB.sample(sd, batch, V.F2_T, pn, tu), V.F2_T)
    return want


def _trajectories(out):
    """(label, coordinates [T+1,n,3], atom types [T+1,n]) of every sampling run of a child's outputs."""
    runs = [(f'sample/{c[0]}/{r[0]}', f'sample/{c[0]}') for c in V.SAMPLE_CASES for r in V.SAMPLE_RUNS]
    runs += [('sbdd', 'sbdd'), ('bp', 'bp')]
    return [(key, oracle_key, out[key + '/x'], out[key + '/c'].argmax(-1)) for key, oracle_key in runs]


def assert_pruning_drops_nodes(out):
    """The pruned node GEMMs only differ from the unpruned ones if the row counts really fall from layer to layer."""
    for case in V.SAMPLE_CASES:
        for run, _, prune in V.SAMPLE_RUNS:
            if prune:
                cnt = out[f'sample/{case[0]}/{run}/prune_counts']
                assert (np.diff(cnt) <= 0).all() and (np.diff(cnt) < 0).any(), (case[0], run, cnt)


def assert_matches_oracle(out, want):
    for case in V.forward_cases():
        for tag, keys in (('l1', 'xh'), ('all', 'xhc')):
            for k in keys:
                key = f'fwd/{case[0]}/{tag}/{k}'
                err = rel_err(out[key], want[key])
                assert err < TOL, f'{key}: rel err {err:.2e} against the oracle'
            assert_close(out[f'fwd/{case[0]}/{tag}/x'], want[f'fwd/{case[0]}/{tag}/x'], what=f'fwd/{case[0]}/{tag}/x')
    for key, oracle_key, x, v in _trajectories(out):
        xo, co = want[oracle_key + '/x'], want[oracle_key + '/c']
        for s in range(x.shape[0]):
            err = rel_err(x[s], xo[s])
            assert err < TOL, f'{key} state {s}: coordinate rel err {err:.2e} against the oracle'
            assert_close(x[s], xo[s], what=f'{key} state {s} coordinates')
            if key == 'sbdd':        # continuous type features
                err = rel_err(out['sbdd/c'][s], co[s])
                assert err < TOL, f'sbdd state {s}: type-feature rel err {err:.2e} against the oracle'
            else:
                assert np.array_equal(v[s], co[s].argmax(-1)), f'{key} state {s}: atom types differ from the oracle'


def assert_close_to(out, ref):
    for case in V.forward_cases():
        key = f'fwd/{case[0]}/l1/h'
        err = rel_err(out[key], ref[key])
        assert err < TOL_VARIANT, f'{key}: rel err {err:.2e} against the default configuration'
    for (key, _, x, v), (_, _, xr, vr) in zip(_trajectories(out), _trajectories(ref)):
        for s in range(x.shape[0]):
            err = rel_err(x[s], xr[s])
            assert err < TOL_VARIANT, f'{key} state {s}: coordinate rel err {err:.2e} against the default configuration'
            assert np.array_equal(v[s], vr[s]), f'{key} state {s}: atom types differ from the default configuration'


def assert_identical(out, ref, what):
    assert sorted(out) == sorted(ref)
    bad = [k for k in sorted(out) if not np.array_equal(out[k], ref[k])]
    assert not bad, f'{what}: not bit-identical in ' + ', '.join(bad)


def check_tolerance(out, default_out, oracle):
    assert_pruning_drops_nodes(out)
    assert_matches_oracle(out, oracle)
    assert_close_to(out, default_out)


def test_default_configuration_matches_oracle(default_out, oracle):
    """The reference child itself: the bars of the suite against the oracle, and pruning that really prunes."""
    assert_pruning_drops_nodes(default_out)
    assert_matches_oracle(default_out, oracle)
    for case in V.SAMPLE_CASES:        # a second graph replay of the same plan repeats the first bit for bit
        for k in ('x', 'c'):
            assert np.array_equal(default_out[f'sample/{case[0]}/graph/{k}'], default_out[f'sample/{case[0]}/graph_repeat/{k}'])


def test_single_stream_orchestration_is_bit_identical(child, default_out):
    """CBG_OVERLAP=0: the same kernels with the same arguments on one stream instead of four."""
    assert_identical(child(CBG_OVERLAP='0'), default_out, 'CBG_OVERLAP=0')


def test_programmatic_dependent_launch_is_bit_identical(child, default_out):
    """CBG_PDL=1: x2h_tc_kernel launched with programmatic stream serialisation, eagerly and inside the captured CUDA
    graph; its griddepcontrol.wait comes before the first read of anything the previous kernel writes."""
    out = child(CBG_PDL='1')
    assert_identical(out, default_out, 'CBG_PDL=1')
    for case in V.SAMPLE_CASES:
        for k in ('x', 'c'):
            assert np.array_equal(out[f'sample/{case[0]}/graph/{k}'], out[f'sample/{case[0]}/graph_repeat/{k}'])
            assert np.array_equal(out[f'sample/{case[0]}/graph/{k}'], out[f'sample/{case[0]}/eager/{k}'])


def test_in_place_edge_gate_is_bit_identical(child, default_out):
    """CBG_GATE_COMPACT=0: the in-place gate kernel and the compacted-list kernel both evaluate gate_value on the same
    (x_i, x_j) pair of every moving edge."""
    assert_identical(child(CBG_GATE_COMPACT='0'), default_out, 'CBG_GATE_COMPACT=0')


def test_sampling_without_static_lists_is_bit_identical(child, default_out):
    """CBG_STATIC_LISTS=0: a full neighbour search and every edge gate at every step instead of the per-batch static
    lists and cached gates (documented as exact)."""
    assert_identical(child(CBG_STATIC_LISTS='0'), default_out, 'CBG_STATIC_LISTS=0')


def test_tf32_node_gemm(child, default_out, oracle):
    """CBG_NODE_GEMM=tf32: the 3xTF32 wgmma node GEMM; under pruning two launches (source planes on a side stream)
    with device-side row counts instead of the f16 kernel's merged launch."""
    check_tolerance(child(CBG_NODE_GEMM='tf32'), default_out, oracle)


@pytest.mark.parametrize('cluster', ['2', '4'])
def test_tf32_node_gemm_weight_multicast_is_bit_identical(child, cluster):
    """CBG_GEMM_CLUSTER: the weight chunks reach each CTA by multicast from the cluster instead of by its own copy; the
    arithmetic per row is unchanged."""
    out = child(CBG_NODE_GEMM='tf32', CBG_GEMM_CLUSTER=cluster)
    assert_identical(out, child(CBG_NODE_GEMM='tf32'), f'CBG_NODE_GEMM=tf32 CBG_GEMM_CLUSTER={cluster}')


def test_simt_node_gemm(child, default_out, oracle):
    """CBG_NODE_GEMM=simt (fp32 SIMT node GEMM), with the side streams and on one stream."""
    a = child(CBG_NODE_GEMM='simt')
    b = child(CBG_NODE_GEMM='simt', CBG_OVERLAP='0')
    check_tolerance(a, default_out, oracle)
    check_tolerance(b, default_out, oracle)
    assert_identical(b, a, 'CBG_NODE_GEMM=simt with CBG_OVERLAP=0')


@pytest.mark.parametrize('warps', ['8', '12', '16'])
def test_simt_h2x_kernel(child, default_out, oracle, warps):
    """CBG_H2X_IMPL=simt: the fp32 SIMT H2X kernel (denoiser layers and the DiffBP CoM head) at every CTA size, while
    X2H stays on the wgmma kernels."""
    check_tolerance(child(CBG_H2X_IMPL='simt', CBG_H2X_WARPS=warps), default_out, oracle)
