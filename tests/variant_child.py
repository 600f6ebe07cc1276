"""One fixed GPU workload, run in a child process by tests/test_kernel_variants.py.

The CBG_* switches pick kernel paths once per process (getenv, cached in a static), so every configuration needs a
process of its own.  This script runs the same workload under whatever switches its environment holds and saves every
output to an .npz file:

    python tests/variant_child.py OUT.npz

It loads the library that is already built and never rebuilds it.  If a library call fails it prints the traceback and
cbg_last_error() and exits non-zero.  The parent imports this module for the workload's inputs (the oracle runs there).
"""
import ctypes as C
import os
import sys
import traceback

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from cbgbench_b200 import _lib, synthetic  # noqa: E402
from helpers import FORWARD_CASES, composed_inputs, make_model  # noqa: E402
from test_f2_samplers import bp_batch, bp_model, sbdd_model  # noqa: E402

# denoiser forward: these cases of helpers.FORWARD_CASES, outputs after one layer and after all layers
FORWARD_NAMES = ('ragged_small', 'partial_gen', 'k8', 'tiny_graphs')
FORWARD_STOPS = (('l1', 1), ('all', -1))
# TargetDiff sample: ~300-atom pockets (as in test_receptive_field_pruning_is_exact), so that receptive-field pruning
# drops nodes from layer to layer and the pruned node-GEMM launches see device-side row counts below n_nodes
SAMPLE_T = 5
SAMPLE_CASES = (('denovo', [300, 120, 40], [24, 10, 6], 111), ('partial', [200, 150], [18, 12], 111))
# (run name, use_graph, use_prune)
SAMPLE_RUNS = (('eager', False, True), ('graph', True, True), ('graph_repeat', True, True), ('noprune', False, False))
# DiffSBDD (pocket moves: no static lists) and DiffBP (CoM head: three more H2X layers), 3 steps on a small batch
F2_T = 3
F2_PROT, F2_LIG, F2_SEED = [40, 33, 20], [9, 6, 4], 17


def forward_cases():
    return [c for c in FORWARD_CASES if c[0] in FORWARD_NAMES]


def forward_inputs(case, sd):
    """Composed (x, h, batch_idx, lig_flag, gen_flag) of one forward case (CPU tensors)."""
    name, n_prot, n_lig, seed, gen_mode, enc = case
    return composed_inputs(sd, synthetic.make_batch(n_prot, n_lig, seed=seed, gen_mode=gen_mode))


def sample_inputs(case):
    gen_mode, n_prot, n_lig, seed = case
    batch = synthetic.make_batch(n_prot, n_lig, seed=seed, gen_mode=gen_mode)
    pn, tu = synthetic.make_noise(SAMPLE_T, sum(n_lig), 13, seed=10)
    return batch, pn, tu


def sbdd_inputs():
    batch = synthetic.make_batch(F2_PROT, F2_LIG, seed=F2_SEED)
    return batch, synthetic.make_sbdd_noise(F2_T, sum(F2_LIG), 13, seed=3)


def bp_inputs():
    batch = bp_batch(F2_PROT, F2_LIG, seed=F2_SEED)
    return batch, synthetic.make_bp_noise(F2_T, sum(F2_LIG), seed=5)


def stack_traj(traj, T):
    """{t: (x, c, batch)} for t = -1 .. T-1 -> two arrays [T+1, n, .] in that order."""
    xs = np.stack([traj[t][0].cpu().numpy() for t in range(-1, T)])
    cs = np.stack([traj[t][1].cpu().numpy() for t in range(-1, T)])
    return xs, cs


def run(out_path):
    torch.set_grad_enabled(False)
    dev = torch.device('cuda:0')
    L = _lib.lib()
    out = {}
    for case in forward_cases():
        model, sd = make_model(10, device=dev, **case[5])
        args = [t.to(dev) for t in forward_inputs(case, sd)]
        for tag, stop in FORWARD_STOPS:
            xg, hg, cg = model.denoiser(*args, stop_after_layers=stop)
            for k, v in (('x', xg), ('h', hg), ('c', cg)):
                out[f'fwd/{case[0]}/{tag}/{k}'] = v.cpu().numpy()

    for case in SAMPLE_CASES:
        batch, pn, tu = sample_inputs(case)
        model, _ = make_model(SAMPLE_T, device=dev)
        states = []
        prepare = model.prepare

        def keep_state(*a, **k):          # sample() does not return its plan: keep it for the prune counts
            states.append(prepare(*a, **k))
            return states[-1]
        model.prepare = keep_state
        for run_name, use_graph, use_prune in SAMPLE_RUNS:
            model.use_graph, model.use_prune = use_graph, use_prune
            traj = model.sample(batch, pos_noise=pn, type_uniform=tu)
            key = f'sample/{case[0]}/{run_name}'
            out[key + '/x'], out[key + '/c'] = stack_traj(traj, SAMPLE_T)
            if use_prune:
                # pruned row counts of the last step: counts[l + 1] = nodes whose h layer l still computes
                plan = states[-1]['plan']
                counts = np.zeros(plan.num_layers + 1, dtype=np.int32)
                _lib.check(L.cbg_sample_prune_counts_host(C.byref(plan), counts.ctypes.data, _lib.stream_ptr(dev)))
                out[key + '/prune_counts'] = counts

    batch, noise = sbdd_inputs()
    model, _ = sbdd_model(F2_T, device=dev)
    out['sbdd/x'], out['sbdd/c'] = stack_traj(model.sample(batch, noise=noise), F2_T)

    batch, (pn, tu) = bp_inputs()
    model, _ = bp_model(F2_T, device=dev)
    out['bp/x'], out['bp/c'] = stack_traj(model.sample(batch, pos_noise=pn, type_uniform=tu), F2_T)

    torch.cuda.synchronize()
    np.savez(out_path, **out)


def main(argv):
    if len(argv) != 1:
        sys.stderr.write('usage: variant_child.py OUT.npz\n')
        return 2
    try:
        run(argv[0])
    except Exception:
        traceback.print_exc()
        try:
            msg = _lib.lib().cbg_last_error()
            sys.stderr.write(f'cbg_last_error: {msg.decode() if msg else ""}\n')
        except Exception:
            pass
        return 1
    return 0


if __name__ == '__main__':
    sys.exit(main(sys.argv[1:]))
