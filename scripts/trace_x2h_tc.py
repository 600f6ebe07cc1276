"""Per-tile stage times of the wgmma X2H tile kernel (csrc/x2h_tc.cu) on the c2 workload (64 pockets x (300 + 24) atoms),
from the SM-clock stamps that warpgroup 0 of CTA 0 writes through cbg_debug_x2h_trace, plus the launch times of the
attention-weight (x2h_k) and aggregation (x2h_v) kernels by CUDA events in the same run.

The traced launch is layer 0 of an eager denoise step with the real pruned node list.  A stage is the time between two
consecutive events of warpgroup 0's loop (the first one starts at the previous tile's last event); medians over the
tiles between the first and the last (the prologue and the drain are shown separately).
Usage: python scripts/trace_x2h_tc.py"""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cbgbench_b200 import _lib  # noqa: E402

# the interval that ends at event e of tile k (TC_STAMP in csrc/x2h_tc.cu)
STAGES = ['epilogue(k-1) done -> MMA1(k) complete', 'S1, MMA2(k) issue', 'G(k+1) build, MMA2(k) wait',
          'G(k+1) hand-off, MMA1(k+1) issue', 'epilogue(k)']
MAX_TILES = 64


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm', '--format=csv,noheader',
                              '-i', str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or out.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f'{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})'


def trace_one(model, state, t, X, Cc, mode_k):
    L = _lib.lib()
    buf = torch.zeros((MAX_TILES + 1) * 16, dtype=torch.int64, device=state['device'])
    torch.cuda.synchronize()
    _lib.check(L.cbg_debug_x2h_trace(buf.data_ptr(), MAX_TILES if mode_k else -MAX_TILES))
    model.run_steps(state, [t], X, Cc)
    torch.cuda.synchronize()
    _lib.check(L.cbg_set_option(b'x2h_trace_off', 0))
    return buf.cpu().numpy().reshape(MAX_TILES + 1, 16)


def report(name, t):
    ev, cta = t[:MAX_TILES, :5], t[MAX_TILES, :3]
    n = int((ev[:, 0] != 0).sum())
    print(f'{name}: CTA 0 ran {n} tiles')
    if n < 3:
        print('  too few tiles for a steady state')
        return
    steady = range(1, n - 1)
    print(f'  {"stage (median cycles per tile)":<44}{"median":>8}{"min":>8}{"max":>8}')
    for e, label in enumerate(STAGES):
        d = [ev[k, e] - (ev[k, e - 1] if e else ev[k - 1, 4]) for k in steady if ev[k, e] and (e or ev[k - 1, 4])]
        if d:
            print(f'  {e}: {label:<41}{np.median(d):8.0f}{min(d):8.0f}{max(d):8.0f}')
    period = [ev[k, 0] - ev[k - 1, 0] for k in steady]
    print(f'  {"tile period":<44}{np.median(period):8.0f}{min(period):8.0f}{max(period):8.0f}')
    first = ev[0][ev[0] != 0].min()
    last = ev[n - 1][ev[n - 1] != 0].max()
    print(f'  prologue: entry -> weights requested, list read {cta[1] - cta[0]:.0f}; -> first event of tile 0 '
          f'{first - cta[1]:.0f}; last event of the last tile -> exit {cta[2] - last:.0f}; entry -> exit '
          f'{cta[2] - cta[0]:.0f} cycles')


def main():
    import bench
    from cbgbench_b200 import synthetic
    from cbgbench_b200.targetdiff import TargetDiffB200

    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    torch.set_grad_enabled(False)
    print('card (name, power limit, SM clock):', card())
    batch, enc = bench.workload_batch('c2', 0)
    model = TargetDiffB200(synthetic.targetdiff_config(num_steps=bench.T_STEPS, **enc))
    model.load_state_dict(synthetic.seeded_state_dict(model, seed=0), strict=True)
    model = model.to(dev).eval()
    model.use_graph = False          # eager steps: the one-shot trace arms the next launch, not a graph capture
    torch.manual_seed(2024)
    state = model.prepare(batch)
    n_lig, K = state['n_lig'], model.num_classes
    X = torch.empty((bench.T_STEPS + 1, n_lig, 3), device=dev)
    Cc = torch.empty((bench.T_STEPS + 1, n_lig, K), device=dev)
    X[bench.T_STEPS].copy_(state['x_lig'])
    Cc[bench.T_STEPS].copy_(state['c_lig'])
    t_seq = list(reversed(range(bench.T_STEPS)))
    model.run_steps(state, t_seq[:3], X, Cc)        # warm-up
    L = _lib.lib()
    L.cbg_profile_enable(1)
    model.run_steps(state, t_seq[3:8], X, Cc)
    prof = _lib.profile_collect()
    L.cbg_profile_enable(0)
    for k in ('x2h_k', 'x2h_v'):
        ms, launches = prof[k]
        print(f'{k}: {1e3 * ms / launches:.1f} us per launch (CUDA events, mean of {launches:.0f} launches over 5 steps, '
              f'every layer)')
    report('x2h_k layer 0 (MODE_K)', trace_one(model, state, t_seq[8], X, Cc, True))
    report('x2h_v layer 0 (MODE_V)', trace_one(model, state, t_seq[9], X, Cc, False))


if __name__ == '__main__':
    main()
