#!/usr/bin/env python
"""Measurement of the validation loss: eval-mode ``TargetDiffB200.forward(batch)`` (R = eval_interval = 10 timesteps,
T = 1000 schedule) on one GPU, device-resident inputs, seeded synthetic weights.

Shapes: c2 (64 pockets x (300 + 24) atoms) and a 4-graph validation batch (the train configs' batch_size: 4).  For
each: ms per forward (CUDA events around each call, mean over --steps calls after --warmup), kernel launches per call,
the same R timesteps as R sequential single-timestep calls (what the reference's loop does, on this path), and, when
the reference has been staged into oracle/_ref/, the reference's eager GPU forward on the same batch.  Prints one
JSON line.  The GPU name and power limit go with the numbers.

    python scripts/bench_eval.py [--steps 5] [--warmup 2] [--no-ref]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T = 1000
SHAPES = {'c2': ([300] * 64, [24] * 64), 'val4': ([300] * 4, [24] * 4)}


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else 'unknown'
    except Exception:          # nvidia-smi missing: the torch name still identifies the card
        import torch
        return torch.cuda.get_device_name(0)


def time_calls(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    starts = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
    ends = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
    for i in range(steps):
        starts[i].record()
        fn()
        ends[i].record()
    torch.cuda.synchronize()
    return sum(s.elapsed_time(e) for s, e in zip(starts, ends)) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--no-ref', action='store_true')
    args = ap.parse_args()
    import torch
    from cbgbench_b200 import synthetic
    from cbgbench_b200.targetdiff import TargetDiffB200, eval_t_values
    if not torch.cuda.is_available():
        raise SystemExit('bench_eval.py measures the GPU path: no CUDA device')
    torch.set_grad_enabled(False)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    model = TargetDiffB200(synthetic.targetdiff_config(num_steps=T))
    model.load_state_dict(synthetic.seeded_state_dict(model, seed=0), strict=True)
    model = model.to(dev).eval()
    t_values = eval_t_values(T, 10)
    ref = None
    if not args.no_ref:
        from baseline import ref_runner
        if ref_runner.ref_root() is not None:
            ref = ref_runner.build_reference_model(T, {}, dev)
    out = {'workload': f'eval-mode TargetDiff.forward, R={len(t_values)} timesteps, T={T}', 'gpu': gpu_info(),
           'n_gpus': 1, 'steps': args.steps, 'warmup': args.warmup, 'dtype': 'f32', 'data': 'synthetic'}
    for name, (n_prot, n_lig) in SHAPES.items():
        batch = {k: v.to(dev) for k, v in synthetic.make_batch(n_prot, n_lig, seed=2024).items()}
        n = batch['ligand_pos'].shape[0]
        pn, tu = synthetic.make_noise(len(t_values), n, 13, seed=7)
        pn, tu = pn.to(dev), tu.to(dev)
        row = {'shape': f'{len(n_prot)} pockets x ({n_prot[0]}+{n_lig[0]}) atoms'}
        row['ms_per_forward'] = round(time_calls(lambda: model(batch, pos_noise=pn, type_uniform=tu),
                                                 args.steps, args.warmup), 3)
        row['launches_per_forward'] = model.last_launches

        def sequential():
            for r, t in enumerate(t_values):
                model.eval_losses(batch, [t], pos_noise=pn[r:r + 1], type_uniform=tu[r:r + 1])
        row['ms_sequential_R_calls'] = round(time_calls(sequential, args.steps, args.warmup), 3)
        if ref is not None:
            # the reference draws its own noise (randn_like / rand_like on the device): same work, other numbers
            torch.cuda.synchronize()
            ref(batch)                                  # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ref(batch)
            torch.cuda.synchronize()
            row['reference_gpu_ms_per_forward'] = round((time.perf_counter() - t0) * 1e3, 3)
        else:
            row['reference_gpu_ms_per_forward'] = None
        out[name] = row
    print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
