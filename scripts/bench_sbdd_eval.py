#!/usr/bin/env python
"""Measurement of DiffSBDD's validation loss: eval-mode ``DiffSBDDB200.forward(batch)`` (R = eval_interval = 10
timesteps, each noised at t and at 0, T = 1000 schedule) on one GPU, device-resident inputs, seeded synthetic weights.

Shapes: c2 (64 pockets x (300 + 24) atoms) and a 4-graph validation batch (the train configs' batch_size: 4).  For
each: ms per forward (CUDA events around each call, mean over --steps calls after --warmup), kernel launches per call,
and the same R timesteps as R sequential single-timestep calls (what the reference's loop does, on this path).  There
is no reference arm.  Prints one JSON line; the GPU name and power limit are read in the same run.

    python scripts/bench_sbdd_eval.py [--steps 5] [--warmup 2]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_eval import SHAPES, T, gpu_info, time_calls  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    args = ap.parse_args()
    import torch
    from cbgbench_b200 import synthetic
    from cbgbench_b200.diffsbdd import DiffSBDDB200, eval_t_values
    if not torch.cuda.is_available():
        raise SystemExit('bench_sbdd_eval.py measures the GPU path: no CUDA device')
    torch.set_grad_enabled(False)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    model = DiffSBDDB200(synthetic.diffsbdd_config(num_steps=T))
    model.load_state_dict(synthetic.seeded_state_dict(model, seed=0), strict=True)
    model = model.to(dev).eval()
    t_values = eval_t_values(T, 10)
    out = {'workload': f'eval-mode DiffSBDD.forward, R={len(t_values)} timesteps x 2 noised copies, T={T}',
           'gpu': gpu_info(), 'n_gpus': 1, 'steps': args.steps, 'warmup': args.warmup, 'dtype': 'f32',
           'data': 'synthetic'}
    for name, (n_prot, n_lig) in SHAPES.items():
        batch = {k: v.to(dev) for k, v in synthetic.make_batch(n_prot, n_lig, seed=2024).items()}
        n = batch['ligand_pos'].shape[0]
        noise = {k: v.to(dev) for k, v in synthetic.make_sbdd_eval_noise(len(t_values), n, model.num_classes, seed=7).items()}
        row = {'shape': f'{len(n_prot)} pockets x ({n_prot[0]}+{n_lig[0]}) atoms'}
        row['ms_per_forward'] = round(time_calls(lambda: model(batch, noise=noise), args.steps, args.warmup), 3)
        row['launches_per_forward'] = model.last_launches

        def sequential():
            for r, t in enumerate(t_values):
                model.eval_losses(batch, [t], noise={k: v[r:r + 1] for k, v in noise.items()})
        row['ms_sequential_R_calls'] = round(time_calls(sequential, args.steps, args.warmup), 3)
        out[name] = row
    print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
