#!/usr/bin/env python
"""Measurement of DiffBP's validation loss: eval-mode ``DiffBPB200.forward(batch)`` (R = eval_interval = 10 timesteps,
T = 1000 schedule) on one GPU, device-resident inputs, seeded synthetic weights.

Shapes: c2 (64 pockets x (300 + 24) atoms) and a 4-graph validation batch (the train configs' batch_size: 4).  For
each: ms per forward (CUDA events around each call, mean over --steps calls after --warmup), kernel launches per call,
and the same R timesteps as R sequential single-timestep calls (what the reference's loop does, on this path).  There
is no reference arm.  Prints one JSON line; the GPU name and power limit are read in the same run.

    python scripts/bench_bp_eval.py [--steps 5] [--warmup 2]
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
    from cbgbench_b200.diffbp import DiffBPB200
    from cbgbench_b200.targetdiff import eval_t_values
    if not torch.cuda.is_available():
        raise SystemExit('bench_bp_eval.py measures the GPU path: no CUDA device')
    torch.set_grad_enabled(False)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    model = DiffBPB200(synthetic.diffbp_config(num_steps=T))
    model.load_state_dict(synthetic.seeded_state_dict(model, seed=0), strict=True)
    model = model.to(dev).eval()
    t_values = eval_t_values(T, 10)
    out = {'workload': f'eval-mode DiffBP.forward, R={len(t_values)} timesteps, T={T}', 'gpu': gpu_info(),
           'n_gpus': 1, 'steps': args.steps, 'warmup': args.warmup, 'dtype': 'f32', 'data': 'synthetic'}
    for name, (n_prot, n_lig) in SHAPES.items():
        batch = {k: v.to(dev) for k, v in synthetic.make_batch(n_prot, n_lig, seed=2024).items()}
        n = batch['ligand_pos'].shape[0]
        pn, tu = synthetic.make_bp_noise(len(t_values), n, seed=7)
        pn, tu = pn.to(dev), tu.to(dev)
        row = {'shape': f'{len(n_prot)} pockets x ({n_prot[0]}+{n_lig[0]}) atoms'}
        row['ms_per_forward'] = round(time_calls(lambda: model(batch, pos_noise=pn, type_uniform=tu),
                                                 args.steps, args.warmup), 3)
        row['launches_per_forward'] = model.last_launches

        def sequential():
            for r, t in enumerate(t_values):
                model.eval_losses(batch, [t], pos_noise=pn[r:r + 1], type_uniform=tu[r:r + 1])
        row['ms_sequential_R_calls'] = round(time_calls(sequential, args.steps, args.warmup), 3)
        out[name] = row
    print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
