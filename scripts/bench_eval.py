#!/usr/bin/env python
"""Measurement of the validation loss: eval-mode ``forward(batch)`` of TargetDiff, DiffBP, DiffSBDD or D3FG (``difffg``)
(R = eval_interval = 10 timesteps, DiffSBDD's each noised at t and at 0, T = 1000 schedule) on one GPU, device-resident
inputs, seeded synthetic weights.

Shapes: c2 (64 pockets x (300 + 24) atoms) and a 4-graph validation batch (the train configs' batch_size: 4); for D3FG
64 and 4 pockets x (100 residues + 12 functional groups), a synthetic choice (the model's constructor builds the T = 1000
angular histograms on the CPU first, about a minute).  For
each: ms per forward (CUDA events around each call, mean over --steps calls after --warmup), kernel launches per call,
the same R timesteps as R sequential single-timestep calls (what the reference's loop does, on this path), and, for
TargetDiff when the reference has been staged into oracle/_ref/, the reference's eager GPU forward on the same batch.
Prints one JSON line.  The GPU name and power limit go with the numbers.

    python scripts/bench_eval.py [--model targetdiff|diffbp|diffsbdd|difffg] [--steps 5] [--warmup 2] [--no-ref]
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
FG_SHAPES = {'c64': ([100] * 64, [12] * 64), 'val4': ([100] * 4, [12] * 4)}


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


def noise_kwargs(model_name, R, n, K, dev):
    """Seeded draws of R timesteps as the keyword arguments of the model's forward / eval_losses, and a slicer that
    picks timesteps r0 .. r1-1 of them."""
    from cbgbench_b200 import synthetic
    if model_name == 'diffsbdd':
        noise = {k: v.to(dev) for k, v in synthetic.make_sbdd_eval_noise(R, n, K, seed=7).items()}
        return {'noise': noise}, lambda r0, r1: {'noise': {k: v[r0:r1] for k, v in noise.items()}}
    if model_name == 'difffg':
        draws = dict(zip(('pos_noise', 'rot_draws', 'type_uniform'),
                         (d.to(dev) for d in synthetic.make_fg_draws(R, n, num_fgtype=K, seed=7))))
        return draws, lambda r0, r1: {k: v[r0:r1] for k, v in draws.items()}
    pn, tu = synthetic.make_bp_noise(R, n, seed=7) if model_name == 'diffbp' else synthetic.make_noise(R, n, K, seed=7)
    pn, tu = pn.to(dev), tu.to(dev)
    return {'pos_noise': pn, 'type_uniform': tu}, lambda r0, r1: {'pos_noise': pn[r0:r1], 'type_uniform': tu[r0:r1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--model', choices=('targetdiff', 'diffbp', 'diffsbdd', 'difffg'), default='targetdiff')
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--no-ref', action='store_true', help='skip the reference arm (TargetDiff only)')
    args = ap.parse_args()
    import torch
    from cbgbench_b200 import synthetic
    from cbgbench_b200.targetdiff import eval_t_values, get_model
    if not torch.cuda.is_available():
        raise SystemExit('bench_eval.py measures the GPU path: no CUDA device')
    torch.set_grad_enabled(False)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    cfg = getattr(synthetic, f'{args.model}_config')(num_steps=T)
    model = get_model(cfg)
    model.load_state_dict(synthetic.seeded_state_dict(model, seed=0), strict=True)
    model = model.to(dev).eval()
    t_values = eval_t_values(T, 10, first=1 if args.model == 'diffsbdd' else 0)
    ref = None
    if args.model == 'targetdiff' and not args.no_ref:
        from baseline import ref_runner
        if ref_runner.ref_root() is not None:
            ref = ref_runner.build_reference_model(T, {}, dev)
    label = {'targetdiff': 'TargetDiff', 'diffbp': 'DiffBP', 'diffsbdd': 'DiffSBDD', 'difffg': 'D3FG'}[args.model]
    copies = ' x 2 noised copies' if args.model == 'diffsbdd' else ''
    out = {'workload': f'eval-mode {label}.forward, R={len(t_values)} timesteps{copies}, T={T}', 'gpu': gpu_info(),
           'n_gpus': 1, 'steps': args.steps, 'warmup': args.warmup, 'dtype': 'f32', 'data': 'synthetic'}
    fg = args.model == 'difffg'
    for shape, (n_prot, n_lig) in (FG_SHAPES if fg else SHAPES).items():
        make = synthetic.make_fg_batch if fg else synthetic.make_batch
        batch = {k: v.to(dev) for k, v in make(n_prot, n_lig, seed=2024).items()}
        n = sum(n_lig)
        kw, part = noise_kwargs(args.model, len(t_values), n, model.num_classes, dev)
        unit = 'residues + FGs' if fg else 'atoms'
        row = {'shape': f'{len(n_prot)} pockets x ({n_prot[0]}+{n_lig[0]}) {unit}'}
        row['ms_per_forward'] = round(time_calls(lambda: model(batch, **kw), args.steps, args.warmup), 3)
        row['launches_per_forward'] = model.last_launches

        def sequential():
            for r, t in enumerate(t_values):
                model.eval_losses(batch, [t], **part(r, r + 1))
        row['ms_sequential_R_calls'] = round(time_calls(sequential, args.steps, args.warmup), 3)
        if args.model == 'targetdiff':
            row['reference_gpu_ms_per_forward'] = None
        if ref is not None:
            # the reference draws its own noise (randn_like / rand_like on the device): same work, other numbers
            torch.cuda.synchronize()
            ref(batch)                                  # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ref(batch)
            torch.cuda.synchronize()
            row['reference_gpu_ms_per_forward'] = round((time.perf_counter() - t0) * 1e3, 3)
        out[shape] = row
    print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
