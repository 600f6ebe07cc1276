"""D3FG sampling step time on one GPU: prints one JSON line.

    python scripts/bench_difffg.py [--steps K] [--warmup W] [--layers 9]

Workloads: 16 pockets (sample.py's default batch size) and 64 pockets, each of 100 residues and 12 functional groups.
These sizes are a synthetic choice, not taken from data.  Schedule: T = 1000 (d3fg_fg.yml); the model's constructor
builds the angular histograms on the CPU exactly like the reference's, which takes minutes at T = 1000.  Reported per
workload: ms/step from CUDA events over K steps after W warm-up steps, kernel launches per step, samples/s =
B / (T * s/step), and the GPU name and power limit read in the same run.  When the reference is staged under
oracle/_ref/, its eager ``D3FG.sample`` on the GPU is timed at T = 5 (time divided by steps); otherwise ``null``.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from cbgbench_b200 import synthetic  # noqa: E402
from cbgbench_b200.difffg import D3FGB200  # noqa: E402

T = 1000
WORKLOADS = [(16, 100, 12), (64, 100, 12)]


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    name, power = (q.stdout.strip().splitlines() or ['?,?'])[0].split(',')[:2]
    return name.strip(), power.strip()


def time_ours(model, batch, steps, warmup):
    model.sample(batch, num_steps=warmup, traj_mode='final')
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    model.sample(batch, num_steps=steps, traj_mode='final')
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / steps, model.last_launches / steps


def time_reference(batch, layers, dev):
    """The reference's eager D3FG.sample at T = 5, from oracle/_ref/ (None when it is not staged)."""
    ref_dir = os.path.join(ROOT, 'oracle', '_ref')
    if not os.path.isdir(os.path.join(ref_dir, 'repo')):
        return None
    sys.path.insert(0, os.path.join(ROOT, 'baseline'))
    import ref_runner
    ref_runner.install()
    from repo.models.diffusion.difffg import D3FG
    cfg = ref_runner.EasyDict(json.loads(json.dumps(synthetic.difffg_config(num_steps=5, num_layers=layers))))
    model = D3FG(cfg).to(dev).eval()
    b = {k: v.to(dev) for k, v in batch.items()}
    with torch.no_grad():
        model.sample(b)
        torch.cuda.synchronize()
        t0 = time.time()
        model.sample(b)
        torch.cuda.synchronize()
    return (time.time() - t0) * 1000.0 / 5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--layers', type=int, default=9)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    name, power = gpu_info()
    model = D3FGB200(synthetic.difffg_config(num_steps=T, num_layers=args.layers))
    model.load_state_dict(synthetic.seeded_state_dict(model, seed=0), strict=True)
    model = model.eval().to(dev)
    out = {'bench': 'difffg', 'gpu': name, 'power_limit': power, 'T': T, 'steps': args.steps, 'layers': args.layers,
           'workloads': []}
    for B, n_res, n_fg in WORKLOADS:
        batch = synthetic.make_fg_batch([n_res] * B, [n_fg] * B, seed=1)
        ms, launches = time_ours(model, batch, args.steps, args.warmup)
        try:
            ref_ms = time_reference(batch, args.layers, dev)
        except ImportError:
            ref_ms = None
        out['workloads'].append({'pockets': B, 'residues': n_res, 'fgs': n_fg, 'ms_per_step': round(ms, 4),
                                 'launches_per_step': launches, 'samples_per_s': round(B / (T * ms / 1000.0), 4),
                                 'reference_ms_per_step': None if ref_ms is None else round(ref_ms, 3)})
    print(json.dumps(out))


if __name__ == '__main__':
    main()
