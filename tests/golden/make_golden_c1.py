"""Golden for BASELINE.json config 1: the UNMODIFIED reference's TargetDiff.sample on one synthetic pocket
(200 protein + 24 ligand atoms), T = 50 denoise steps, with injected noise (needs a checkout of the reference).

    python tests/golden/make_golden_c1.py      ->  tests/golden/trajectory_c1_T50.npz

Inputs and weights are regenerated bit-identically by the tests (cbgbench_b200/synthetic.py); only the reference's
outputs are stored: ligand coordinates and atom types after every step.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import ref_shims  # noqa: E402
from cbgbench_b200 import synthetic  # noqa: E402
from cbgbench_b200.targetdiff import TargetDiffB200  # noqa: E402

T = 50
DATA_SEED, NOISE_SEED = 2024, 31


def main():
    torch.set_grad_enabled(False)
    ref = ref_shims.load_targetdiff(ref_shims.targetdiff_cfg(num_steps=T))
    mine = TargetDiffB200(synthetic.targetdiff_config(num_steps=T))
    ref.load_state_dict(synthetic.seeded_state_dict(mine, seed=0), strict=True)
    batch = synthetic.make_batch([200], [24], seed=DATA_SEED)
    pn, tu = synthetic.make_noise(T, 24, 13, seed=NOISE_SEED)
    calls = {'randn': 0, 'rand': 0}
    orig_randn, orig_rand = torch.randn_like, torch.rand_like

    def fake_randn_like(a, *aa, **kk):      # once per step, t = T-1 ... 0 (diffusion_scheduler.py:163)
        t = T - 1 - calls['randn']
        calls['randn'] += 1
        return pn[t]

    def fake_rand_like(a, *aa, **kk):       # categorical.py:27
        t = T - 1 - calls['rand']
        calls['rand'] += 1
        return tu[t]

    torch.randn_like, torch.rand_like = fake_randn_like, fake_rand_like
    try:
        traj = ref.sample(batch)
    finally:
        torch.randn_like, torch.rand_like = orig_randn, orig_rand
    assert calls == {'randn': T, 'rand': T}, calls
    out = {}
    for t in range(-1, T):
        out[f'x{t}'] = traj[t][0].cpu().numpy()
        out[f'v{t}'] = traj[t][1].cpu().argmax(-1).numpy().astype(np.int16)
    np.savez_compressed(os.path.join(HERE, 'trajectory_c1_T50.npz'), **out)
    print('c1 T=50: final |x| max', float(np.abs(out['x-1']).max()), 'types', out['v-1'])


if __name__ == '__main__':
    main()
