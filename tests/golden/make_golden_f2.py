"""Golden fixtures for SURVEY.md section 8 row f2 (DiffSBDD / DiffBP samplers) from the UNMODIFIED reference.

Run where a checkout of the reference exists (tests/golden/ref_shims.py: REF_ROOT):

    python tests/golden/make_golden_f2.py

Like make_golden.py: the reference ships no known-answer vectors, so the fixtures are outputs of the reference's own
``DiffSBDD.sample`` / ``DiffBP.sample`` (imported through tests/golden/ref_shims.py) on seeded synthetic inputs and
seeded weights that the tests regenerate bit-identically; only OUTPUTS are stored.  The random draws of the
reference (``torch.randn`` / ``torch.randn_like`` / ``torch.rand_like``) are replaced by queued seeded tensors.

Files written next to this script:
  sbdd_trajectory.npz   DiffSBDD.sample over T=10 steps (+ final stage), 2 pockets
  sbdd_state_keys.json  DiffSBDD state-dict keys and shapes
  bp_trajectory.npz     DiffBP.sample over T=10 steps, 2 pockets (ligand types start at the absorbing state
                        except a few atoms), plus eps / eps_com of the first step
  bp_state_keys.json    DiffBP state-dict keys and shapes
"""
import json
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
from cbgbench_b200.diffsbdd import DiffSBDDB200  # noqa: E402
from cbgbench_b200.diffbp import DiffBPB200  # noqa: E402

WEIGHT_SEED = 0


def easy(cfg):
    """cbgbench_b200.synthetic.Cfg -> the shim's EasyDict (the reference calls cfg.get / attribute access)."""
    def plain(c):
        return {k: plain(v) if isinstance(v, dict) else v for k, v in dict(c).items()}
    return ref_shims.EasyDict(plain(cfg))


def sbdd():
    ref_shims.install()
    from repo.models.diffusion.diffsbdd import DiffSBDD
    T = 10
    cfg = synthetic.diffsbdd_config(num_steps=T)
    ref = DiffSBDD(easy(cfg)).eval()
    weights = synthetic.seeded_state_dict(DiffSBDDB200(synthetic.diffsbdd_config(num_steps=T)), seed=WEIGHT_SEED)
    ref.load_state_dict(weights, strict=True)
    with open(os.path.join(HERE, 'sbdd_state_keys.json'), 'w') as f:
        json.dump({k: list(v.shape) for k, v in ref.state_dict().items()}, f, indent=0)
    batch = synthetic.make_batch([150, 60], [20, 9], seed=31)
    n_lig = batch['ligand_pos'].shape[0]
    noise = synthetic.make_sbdd_noise(T, n_lig, 13, seed=9)
    queue = [noise['init_x'], noise['init_c']]
    for t in reversed(range(T)):
        queue += [noise['step_x'][t], noise['step_c'][t]]
    queue += [noise['final_x'], noise['final_c']]
    calls = {'n': 0}
    orig = torch.randn

    def fake_randn(*size, **kw):
        shape = tuple(size[0]) if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)) else tuple(size)
        v = queue[calls['n']]
        assert tuple(v.shape) == shape, (calls['n'], v.shape, shape)
        calls['n'] += 1
        return v.clone()

    torch.randn = fake_randn
    try:
        traj = ref.sample(batch)
    finally:
        torch.randn = orig
    assert calls['n'] == len(queue), calls
    out = {}
    for t in range(-1, T):
        out[f'x{t}'] = traj[t][0].cpu().numpy()
        out[f'c{t}'] = traj[t][1].cpu().numpy()
    from repo.models.diffusion.schedule_utils import PredefinedNoiseSchedule
    out['gamma_T10'] = ref.state_dict()['pos_scheduler.gamma.gamma'].numpy()
    out['gamma_T1000'] = PredefinedNoiseSchedule('polynomial_2', timesteps=1000, precision=5e-4).gamma.numpy()
    np.savez_compressed(os.path.join(HERE, 'sbdd_trajectory.npz'), **out)
    print('sbdd: final |x|max', float(np.abs(out['x0']).max()), ' c0[0,:4]', out['c0'][0, :4])

    # the oracle restatement against the live reference, same inputs
    from oracle import diffusion_sbdd
    otraj, _ = diffusion_sbdd.sample({k: v.clone() for k, v in weights.items()}, batch, T, noise)
    for t in range(-1, T):
        dx = float((otraj[t][0] - traj[t][0].cpu()).abs().max())
        dc = float((otraj[t][1] - traj[t][1].cpu()).abs().max())
        assert dx < 1e-5 and dc < 1e-5, (t, dx, dc)
    print('sbdd: oracle == reference (max abs diff < 1e-5 at every step)')


def bp_batch(n_prot, n_lig, seed):
    """Synthetic pockets for DiffBP: ligand atom types start at the absorbing state 0 (what the reference's
    sampling transform assigns), except every 5th atom which keeps a random type (exercises fix_pred)."""
    batch = synthetic.make_batch(n_prot, n_lig, seed=seed)
    v = batch['ligand_atom_type'].clone()
    keep = torch.arange(v.numel()) % 5 == 4
    batch['ligand_atom_type'] = torch.where(keep, v, torch.zeros_like(v))
    return batch


def bp():
    ref_shims.install()
    from repo.models.diffusion.diffbp import DiffBP
    T = 10
    ref = DiffBP(easy(synthetic.diffbp_config(num_steps=T))).eval()
    weights = synthetic.seeded_state_dict(DiffBPB200(synthetic.diffbp_config(num_steps=T)), seed=WEIGHT_SEED)
    ref.load_state_dict(weights, strict=True)
    with open(os.path.join(HERE, 'bp_state_keys.json'), 'w') as f:
        json.dump({k: list(v.shape) for k, v in ref.state_dict().items()}, f, indent=0)
    batch = bp_batch([150, 60], [20, 9], seed=41)
    n_lig = batch['ligand_pos'].shape[0]
    pn, tu = synthetic.make_bp_noise(T, n_lig, seed=13)
    calls = {'randn': 0, 'rand': 0}
    orig_randn, orig_rand = torch.randn_like, torch.rand_like

    def fake_randn_like(a, *aa, **kk):       # diffusion_scheduler.py:158, once per step, t = T-1 ... 0
        t = T - 1 - calls['randn']
        calls['randn'] += 1
        assert tuple(a.shape) == (n_lig, 3)
        return pn[t]

    def fake_rand_like(a, *aa, **kk):        # diffusion_scheduler.py:486
        t = T - 1 - calls['rand']
        calls['rand'] += 1
        assert tuple(a.shape) == (n_lig,)
        return tu[t]

    # record eps / eps_com of every step through the reference's own com_head
    seen = []
    orig_com = ref.com_head.forward

    def spy(*a, **k):
        out = orig_com(*a, **k)
        seen.append((out[0].clone(), out[1].clone()))
        return out

    ref.com_head.forward = spy
    torch.randn_like, torch.rand_like = fake_randn_like, fake_rand_like
    try:
        traj = ref.sample(batch)
    finally:
        torch.randn_like, torch.rand_like = orig_randn, orig_rand
    assert calls == {'randn': T, 'rand': T}, calls
    out = {}
    for t in range(-1, T):
        out[f'x{t}'] = traj[t][0].cpu().numpy()
        out[f'v{t}'] = traj[t][1].cpu().argmax(-1).numpy()
    for i, (e, ec) in enumerate(seen):
        out[f'eps{T - 1 - i}'] = (e + ec).numpy()
    np.savez_compressed(os.path.join(HERE, 'bp_trajectory.npz'), **out)
    print('bp: final |x|max', float(np.abs(out['x-1']).max()), 'types', out['v-1'][:12], '|eps_com|max',
          float(seen[0][1].abs().max()))

    from oracle import diffusion_bp
    otraj = diffusion_bp.sample({k: v.clone() for k, v in weights.items()}, batch, T, pn, tu)
    for t in range(-1, T):
        dx = float((otraj[t][0] - traj[t][0].cpu()).abs().max())
        assert dx < 1e-5, (t, dx)
        assert torch.equal(otraj[t][1].argmax(-1), traj[t][1].cpu().argmax(-1)), t
    print('bp: oracle == reference (x max abs diff < 1e-5, types equal at every step)')


def main():
    torch.set_grad_enabled(False)
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
    if len(sys.argv) < 2 or sys.argv[1] == 'sbdd':
        sbdd()
    if len(sys.argv) < 2 or sys.argv[1] == 'bp':
        bp()


if __name__ == '__main__':
    main()
