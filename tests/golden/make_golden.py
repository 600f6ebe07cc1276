"""Generate the golden fixtures from the UNMODIFIED reference (/root/reference).

Run where a checkout of the reference exists (tests/golden/ref_shims.py: REF_ROOT):

    python tests/golden/make_golden.py

The reference ships no tests or known-answer vectors for this path (SURVEY.md section 8c), so
the fixtures are outputs of the reference's own modules (TargetDiff, UniTransformer,
CTNVPScheduler, TypeVPScheduler) imported through tests/golden/ref_shims.py, on seeded
synthetic inputs (cbgbench_b200/synthetic.py: numpy RandomState => inputs and weights are
regenerated bit-identically by the tests; only OUTPUTS are stored).

Files written next to this script:
  forward_cases.npz   x/h/c outputs of reference denoiser forwards (several shapes/modes)
  reverse_step.npz    one reference reverse step (positions + types) at three timesteps
  trajectory.npz      reference TargetDiff.sample over T=10 steps with injected noise
  schedules_T1000.npz the 16 schedule tables of the shipped config
  state_keys.json     TargetDiff state-dict keys and shapes
"""
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import ref_shims  # noqa: E402
from cbgbench_b200 import synthetic  # noqa: E402
from cbgbench_b200.targetdiff import TargetDiffB200  # noqa: E402

# (name, n_prot, n_lig, data seed, gen_mode, encoder overrides)
FORWARD_CASES = [
    ('c1_single', [200], [24], 2024, 'denovo', {}),
    ('ragged_small', [200, 40, 20], [24, 10, 5], 11, 'denovo', {}),      # graph 3 has 25 atoms < k+1
    ('partial_gen', [120, 90], [24, 18], 12, 'partial', {}),             # linker/scaffold-like fixed context
    ('k8', [64, 50], [12, 9], 13, 'denovo', {'k': 8}),
    ('tiny_graphs', [1, 2, 0], [1, 3, 4], 14, 'denovo', {}),             # 2-, 5- and 4-atom graphs
]
WEIGHT_SEED = 0


def seeded_weights(num_steps, **enc):
    model = TargetDiffB200(synthetic.targetdiff_config(num_steps=num_steps, **enc))
    return synthetic.seeded_state_dict(model, seed=WEIGHT_SEED)


def reference_forward(ref, batch):
    """embed -> compose -> denoiser exactly as targetdiff.py:155-162 does it."""
    from repo.modules.common import compose_context
    c_lig = F.one_hot(batch['ligand_atom_type'], ref.num_classes).float()
    aa = F.one_hot(batch['protein_aa_type'], 20).float()
    lig_flag, rec_flag = batch['ligand_lig_flag'], batch['protein_lig_flag']
    gen_lig = batch.get('ligand_gen_flag', lig_flag)
    gen_rec = batch.get('protein_gen_flag', torch.zeros_like(rec_flag))
    B = int(batch['ligand_element_batch'].max()) + 1
    t = torch.zeros(B, dtype=torch.long)
    x_lig, x_rec, h_lig, h_rec = ref.context_embedder(
        batch['ligand_pos'], batch['protein_pos'], c_lig, batch['protein_atom_feature'], aa,
        batch['ligand_element_batch'], batch['protein_element_batch'], lig_flag, rec_flag, t)
    ctx, batch_idx, _ = compose_context(
        {'x': x_lig, 'h': h_lig, 'gen_flag': gen_lig, 'lig_flag': lig_flag},
        {'x': x_rec, 'h': h_rec, 'gen_flag': gen_rec, 'lig_flag': rec_flag},
        batch['ligand_element_batch'], batch['protein_element_batch'])
    x, h, c = ref.denoiser(batch_idx=batch_idx, **ctx)
    return ctx, batch_idx, x, h, c


def main():
    torch.set_grad_enabled(False)
    torch.set_num_threads(max(1, os.cpu_count() or 1))

    # ---- forward cases --------------------------------------------------------------------
    out = {}
    for name, n_prot, n_lig, seed, gen_mode, enc in FORWARD_CASES:
        ref = ref_shims.load_targetdiff(ref_shims.targetdiff_cfg(num_steps=10, **enc))
        ref.load_state_dict(seeded_weights(10, **enc), strict=True)
        batch = synthetic.make_batch(n_prot, n_lig, seed=seed, gen_mode=gen_mode)
        ctx, batch_idx, x, h, c = reference_forward(ref, batch)
        out[f'{name}/x_in'] = ctx['x'].numpy()
        out[f'{name}/h_in'] = ctx['h'].numpy()
        out[f'{name}/x'] = x.numpy()
        out[f'{name}/h'] = h.numpy()
        out[f'{name}/c'] = c.numpy()
        print(f'forward {name}: N={x.shape[0]} |dx|max={float((x - ctx["x"]).abs().max()):.4f}')
    np.savez_compressed(os.path.join(HERE, 'forward_cases.npz'), **out)

    # ---- reverse step -----------------------------------------------------------------------
    T = 1000
    ref = ref_shims.load_targetdiff(ref_shims.targetdiff_cfg(num_steps=T))
    rs = np.random.RandomState(5)
    n, K = 37, 13
    bidx = torch.from_numpy(np.sort(rs.randint(0, 3, size=n)))
    gen = torch.from_numpy(rs.rand(n) < 0.8)
    x0 = torch.from_numpy(rs.normal(size=(n, 3)).astype(np.float32))
    xt = torch.from_numpy(rs.normal(size=(n, 3)).astype(np.float32))
    logits = torch.from_numpy((3 * rs.normal(size=(n, K))).astype(np.float32))
    ct = F.one_hot(torch.from_numpy(rs.randint(0, K, size=n)), K).float()
    noise = torch.from_numpy(rs.normal(size=(n, 3)).astype(np.float32))
    uni = torch.from_numpy(rs.random_sample(size=(n, K)).astype(np.float32))
    rev = dict(batch_idx=bidx.numpy(), gen=gen.numpy(), x0=x0.numpy(), xt=xt.numpy(), logits=logits.numpy(),
               ct=ct.numpy(), noise=noise.numpy(), uni=uni.numpy())
    orig_randn, orig_rand = torch.randn_like, torch.rand_like
    for t_idx in (0, 1, 500, 999):
        t = torch.full((3,), t_idx, dtype=torch.long)
        torch.randn_like = lambda a, *aa, **kk: noise
        torch.rand_like = lambda a, *aa, **kk: uni
        try:
            xn = ref.pos_scheduler.backward_remove_noise(x0, xt, t, bidx, gen, type='denoise')
            cn, vn = ref.type_scheduler.backward_remove_noise(logits, ct, t, bidx, gen, pred_logit=True)
        finally:
            torch.randn_like, torch.rand_like = orig_randn, orig_rand
        rev[f't{t_idx}/x_next'] = xn.numpy()
        rev[f't{t_idx}/v_next'] = vn.numpy()
        rev[f't{t_idx}/c_next'] = cn.numpy()
    np.savez_compressed(os.path.join(HERE, 'reverse_step.npz'), **rev)

    # ---- schedule tables of the shipped config ------------------------------------------------
    tabs = {k: v.numpy() for k, v in ref.state_dict().items() if k.startswith(('pos_scheduler.', 'type_scheduler.'))}
    np.savez_compressed(os.path.join(HERE, 'schedules_T1000.npz'), **tabs)
    with open(os.path.join(HERE, 'state_keys.json'), 'w') as f:
        json.dump({k: list(v.shape) for k, v in ref.state_dict().items()}, f, indent=0)

    # ---- short trajectory through the reference's own sample() --------------------------------
    Tt = 10
    ref = ref_shims.load_targetdiff(ref_shims.targetdiff_cfg(num_steps=Tt))
    ref.load_state_dict(seeded_weights(Tt), strict=True)
    batch = synthetic.make_batch([150, 60], [20, 9], seed=21)
    n_lig = batch['ligand_pos'].shape[0]
    pn, tu = synthetic.make_noise(Tt, n_lig, 13, seed=7)
    calls = {'randn': 0, 'rand': 0}

    def fake_randn_like(a, *aa, **kk):      # called once per step, t = Tt-1 ... 0 (diffusion_scheduler.py:163)
        t = Tt - 1 - calls['randn']
        calls['randn'] += 1
        return pn[t]

    def fake_rand_like(a, *aa, **kk):       # categorical.py:27
        t = Tt - 1 - calls['rand']
        calls['rand'] += 1
        return tu[t]

    torch.randn_like, torch.rand_like = fake_randn_like, fake_rand_like
    try:
        traj = ref.sample(batch)
    finally:
        torch.randn_like, torch.rand_like = orig_randn, orig_rand
    assert calls == {'randn': Tt, 'rand': Tt}, calls
    tr = {}
    for t in range(-1, Tt):
        tr[f'x{t}'] = traj[t][0].cpu().numpy()
        tr[f'v{t}'] = traj[t][1].cpu().argmax(-1).numpy()
    np.savez_compressed(os.path.join(HERE, 'trajectory.npz'), **tr)
    print('trajectory: final |x| max', float(np.abs(tr['x-1']).max()), 'types', tr['v-1'][:10])


if __name__ == '__main__':
    main()
