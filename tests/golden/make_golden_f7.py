"""Generate tests/golden/sbdd_eval_loss.npz from the UNMODIFIED reference's eval-mode ``DiffSBDD.forward``.

Run where a checkout of the reference exists (tests/golden/ref_shims.py: REF_ROOT):

    python tests/golden/make_golden_f7.py

``model.eval(); model(batch)`` is DiffSBDD's validation loss (train.py ``validate``): for each of the ``eval_interval``
timesteps t it noises the batch at t and at 0, runs the denoiser on both copies, and reduces the variational position
and type losses.  Its four ``torch.randn_like`` draws per t are replaced by seeded tensors handed out in call order
(positions at t, types at t, positions at 0, types at 0), the same tensors the tests inject.  Inputs and weights are
regenerated bit-identically from seeds (cbgbench_b200/synthetic.py); only outputs are stored.  The CPU oracle
(tests/sbdd_eval_loss_oracle.py) is checked against the reference on every case before anything is written.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import ref_shims  # noqa: E402
import sbdd_eval_loss_oracle as SO  # noqa: E402
from make_golden_f2 import easy  # noqa: E402
from cbgbench_b200 import synthetic  # noqa: E402
from cbgbench_b200.diffsbdd import DiffSBDDB200  # noqa: E402

# (name, T, eval_interval, n_prot, n_lig, data seed, gen_mode, graphs without generated atoms, noise seed)
SBDD_EVAL_CASES = [
    ('ragged_denovo', 1000, 10, [120, 60, 90], [20, 12, 30], 241, 'denovo', [], 251),       # t = T is the last t
    ('partial_empty', 1000, 10, [80, 60, 50, 40], [15, 10, 12, 9], 242, 'partial', [1], 252),
    ('middle_empty_one_atom', 1000, 10, [70, 50, 40], [14, 0, 1], 243, 'denovo', [], 253),
    ('t50_interval7', 50, 7, [90, 70], [14, 9], 244, 'denovo', [], 254),
    ('interval1', 1000, 1, [100, 50], [16, 8], 245, 'denovo', [], 255),                      # t = 1 only
]
WEIGHT_SEED = 0
K = 13
VEC_KEYS = ('eps_0_pos', 'eps_pred_pos', 'score_0_pos', 'score_pred_pos',
            'eps_0_atom', 'eps_pred_atom', 'score_0_atom', 'score_pred_atom')


def case_batch(n_prot, n_lig, seed, gen_mode, empty_graphs):
    batch = synthetic.make_batch(n_prot, n_lig, seed=seed, gen_mode=gen_mode)
    if empty_graphs:
        gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag']).clone()
        for g in empty_graphs:
            gen[batch['ligand_element_batch'] == g] = False
        batch['ligand_gen_flag'] = gen
    return batch


def main():
    torch.set_grad_enabled(False)
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
    ref_shims.install()
    from repo.models.diffusion.diffsbdd import DiffSBDD
    out = {}
    for name, T, interval, n_prot, n_lig, seed, gen_mode, empty, noise_seed in SBDD_EVAL_CASES:
        cfg = synthetic.diffsbdd_config(num_steps=T)
        cfg['eval_interval'] = interval
        ref = DiffSBDD(easy(cfg)).eval()
        sd = synthetic.seeded_state_dict(DiffSBDDB200(synthetic.diffsbdd_config(num_steps=T)), seed=WEIGHT_SEED)
        ref.load_state_dict(sd, strict=True)
        batch = case_batch(n_prot, n_lig, seed, gen_mode, empty)
        t_values = SO.eval_t_values(T, interval)
        R, n = len(t_values), batch['ligand_pos'].shape[0]
        noise = synthetic.make_sbdd_eval_noise(R, n, K, seed=noise_seed)
        queue = [noise[key][j] for j in range(R) for key in ('x_t', 'c_t', 'x_0', 'c_0')]
        orig = torch.randn_like

        def draw(a, *aa, **kk):
            d = queue.pop(0)
            assert d.shape == a.shape and d.dtype == a.dtype, (d.shape, a.shape)
            return d
        torch.randn_like = draw
        try:
            loss, results = ref(batch)
        finally:
            torch.randn_like = orig
        assert queue == [], len(queue)
        assert len(results) == R and list(loss) == ['pos', 'atom']
        o_loss, o_res, o_per_t, o_terms = SO.eval_losses(sd, batch, t_values, noise, T, K)
        for key in ('pos', 'atom'):
            assert loss[key].dtype == torch.float32 and loss[key].dim() == 0 and loss[key].device.type == 'cpu'
            want, got = float(loss[key]), float(o_loss[key])
            assert abs(got - want) <= 1e-6 * abs(want), (name, key, got, want)
        for r in range(R):
            assert list(results[r]) == list(SO.RESULT_KEYS), list(results[r])
            for key in VEC_KEYS:
                err = float((o_res[r][key] - results[r][key]).abs().max()) / max(float(results[r][key].abs().max()), 1e-30)
                assert err < 1e-6, (name, r, key, err)
            for key in ('mask_gen_pos', 'mask_gen_atom'):
                assert torch.equal(o_res[r][key], results[r][key]), (name, r, key)
        out[f'{name}/t_values'] = np.asarray(t_values, dtype=np.int64)
        for key in ('pos', 'atom'):
            out[f'{name}/{key}'] = loss[key].numpy()
        out[f'{name}/per_t'] = np.asarray([[float(v) for v in p] for p in o_per_t], dtype=np.float32)
        out[f'{name}/terms'] = o_terms.numpy()
        for key in VEC_KEYS + ('mask_gen_pos',):
            out[f'{name}/{key}'] = torch.stack([res[key] for res in results]).numpy()
        print(f'{name}: t={t_values} ' + ' '.join(f'{k}={float(loss[k]):.6g}' for k in ('pos', 'atom')))
    np.savez_compressed(os.path.join(HERE, 'sbdd_eval_loss.npz'), **out)


if __name__ == '__main__':
    main()
