"""Generate tests/golden/bp_eval_loss.npz from the UNMODIFIED reference's eval-mode ``DiffBP.forward``.

Run where a checkout of the reference exists (tests/golden/ref_shims.py: REF_ROOT):

    python tests/golden/make_golden_f6.py

``model.eval(); model(batch)`` is DiffBP's validation loss (train.py ``validate``): for each of the ``eval_interval``
timesteps it noises the batch, runs the denoiser and the CoM head, and reduces the position, CoM, masked-type and
interior losses.  Its ``torch.randn_like`` / ``torch.rand_like`` draws are replaced by seeded tensors handed out in
call order (for each t: positions [n_lig,3], then the type mask [n_lig]), the same tensors the tests inject.  The shims
give a MagicMock for ``torch_geometric.nn.knn``; the interior loss's module-level ``knn`` is patched here with the
restatement of tests/bp_eval_loss_oracle.py (ref_shims.install itself is unchanged, so the other fixtures regenerate
byte-identically).  Inputs and weights are regenerated bit-identically from seeds (cbgbench_b200/synthetic.py); only
outputs are stored.  The CPU oracle is checked against the reference on every case before anything is written.
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
import bp_eval_loss_oracle as BO  # noqa: E402
from make_golden_f2 import easy  # noqa: E402
from cbgbench_b200 import synthetic  # noqa: E402
from cbgbench_b200.diffbp import DiffBPB200  # noqa: E402

# (name, T, eval_interval, n_prot, n_lig, data seed, gen_mode, graphs without generated atoms, noise seed)
BP_EVAL_CASES = [
    ('ragged_denovo', 1000, 10, [120, 60, 90], [20, 12, 60], 141, 'denovo', [], 151),      # graph 2: 60 > 48 atoms
    ('partial_empty', 1000, 10, [80, 60, 50, 40], [15, 10, 12, 9], 142, 'partial', [1, 3], 152),
    ('t50_interval7', 50, 7, [90, 70], [14, 9], 143, 'denovo', [], 153),
    ('interval1', 1000, 1, [100, 50], [16, 8], 144, 'denovo', [], 154),                     # t = 0 only: atom = 0
]
WEIGHT_SEED = 0
VEC_KEYS = ('eps_0', 'eps_pred', 'score_0', 'score_pred', 'eps_0_com', 'eps_pred_com', 'score_0_com', 'score_pred_com')


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
    import repo.models.diffusion.diffbp as ref_diffbp
    from repo.utils.evaluate import AUROC
    ref_diffbp.knn = BO.knn
    out = {}
    for name, T, interval, n_prot, n_lig, seed, gen_mode, empty, noise_seed in BP_EVAL_CASES:
        cfg = synthetic.diffbp_config(num_steps=T)
        cfg['eval_interval'] = interval
        ref = ref_diffbp.DiffBP(easy(cfg)).eval()
        sd = synthetic.seeded_state_dict(DiffBPB200(synthetic.diffbp_config(num_steps=T)), seed=WEIGHT_SEED)
        ref.load_state_dict(sd, strict=True)
        batch = case_batch(n_prot, n_lig, seed, gen_mode, empty)
        t_values = BO.eval_t_values(T, interval)
        R, n = len(t_values), batch['ligand_pos'].shape[0]
        pn, tu = synthetic.make_bp_noise(R, n, seed=noise_seed)
        queue = {'randn': list(pn), 'rand': list(tu)}
        orig = torch.randn_like, torch.rand_like
        torch.randn_like = lambda a, *aa, **kk: queue['randn'].pop(0)
        torch.rand_like = lambda a, *aa, **kk: queue['rand'].pop(0)
        try:
            loss, results = ref(batch)
        finally:
            torch.randn_like, torch.rand_like = orig
        assert queue == {'randn': [], 'rand': []}, {k: len(v) for k, v in queue.items()}
        assert len(results) == R and set(loss) == {'pos', 'atom', 'com', 'inter'}
        o_loss, o_res, o_per_t = BO.eval_losses(sd, batch, t_values, pn, tu, T)
        for key in ('pos', 'atom', 'com', 'inter'):
            assert loss[key].dtype == torch.float32 and loss[key].dim() == 0
            want, got = float(loss[key]), float(o_loss[key])
            assert (np.isnan(want) and np.isnan(got)) or abs(got - want) <= 1e-6 * abs(want), (name, key, got, want)
        for r in range(R):
            assert set(results[r]) == set(BO.RESULT_KEYS), sorted(results[r])
            for key in VEC_KEYS + ('c_pred',):
                err = float((o_res[r][key] - results[r][key]).abs().max()) / max(float(results[r][key].abs().max()), 1e-30)
                assert err < 1e-6, (name, r, key, err)
            for key in ('vt', 'v0', 'mask_gen', 'mask_gen_com'):
                assert torch.equal(o_res[r][key], results[r][key]), (name, r, key)
        auroc = AUROC(true_key='v0', pred_key='c_pred', mask_key='mask_gen')(results)
        o_auroc = BO.auroc(results)
        assert (np.isnan(auroc) and np.isnan(o_auroc)) or abs(o_auroc - auroc) < 1e-12
        out[f'{name}/t_values'] = np.asarray(t_values, dtype=np.int64)
        for key in ('pos', 'atom', 'com', 'inter'):
            out[f'{name}/{key}'] = loss[key].numpy()
        out[f'{name}/per_t'] = np.asarray([[float(v) for v in p] for p in o_per_t], dtype=np.float32)
        for key in VEC_KEYS + ('c_pred', 'vt', 'mask_gen'):
            out[f'{name}/{key}'] = torch.stack([res[key] for res in results]).numpy()
        out[f'{name}/auroc'] = np.float64(auroc)
        print(f'{name}: t={t_values} ' + ' '.join(f'{k}={float(loss[k]):.6g}' for k in ('pos', 'atom', 'com', 'inter'))
              + f' auroc={auroc:.4f}')
    np.savez_compressed(os.path.join(HERE, 'bp_eval_loss.npz'), **out)


if __name__ == '__main__':
    main()
