"""Generate tests/golden/eval_loss.npz from the UNMODIFIED reference's eval-mode ``TargetDiff.forward``.

Run where a checkout of the reference exists (tests/golden/ref_shims.py: REF_ROOT):

    python tests/golden/make_golden_f5.py

``model.eval(); model(batch)`` is the validation loss of the reference (train.py ``validate``): for each of the
``eval_interval`` timesteps it noises the batch, runs the denoiser and reduces the position / type losses.  Its
``torch.randn_like`` / ``torch.rand_like`` draws are replaced by seeded tensors handed out in call order (for each t:
positions, then types), the same tensors the tests inject.  Inputs and weights are regenerated bit-identically from
seeds (cbgbench_b200/synthetic.py); only outputs are stored.  The CPU oracle (tests/eval_loss_oracle.py) is checked
against the reference on every case before anything is written.
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
import eval_loss_oracle as EO  # noqa: E402
from cbgbench_b200 import synthetic  # noqa: E402
from cbgbench_b200.targetdiff import TargetDiffB200  # noqa: E402

# (name, T, eval_interval, n_prot, n_lig, data seed, gen_mode, graphs without generated atoms, noise seed)
EVAL_CASES = [
    ('ragged_denovo', 1000, 10, [120, 60, 40], [20, 12, 7], 41, 'denovo', [], 51),     # t = 0 ... 999
    ('partial_mid_empty', 1000, 10, [80, 60, 50], [15, 10, 12], 42, 'partial', [1], 52),
    ('t50_interval7', 50, 7, [90, 70], [14, 9], 43, 'denovo', [], 53),                   # truncation of linspace
    ('interval1', 1000, 1, [100, 50], [16, 8], 44, 'denovo', [], 54),                    # t = 0 only
]
WEIGHT_SEED = 0


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
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    ref_shims.install()
    from repo.utils.evaluate import AUROC
    out = {}
    for name, T, interval, n_prot, n_lig, seed, gen_mode, empty, noise_seed in EVAL_CASES:
        cfg = ref_shims.targetdiff_cfg(num_steps=T)
        cfg['eval_interval'] = interval
        ref = ref_shims.load_targetdiff(cfg)
        sd = synthetic.seeded_state_dict(TargetDiffB200(synthetic.targetdiff_config(num_steps=T)), seed=WEIGHT_SEED)
        ref.load_state_dict(sd, strict=True)
        batch = case_batch(n_prot, n_lig, seed, gen_mode, empty)
        t_values = EO.eval_t_values(T, interval)
        R, n = len(t_values), batch['ligand_pos'].shape[0]
        pn, tu = synthetic.make_noise(R, n, 13, seed=noise_seed)
        queue = {'randn': list(pn), 'rand': list(tu)}
        orig = torch.randn_like, torch.rand_like
        torch.randn_like = lambda a, *aa, **kk: queue['randn'].pop(0)
        torch.rand_like = lambda a, *aa, **kk: queue['rand'].pop(0)
        try:
            loss, results = ref(batch)
        finally:
            torch.randn_like, torch.rand_like = orig
        assert queue == {'randn': [], 'rand': []}, {k: len(v) for k, v in queue.items()}
        assert len(results) == R
        o_loss, o_res, o_per_t = EO.eval_losses(sd, batch, t_values, pn, tu)
        for key in ('pos', 'atom'):
            assert loss[key].dtype == torch.float32 and loss[key].dim() == 0
            err = abs(float(o_loss[key]) - float(loss[key])) / max(abs(float(loss[key])), 1e-30)
            assert err < 1e-6, (name, key, float(o_loss[key]), float(loss[key]))
        for r in range(R):
            for key in ('xt', 'x_pred', 'c_pred'):
                err = float((o_res[r][key] - results[r][key]).abs().max()) / max(float(results[r][key].abs().max()), 1e-30)
                assert err < 1e-6, (name, r, key, err)
            for key in ('vt', 'v0', 'mask_gen', 'x0'):
                assert torch.equal(o_res[r][key], results[r][key]), (name, r, key)
        auroc = AUROC(true_key='v0', pred_key='c_pred', mask_key='mask_gen')(results)
        assert abs(EO.auroc(results) - auroc) < 1e-12
        out[f'{name}/t_values'] = np.asarray(t_values, dtype=np.int64)
        out[f'{name}/pos'] = loss['pos'].numpy()
        out[f'{name}/atom'] = loss['atom'].numpy()
        out[f'{name}/per_t'] = np.asarray([[float(p), float(a)] for p, a in o_per_t], dtype=np.float32)
        for key in ('xt', 'x_pred', 'c_pred', 'vt'):
            out[f'{name}/{key}'] = torch.stack([res[key] for res in results]).numpy()
        out[f'{name}/auroc'] = np.float64(auroc)
        print(f'{name}: t={t_values} pos={float(loss["pos"]):.6g} atom={float(loss["atom"]):.6g} auroc={auroc:.4f}')
    np.savez_compressed(os.path.join(HERE, 'eval_loss.npz'), **out)


if __name__ == '__main__':
    main()
