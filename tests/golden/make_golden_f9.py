"""Golden fixtures of the D3FG validation losses from the UNMODIFIED reference's eval-mode ``D3FG.forward``
(/root/reference repo/models/diffusion/difffg.py:65-171 for ``difffg``, :283-389 for ``difffg_v2``), imported through
tests/golden/ref_shims.py.

    python tests/golden/make_golden_f9.py          (needs a checkout of the reference)

``model.eval(); model(batch)`` under ``torch.no_grad`` is the validation loss of the reference (train.py ``validate``).
Both classes are taken from the reference's registry: ``from repo.models.diffusion.difffg import D3FG`` binds the second
definition (``difffg_v2``) only.  The reference's random calls are fed from a queue in its own order (per timestep:
randn_like positions, randn axes, multinomial, rand_like in-bin offset, randn_like Gaussian branch, rand_like Gumbel), its
``torch.multinomial`` is replaced by the definition ``cbgbench_b200.difffg.multinomial_bin``.  The batch, weights and
draws are regenerated bit-identically by the tests from the seeds in CASES; only OUTPUTS are stored.  Checked here
before anything is written: the oracle (tests/fg_eval_loss_oracle.py) equals the reference to 1e-6, the fixtures hit
both branches of the forward angle draw, and no generated FG's noised rotation angle lies within 0.05 of pi (where the
reference's fp32 log map, so3.py:10-22, loses its accuracy).  Writes fg_eval_loss.npz.
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
sys.path.insert(0, os.path.dirname(HERE))

import ref_shims  # noqa: E402
from cbgbench_b200 import synthetic  # noqa: E402

HIDDEN, NUM_LAYERS, WEIGHT_SEED = 256, 2, 3
# name -> (T, eval_interval, residues per graph, FGs per graph, batch seed, partial graphs, graphs without generated FGs,
#          draw seed)
CASES = {
    'ragged': (20, 10, [42, 70, 24], [6, 9, 4], 8, (), (), 41),
    'partial_mid_empty': (20, 10, [40, 30, 50, 36], [7, 0, 6, 5], 11, (0,), (3,), 33),
    'interval1': (20, 1, [38, 52], [5, 8], 12, (), (), 33),
    'one_fg': (20, 10, [30], [1], 13, (), (), 31),
}
MODELS = ('difffg', 'difffg_v2')
NEAR_PI = 0.05


def case_batch(name):
    T, interval, n_res, n_fg, seed, partial, no_gen, dseed = CASES[name]
    batch = synthetic.make_fg_batch(n_res, n_fg, seed=seed, partial_graphs=partial)
    if no_gen:
        gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag']).clone()
        for g in no_gen:
            gen[batch['ligand_type_fg_batch'] == g] = False
        batch['ligand_gen_flag'] = gen
    return batch


def case_draws(name, R):
    """pos [R,n,3], rot [R,n,6], type [R,n,K]: make_fg_draws with the eval timesteps in place of the sampling steps."""
    T, interval, n_res, n_fg, seed, partial, no_gen, dseed = CASES[name]
    return synthetic.make_fg_draws(R, sum(n_fg), seed=dseed)


def case_t_values(name):
    from cbgbench_b200.targetdiff import eval_t_values
    T, interval = CASES[name][:2]
    return eval_t_values(T, interval)


def model_cfg(name, model):
    T, interval = CASES[name][:2]
    c = synthetic.difffg_config(num_steps=T, num_layers=NUM_LAYERS, hidden=HIDDEN)
    c['type'] = model
    c['eval_interval'] = interval
    return c


def weights(T):
    from cbgbench_b200.difffg import D3FGB200
    return synthetic.seeded_state_dict(D3FGB200(synthetic.difffg_config(num_steps=T, num_layers=NUM_LAYERS,
                                                                         hidden=HIDDEN)), seed=WEIGHT_SEED)


class DrawQueue:
    """Feeds the reference's random calls of one eval-mode forward from the injected draws, checking order and shapes."""

    def __init__(self, draws):
        pos, rot, typ = draws
        self.items = []
        for r in range(pos.shape[0]):
            self.items += [('randn_like', pos[r]), ('randn', rot[r, :, 0:3]), ('multinomial', rot[r, :, 3]),
                           ('rand_like', rot[r, :, 4]), ('randn_like', rot[r, :, 5]), ('rand_like', typ[r])]

    def pop(self, kind, shape):
        k, v = self.items.pop(0)
        assert k == kind and tuple(v.shape) == tuple(shape), (k, kind, tuple(v.shape), tuple(shape))
        return v.clone()

    def install(self):
        from cbgbench_b200.difffg import multinomial_bin
        self.saved = {n: getattr(torch, n) for n in ('randn_like', 'randn', 'rand_like', 'multinomial')}
        torch.randn_like = lambda x, **kw: self.pop('randn_like', x.shape)
        torch.rand_like = lambda x, **kw: self.pop('rand_like', x.shape)
        torch.randn = lambda *size, **kw: self.pop('randn', size[0] if len(size) == 1 else size)
        torch.multinomial = lambda prob, num_samples=1, **kw: multinomial_bin(
            prob, self.pop('multinomial', prob.shape[:1])).unsqueeze(-1)

    def restore(self):
        for n, f in self.saved.items():
            setattr(torch, n, f)


def main():
    ref_shims.install()
    torch.set_grad_enabled(False)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    import repo.models.diffusion.difffg  # noqa: F401  (registers difffg and difffg_v2)
    from repo.models._base import _MODEL_DICT
    from repo.utils.evaluate import AUROC
    import fg_eval_loss_oracle as OE
    out = {}
    branches = set()
    for name in CASES:
        T = CASES[name][0]
        sd = weights(T)
        batch = case_batch(name)
        ref_batch = dict(batch, ligand_mask_heavyatom=torch.ones(batch['ligand_pos_heavyatom'].shape[:2], dtype=torch.bool))
        t_values = case_t_values(name)
        R = len(t_values)
        draws = case_draws(name, R)
        gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag'])
        ang = OE.noised_angles_f64(sd, batch, t_values, draws[1])
        worst = float((np.pi - ang[:, gen]).min())
        assert worst > NEAR_PI, (name, 'a generated FG is noised to within 0.05 of pi: change the draw seed', worst)
        flags = sd['rot_scheduler.angular_distrib_fwd.approx_flag']
        if bool(gen.any()):
            branches |= {bool(flags[t]) for t in t_values}
        for model in MODELS:
            ref = _MODEL_DICT[model](ref_shims.EasyDict(json.loads(json.dumps(model_cfg(name, model))))).eval()
            ref.load_state_dict(sd, strict=True)
            q = DrawQueue(draws)
            q.install()
            try:
                loss, results = ref(ref_batch)
            finally:
                q.restore()
            assert not q.items
            assert len(results) == R
            form = 'score' if model == 'difffg' else 'denoise'
            o_loss, o_res, per_t, ot = OE.eval_losses(sd, batch, t_values, *draws, form=form)
            key = f'{name}/{model}'
            for k in ('pos', 'rot', 'fg'):
                a, b = float(loss[k]), float(o_loss[k])
                assert loss[k].dtype == torch.float32 and loss[k].dim() == 0
                assert (np.isnan(a) and np.isnan(b)) or abs(a - b) <= 1e-6 * max(abs(a), 1e-30), (key, k, a, b)
                out[f'{key}/{k}'] = loss[k].numpy()
            for r in range(R):
                assert list(results[r]) == list(o_res[r]), (key, list(results[r]), list(o_res[r]))
                for k, v in results[r].items():
                    w = o_res[r][k]
                    if v.dtype in (torch.int64, torch.bool):
                        assert torch.equal(v, w), (key, r, k)
                    else:
                        err = float((v - w).abs().max()) / max(float(v.abs().max()), 1e-30)
                        assert err < 1e-6, (key, r, k, err)
            for k in results[0]:
                if k not in ('mask_gen', 'v0', 'x0', 'eps_0', 'R0'):
                    out[f'{key}/{k}'] = torch.stack([res[k] for res in results]).numpy()
            out[f'{key}/R0'] = results[0]['R0'].numpy()
            out[f'{key}/per_t'] = per_t.numpy()
            auroc = AUROC(true_key='v0', pred_key='c_pred', mask_key='mask_gen')(results) if bool(gen.any()) else np.nan
            out[f'{key}/auroc'] = np.float64(auroc)
            print(f'{key}: t={t_values} pos={float(loss["pos"]):.6g} rot={float(loss["rot"]):.6g} '
                  f'fg={float(loss["fg"]):.6g} auroc={float(auroc):.4f} closest to pi={worst:.3f}')
    assert branches == {True, False}, 'the fixtures must hit both branches of the forward angle draw'
    np.savez_compressed(os.path.join(HERE, 'fg_eval_loss.npz'), **out)


if __name__ == '__main__':
    main()
