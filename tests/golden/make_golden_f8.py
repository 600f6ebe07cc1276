"""Golden fixtures of the D3FG sampler from the UNMODIFIED reference ``D3FG.sample``
(/root/reference repo/models/diffusion/difffg.py:174-246), imported through tests/golden/ref_shims.py.

    python tests/golden/make_golden_f8.py          (needs a checkout of the reference)

The batch, weights and draws are regenerated bit-identically by the tests (numpy RandomState seeds in CASE below and
cbgbench_b200.synthetic); only OUTPUTS are stored.  The reference's random calls are fed from a queue in its own order
(randn_like positions, randn axes, multinomial, rand_like in-bin offset, randn_like Gaussian branch, rand_like Gumbel),
and its ``torch.multinomial`` is replaced by the definition ``cbgbench_b200.difffg.multinomial_bin``.  Checked here:
the host module's state-dict keys, shapes and angular buffers equal the reference's, the oracle
(tests/fg_sample_oracle.py) equals the reference to 1e-5 at every step, and the fixture hits both the Gaussian and the
histogram branch of the angle draw.  Writes fg_trajectory.npz, fg_state_keys.json.
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

# (T, hidden, num_layers, residues per graph, FGs per graph, batch seed, partial graphs, weight seed, draw seed)
CASE = dict(T=20, hidden=256, num_layers=2, n_res=[42, 70, 24], n_fg=[6, 9, 4], seed=8, partial=(2,), wseed=3, dseed=9)
Y_ROWS = (2, 10, 19)     # stored rows of angular_distrib_inv.Y


def ref_cfg(T, hidden, num_layers):
    c = synthetic.difffg_config(num_steps=T, num_layers=num_layers, hidden=hidden)
    return ref_shims.EasyDict(json.loads(json.dumps(c)))


def build_inputs(model):
    c = CASE
    sd = synthetic.seeded_state_dict(model, seed=c['wseed'])
    batch = synthetic.make_fg_batch(c['n_res'], c['n_fg'], seed=c['seed'], partial_graphs=c['partial'])
    draws = synthetic.make_fg_draws(c['T'], sum(c['n_fg']), seed=c['dseed'])
    return sd, batch, draws


class DrawQueue:
    """Feeds the reference's random calls from the injected draws, checking order and shapes."""

    def __init__(self, T, draws):
        pos, rot, typ = draws
        self.items = []
        for t in reversed(range(T)):
            self.items += [('randn_like', pos[t]), ('randn', rot[t, :, 0:3]), ('multinomial', rot[t, :, 3]),
                           ('rand_like', rot[t, :, 4]), ('randn_like', rot[t, :, 5]), ('rand_like', typ[t])]

    def pop(self, kind, shape):
        k, v = self.items.pop(0)
        assert k == kind and tuple(v.shape) == tuple(shape), (k, kind, tuple(v.shape), tuple(shape))
        return v.clone()

    def install(self):
        from cbgbench_b200.difffg import multinomial_bin
        self.saved = {n: getattr(torch, n) for n in ('randn_like', 'randn', 'rand_like', 'multinomial')}
        torch.randn_like = lambda x, **kw: self.pop('randn_like', x.shape)
        torch.rand_like = lambda x, **kw: self.pop('rand_like', x.shape)
        torch.randn = lambda size, **kw: self.pop('randn', size)
        torch.multinomial = lambda prob, num_samples=1, **kw: multinomial_bin(
            prob, self.pop('multinomial', prob.shape[:1])).unsqueeze(-1)

    def restore(self):
        for n, f in self.saved.items():
            setattr(torch, n, f)


def main():
    ref_shims.install()
    torch.set_grad_enabled(False)
    from repo.models.diffusion.difffg import D3FG
    from cbgbench_b200.difffg import D3FGB200
    import fg_sample_oracle as OF
    c = CASE
    T = c['T']
    ref = D3FG(ref_cfg(T, c['hidden'], c['num_layers'])).eval()
    ours = D3FGB200(synthetic.difffg_config(num_steps=T, num_layers=c['num_layers'], hidden=c['hidden']))
    rsd, osd = ref.state_dict(), ours.state_dict()
    assert list(rsd.keys()) == list(osd.keys())
    for k in rsd:
        assert rsd[k].shape == osd[k].shape and rsd[k].dtype == osd[k].dtype, k
        if not k.startswith(('context_embedder.', 'denoiser.')) or k.endswith('freq_bands'):
            assert torch.equal(rsd[k], osd[k]), k          # schedules and angular histograms: bit for bit
    sd, batch, draws = build_inputs(ours)
    ref.load_state_dict(sd, strict=True)
    flags = sd['rot_scheduler.angular_distrib_inv.approx_flag'][2:]
    assert bool(flags.any()) and bool((~flags).any()), 'the fixture must hit both angle branches'
    q = DrawQueue(T, draws)
    q.install()
    try:
        traj = ref.sample(batch)
    finally:
        q.restore()
    assert not q.items
    want = OF.sample(sd, batch, T, *draws)
    out = {}
    for t in range(-1, T):
        for j, nm in enumerate(('xc', 'c', 'o')):
            a, w = traj[t][j].float(), want[t][j]
            err = float((a - w).abs().max() / (w.abs().max() + 1e-12))
            assert err < 1e-5, (t, nm, err)
            out[f't{t}/{nm}'] = a.numpy()
    for r in Y_ROWS:
        out[f'Y{r}'] = rsd['rot_scheduler.angular_distrib_inv.Y'][r].numpy()
    np.savez_compressed(os.path.join(HERE, 'fg_trajectory.npz'), **out)
    with open(os.path.join(HERE, 'fg_state_keys.json'), 'w') as f:
        json.dump({k: list(v.shape) for k, v in rsd.items()}, f, indent=0)
    print('ok: T =', T, 'FGs =', sum(c['n_fg']), 'changed types:',
          int((traj[-1][1].argmax(-1) != traj[T - 1][1].argmax(-1)).sum()))


if __name__ == '__main__':
    main()
