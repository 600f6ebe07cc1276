"""Golden fixtures of SURVEY.md section 8 row f4 from the UNMODIFIED reference `IPATransformer`
(/root/reference repo/modules/e3nn/itatransformer.py), imported through tests/golden/ref_shims.py.

    python tests/golden/make_golden_f4.py          (needs a checkout of the reference)

Inputs and weights are regenerated bit-identically by the tests (numpy RandomState seeds below, weights through
cbgbench_b200.synthetic.seeded_state_dict on the host module, whose state-dict keys equal the reference's: asserted
here); only OUTPUTS are stored: ipa_cases.npz = eps_pos / h / o_next / R_next / c per case, ipa_state_keys.json.
The oracle restatement (oracle/ipa.py) is checked against the reference on every case (1e-5).
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

IPA_CASES, WEIGHT_SEED, make_inputs = synthetic.IPA_CASES, synthetic.IPA_WEIGHT_SEED, synthetic.make_ipa_inputs


def ipa_cfg(hidden, num_layers, num_classes):
    return ref_shims.EasyDict(dict(type='ipatransformer', node_feat_dim=hidden, n_heads=16, num_layers=num_layers,
                                   num_classes=num_classes))


def main():
    ref_shims.install()
    torch.set_grad_enabled(False)
    from repo.modules.e3nn.itatransformer import IPATransformer
    from cbgbench_b200.ipatransformer import IPATransformerB200
    from oracle import ipa as OI
    out, keys = {}, {}
    for name, hidden, nl, nc, n_nodes, n_lig, seed, gen_mode in IPA_CASES:
        ref = IPATransformer(ipa_cfg(hidden, nl, nc)).eval()
        ours = IPATransformerB200(ipa_cfg(hidden, nl, nc))
        assert list(ref.state_dict().keys()) == list(ours.state_dict().keys())
        assert all(tuple(a.shape) == tuple(b.shape) for a, b in zip(ref.state_dict().values(), ours.state_dict().values()))
        sd = synthetic.seeded_state_dict(ours, seed=WEIGHT_SEED, skip_prefixes=())
        ref.load_state_dict(sd, strict=True)
        x, o, h, b, lig, gen = make_inputs(hidden, n_nodes, n_lig, seed, gen_mode)
        got = ref(x, o, h, b, lig, gen)
        want = OI.ipatransformer_forward(sd, x, o, h, b, lig, gen)
        for a, w, nm in zip(got, want, ('eps_pos', 'h', 'o_next', 'R_next', 'c')):
            err = float((a - w).abs().max() / (w.abs().max() + 1e-12))
            assert err < 1e-5, (name, nm, err)
            out[f'{name}/{nm}'] = a.numpy()
        keys[name] = {k: list(v.shape) for k, v in ref.state_dict().items()}
        print(name, 'ok:', {nm: float(a.abs().max()) for a, nm in zip(got, ('eps_pos', 'h', 'o_next', 'R_next', 'c'))})
    np.savez_compressed(os.path.join(HERE, 'ipa_cases.npz'), **out)
    with open(os.path.join(HERE, 'ipa_state_keys.json'), 'w') as f:
        json.dump(keys['h256_two_graphs'], f, indent=0)


if __name__ == '__main__':
    main()
