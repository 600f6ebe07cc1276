"""Shared test helpers: seeded models/batches and the golden fixtures."""
import math
import os

import numpy as np
import torch

from cbgbench_b200 import synthetic
from cbgbench_b200.targetdiff import TargetDiffB200

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')

# must match tests/golden/make_golden.py
FORWARD_CASES = [
    ('c1_single', [200], [24], 2024, 'denovo', {}),
    ('ragged_small', [200, 40, 20], [24, 10, 5], 11, 'denovo', {}),
    ('partial_gen', [120, 90], [24, 18], 12, 'partial', {}),
    ('k8', [64, 50], [12, 9], 13, 'denovo', {'k': 8}),
    ('tiny_graphs', [1, 2, 0], [1, 3, 4], 14, 'denovo', {}),
]
WEIGHT_SEED = 0


def golden(name):
    return np.load(os.path.join(GOLDEN, name))


def case_batch(n_prot, n_lig, seed, gen_mode='denovo', empty_graphs=()):
    """synthetic.make_batch, with the ligand atoms of the graphs ``empty_graphs`` not generated (validation-loss cases)."""
    batch = synthetic.make_batch(n_prot, n_lig, seed=seed, gen_mode=gen_mode)
    if empty_graphs:
        gen = batch.get('ligand_gen_flag', batch['ligand_lig_flag']).clone()
        for g in empty_graphs:
            gen[batch['ligand_element_batch'] == g] = False
        batch['ligand_gen_flag'] = gen
    return batch


def to_dev(batch):
    return {k: v.cuda() for k, v in batch.items()}


def stack(res, key):
    """The per-t result dicts' ``key`` stacked into one CPU tensor."""
    return torch.stack([r[key] for r in res]).cpu()


def make_model(num_steps=10, device=None, **enc):
    model = TargetDiffB200(synthetic.targetdiff_config(num_steps=num_steps, **enc))
    sd = synthetic.seeded_state_dict(model, seed=WEIGHT_SEED)
    model.load_state_dict(sd, strict=True)
    model.eval()
    if device is not None:
        model = model.to(device)
    return model, sd


def composed_inputs(sd, batch):
    """(x, h, batch_idx, lig_flag, gen_flag) in composed node order, computed by the ORACLE's
    embed/compose restatement (CPU)."""
    import torch.nn.functional as F
    from oracle import diffusion as OD
    lig_flag, rec_flag = batch['ligand_lig_flag'], batch['protein_lig_flag']
    gen_lig = batch.get('ligand_gen_flag', lig_flag)
    gen_rec = batch.get('protein_gen_flag', torch.zeros_like(rec_flag))
    c_lig = F.one_hot(batch['ligand_atom_type'], 13).float()
    h_lig, h_rec = OD.context_embed(sd, c_lig, batch['protein_atom_feature'], batch['protein_aa_type'], lig_flag, rec_flag)
    sort_idx, batch_idx, _ = OD.compose(batch['ligand_element_batch'], batch['protein_element_batch'])
    x = torch.cat([batch['protein_pos'], batch['ligand_pos']], 0)[sort_idx]
    h = torch.cat([h_rec, h_lig], 0)[sort_idx]
    gen = torch.cat([gen_rec, gen_lig], 0)[sort_idx]
    lig = torch.cat([rec_flag, lig_flag], 0)[sort_idx]
    return x, h, batch_idx, lig, gen


def rel_err(a, b):
    """max |a-b| / max |b| (the 'relative fp32' measure of the parity bar)."""
    a, b = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64)
    if b.numel() == 0:
        return 0.0
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-30))


def assert_close(a, b, rtol=1e-4, atol=1e-5, what=''):
    """Element-wise check beside the global max-norm of ``rel_err``: |a - b| <= atol + rtol * |b| for EVERY element
    (rel_err alone would admit 2e-3 A on any atom when |x| ~ 20 A)."""
    a, b = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64)
    bad = (a - b).abs() > atol + rtol * b.abs()
    if bool(bad.any()):
        i = int(torch.argmax(((a - b).abs() - rtol * b.abs()).flatten()))
        raise AssertionError(f'{what}: {int(bad.sum())} of {bad.numel()} elements outside rtol={rtol} atol={atol}; worst '
                             f'got {float(a.flatten()[i]):.7g} want {float(b.flatten()[i]):.7g}')


def loss_close(got, want, rtol, atol=0.0, nan_equal=False):
    """Two scalar losses agree: |got - want| <= atol + rtol |want|; with ``nan_equal`` a NaN ``want`` asks for a NaN."""
    if nan_equal and math.isnan(want):
        return math.isnan(got)
    return abs(got - want) <= atol + rtol * abs(want)


def assert_bitwise(a, b, loss_keys, nan_equal=False):
    """Two validation-loss outputs (loss_dict, then dicts of tensors or tensors) are bit-identical: the losses of
    ``loss_keys`` (NaN equal to NaN with ``nan_equal``) and every tensor after them."""
    for k in loss_keys:
        assert torch.equal(a[0][k], b[0][k]) or (nan_equal and math.isnan(float(a[0][k])) and
                                                 math.isnan(float(b[0][k]))), k
    for x, y in zip(a[1:], b[1:], strict=True):
        if isinstance(x, dict):
            for k in x:
                assert torch.equal(x[k], y[k]), k
        else:
            assert torch.equal(x, y)
