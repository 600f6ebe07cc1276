"""CPU-side checks: the C-ABI library loads and exports every declared symbol, the weight blob
layout/packing, state-dict compatibility, schedule tables, configuration gating, sharding."""
import json
import os
import re

import numpy as np
import pytest
import torch

from cbgbench_b200 import _lib, sharding, synthetic
from cbgbench_b200.modules import UniTransformerB200, pack_denoiser_blob
from cbgbench_b200.targetdiff import TargetDiffB200, get_model
from helpers import GOLDEN, golden, make_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_loads_and_exports_every_declared_symbol():
    L = _lib.lib()
    header = open(os.path.join(ROOT, 'include', 'cbg_b200.h')).read()
    header = re.sub(r'/\*.*?\*/', '', header, flags=re.S)
    declared = set(re.findall(r'\b(cbg_[a-z0-9_]+)\s*\(', header))
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(L, name), f'{name} declared in include/cbg_b200.h but not exported'
        assert name in _lib.SIGNATURES, f'{name} has no ctypes signature'
    assert set(_lib.SIGNATURES) == declared
    assert L.cbg_version() >= 100


def test_blob_layout_is_consistent():
    lay = _lib.blob_layout()
    for sec, total in (('global', lay['global_floats']), ('layer', lay['layer_floats'])):
        off = 0
        for name, (o, n) in lay[sec].items():
            assert o == off and n % 4 == 0, name        # contiguous, 16-byte aligned fields
            off += n
        assert off == total
    assert _lib.lib().cbg_workspace_bytes(20736, 1536) > 20736 * 128 * 4 * 6


def test_state_dict_keys_match_reference():
    want = json.load(open(os.path.join(GOLDEN, 'state_keys.json')))
    model = TargetDiffB200(synthetic.targetdiff_config(num_steps=1000))
    got = {k: list(v.shape) for k, v in model.state_dict().items()}
    assert list(got.keys()) == list(want.keys())
    assert got == want
    assert len(want) == 389


def test_schedule_tables_match_reference():
    g = golden('schedules_T1000.npz')
    model = TargetDiffB200(synthetic.targetdiff_config(num_steps=1000))
    sd = model.state_dict()
    for k in g.files:
        assert np.array_equal(sd[k].numpy(), g[k]), k


def test_packing_places_reference_weights():
    model, sd = make_model(10)
    den = {k[len('denoiser.'):]: v for k, v in sd.items() if k.startswith('denoiser.')}
    blob = pack_denoiser_blob(den, '', 9, 13)
    lay = _lib.blob_layout()
    assert blob.numel() == lay['global_floats'] + 9 * lay['layer_floats']
    base = lay['global_floats'] + 4 * lay['layer_floats']
    # the first Linear of the X2H edge MLPs is packed CENTRED over its output-feature axis (exact: LayerNorm follows it)
    w0_raw = den['blocks.4.x2h_layers.0.hk_func.net.0.weight']
    w0 = (w0_raw.double() - w0_raw.double().mean(0, keepdim=True)).float()
    b0_raw = den['blocks.4.x2h_layers.0.hk_func.net.0.bias']
    b0 = (b0_raw.double() - b0_raw.double().mean()).float()
    o, n = lay['layer']['X2H_K_WRF']
    wrf = blob[base + o: base + o + n].view(4, 20, 128)
    assert torch.equal(wrf[2, 7], w0[:, 4 + 2 * 20 + 7])
    assert float(wrf[2, 7].double().sum().abs()) < 1e-5
    o, n = lay['layer']['X2H_K_C']
    assert torch.equal(blob[base + o: base + o + n].view(4, 128)[3], w0[:, 3])
    o, n = lay['layer']['X2H_NODE_WT']
    wt = blob[base + o: base + o + n].view(128, 640)
    assert torch.equal(wt[5, 0:128], w0[:, 212 + 5])              # Pj_k plane = h_src block
    assert torch.equal(wt[5, 256:384], w0[:, 84 + 5])             # Pi_k plane = h_dst block
    o, n = lay['layer']['X2H_NODE_B']
    nb = blob[base + o: base + o + n]
    assert torch.equal(nb[:256], torch.zeros(256)) and torch.equal(nb[256:384], b0)
    # f16 (hi | lo) images of the wgmma X2H kernels: hi + lo reproduces the scaled fp64 weight to ~2^-22
    import numpy as np
    o, n = lay['layer']['X2H_K_TCWG']
    img = blob.view(torch.int32)[base + o: base + o + n].numpy().view(np.float16)
    unpack = lambda a, k: a.reshape(16, k // 8, 8, 8).transpose(0, 2, 1, 3).reshape(128, k).astype(np.float64)
    wg = unpack(img[:128 * 96], 96) + unpack(img[128 * 96:], 96)
    w64 = w0_raw.double() - w0_raw.double().mean(0, keepdim=True)
    assert np.abs(wg[:, 20 * 2 + 7] - 16.0 * w64[:, 4 + 2 * 20 + 7].numpy()).max() < 16.0 * 3e-7 * float(w64.abs().max())
    assert np.abs(wg[:, 80 + 3] - 16.0 * w64[:, 3].numpy()).max() < 16.0 * 3e-7 * float(w64.abs().max())
    assert (wg[:, 84:] == 0).all()                                   # the kernel writes the tile's Pi rows here
    o, n = lay['layer']['X2H_V_TCW1']
    img = blob.view(torch.int32)[base + o: base + o + n].numpy().view(np.float16)
    w1 = unpack(img[:128 * 128], 128) + unpack(img[128 * 128:], 128)
    w1_ref = 64.0 * den['blocks.4.x2h_layers.0.hv_func.net.3.weight'].double().numpy()
    assert np.abs(w1 - w1_ref).max() < 3e-7 * np.abs(w1_ref).max()
    # the H2X edge MLPs are centred the same way; the second Linears are packed as they are
    xk0 = den['blocks.4.h2x_layers.0.xk_func.net.0.weight'].double()
    xk0c = (xk0 - xk0.mean(0, keepdim=True)).float()
    assert torch.equal(blob[base + lay['layer']['H2X_K_C'][0]: base + lay['layer']['H2X_K_C'][0] + 512].view(4, 128)[1],
                       xk0c[:, 1])
    o, n = lay['layer']['H2X_V_W1']
    assert torch.equal(blob[base + o: base + o + n].view(16, 128), den['blocks.4.h2x_layers.0.xv_func.net.3.weight'])
    # f16 images of the wgmma H2X kernels: the value head's second Linear is a [16 n][128 k] image
    o, n = lay['layer']['H2X_V_TCW1']
    assert n == 16 * 128
    img = blob.view(torch.int32)[base + o: base + o + n].numpy().view(np.float16)
    unpack16 = lambda a: a.reshape(2, 16, 8, 8).transpose(0, 2, 1, 3).reshape(16, 128).astype(np.float64)
    w1x = unpack16(img[:16 * 128]) + unpack16(img[16 * 128:])
    w1x_ref = 64.0 * den['blocks.4.h2x_layers.0.xv_func.net.3.weight'].double().numpy()
    assert np.abs(w1x - w1x_ref).max() < 3e-7 * np.abs(w1x_ref).max()
    o, n = lay['layer']['H2X_K_TCWG']
    img = blob.view(torch.int32)[base + o: base + o + n].numpy().view(np.float16)
    wgx = unpack(img[:128 * 96], 96) + unpack(img[128 * 96:], 96)
    xk64 = xk0 - xk0.mean(0, keepdim=True)
    assert np.abs(wgx[:, 20 * 1 + 3] - 16.0 * xk64[:, 4 + 20 + 3].numpy()).max() < 16.0 * 3e-7 * float(xk64.abs().max())
    o, n = lay['global']['GATE_RBF']
    rbf = blob[o: o + n]
    assert float(rbf[20]) == -0.5 and float(rbf[1]) == 1.0 and float(rbf[19]) == 10.0
    o, n = lay['global']['CLS_W1']
    cls = blob[o: o + n].view(16, 128)
    assert torch.equal(cls[:13], den['classifier.2.weight']) and torch.equal(cls[13:], torch.zeros(3, 128))


def test_unsupported_configurations_fail_loudly():
    cfg = synthetic.targetdiff_config()
    cfg.encoder['n_heads'] = 8
    with pytest.raises(NotImplementedError):
        TargetDiffB200(cfg)
    cfg = synthetic.targetdiff_config()
    cfg.encoder['cutoff_mode'] = 'hybrid'
    with pytest.raises(NotImplementedError):
        TargetDiffB200(cfg)
    cfg = synthetic.targetdiff_config()
    cfg.embedder['time'] = {'type': 'sin'}
    with pytest.raises(NotImplementedError):
        TargetDiffB200(cfg)
    with pytest.raises(ValueError):
        TargetDiffB200(synthetic.targetdiff_config(num_steps=1))


def test_registry_mirrors_reference_factory():
    cfg = synthetic.targetdiff_config(num_steps=5, num_layers=2)
    m = get_model(cfg)
    assert isinstance(m, TargetDiffB200) and isinstance(m.denoiser, UniTransformerB200)
    assert m.denoiser.num_layers == 2 and m.denoiser.cut_off == 32 and m.denoiser.cutoff_mode == 'knn'


def test_no_cpu_fallback():
    model, sd = make_model(4)
    batch = synthetic.make_batch([10], [4], seed=1)
    with pytest.raises(RuntimeError):
        model.sample(batch)                     # model on CPU: refuse instead of falling back
    with pytest.raises(RuntimeError):
        model.denoiser(torch.zeros(4, 3), torch.zeros(4, 128), torch.zeros(4, dtype=torch.long),
                       torch.zeros(4, dtype=torch.bool), torch.zeros(4, dtype=torch.bool))


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, 'cbgbench_b200')
    for fn in os.listdir(pkg):
        if fn.endswith('.py'):
            src = open(os.path.join(pkg, fn)).read()
            assert not re.search(r'^\s*(from|import)\s+oracle\b', src, flags=re.M), fn


def test_synthetic_inputs_are_bit_stable():
    b = synthetic.make_batch([5, 3], [2, 2], seed=2024)
    assert b['ligand_atom_type'].tolist() == synthetic.make_batch([5, 3], [2, 2], seed=2024)['ligand_atom_type'].tolist()
    assert abs(float(b['protein_pos'][:5].mean())) < 1e-5           # centred per pocket
    g = golden('forward_cases.npz')
    c1 = synthetic.make_batch([200], [24], seed=2024)
    assert np.array_equal(np.concatenate([c1['protein_pos'].numpy(), c1['ligand_pos'].numpy()]), g['c1_single/x_in'])


# ---- sharding host logic -------------------------------------------------------------------------
def test_assign_graphs_balances_and_is_deterministic():
    sizes = [824, 124, 474, 300, 300, 650, 210, 333]
    parts = sharding.assign_graphs(sizes, 3)
    assert sorted(g for p in parts for g in p) == list(range(8))
    loads = [sum(sizes[g] for g in p) for p in parts]
    assert max(loads) - min(loads) <= max(sizes)
    assert parts == sharding.assign_graphs(sizes, 3)
    assert sharding.assign_graphs([5, 5], 4)[2:] == [[], []]


def test_take_graphs_renumbers_and_selects():
    batch = synthetic.make_batch([4, 3, 5], [2, 1, 3], seed=3, gen_mode='partial')
    sub = sharding.take_graphs(batch, [0, 2])
    assert sub['ligand_element_batch'].tolist() == [0, 0, 1, 1, 1]
    assert sub['protein_element_batch'].tolist() == [0] * 4 + [1] * 5
    assert torch.equal(sub['ligand_pos'][2:], batch['ligand_pos'][3:])
    assert torch.equal(sub['protein_pos'][:4], batch['protein_pos'][:4])
    assert sub['ligand_gen_flag'].shape[0] == 5 and sub['protein_translation'].shape[0] == 9
    assert sharding.graph_sizes(batch).tolist() == [6, 4, 8]
