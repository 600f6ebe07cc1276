"""Denoiser forwards at the tile-loop sizes where the staged node-plane rows of the wgmma tile kernel (csrc/x2h_tc.cu)
change hands most often, run in a child process by tests/test_x2h_tc_staging.py:

    python tests/staging_child.py OUT.npz

Every CTA of the X2H launches runs six tiles and the last one is ragged (4 S - 1 listed nodes per 4 S slots, S = SM
count); the H2X launches run five tiles per CTA over a generated-atom count that is not a multiple of 4.  Outputs after
one layer and after all layers go to an .npz file.  It loads the library that is already built and never rebuilds it.
"""
import os
import sys
import traceback

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from cbgbench_b200 import _lib, synthetic  # noqa: E402
from helpers import composed_inputs, make_model  # noqa: E402


def sizes(sms):
    """(atoms, generated atoms): 6 X2H tiles per CTA with a ragged last tile, 5 H2X tiles per CTA with a ragged last tile."""
    return 24 * sms - 1, 20 * sms - 3


def split(total, parts):
    return [total // parts + (1 if g < total % parts else 0) for g in range(parts)]


def run(out_path):
    torch.set_grad_enabled(False)
    dev = torch.device('cuda:0')
    n_nodes, n_gen = sizes(torch.cuda.get_device_properties(0).multi_processor_count)
    graphs = -(-n_nodes // 400)
    batch = synthetic.make_batch(split(n_nodes - n_gen, graphs), split(n_gen, graphs), seed=77, gen_mode='denovo')
    model, sd = make_model(10, device=dev)
    x, h, bidx, lig, gen = composed_inputs(sd, batch)
    assert x.shape[0] == n_nodes and int(gen.sum()) == n_gen
    args = [t.to(dev) for t in (x, h, bidx, lig, gen)]
    out = {}
    for tag, stop in (('l1', 1), ('all', -1)):
        for k, v in zip('xhc', model.denoiser(*args, stop_after_layers=stop)):
            out[f'{tag}/{k}'] = v.cpu().numpy()
    out['moved'] = np.float64((torch.from_numpy(out['all/x']) - x).abs().max())
    torch.cuda.synchronize()
    np.savez(out_path, **out)


def main(argv):
    if len(argv) != 1:
        sys.stderr.write('usage: staging_child.py OUT.npz\n')
        return 2
    try:
        run(argv[0])
    except Exception:
        traceback.print_exc()
        try:
            msg = _lib.lib().cbg_last_error()
            sys.stderr.write(f'cbg_last_error: {msg.decode() if msg else ""}\n')
        except Exception:
            pass
        return 1
    return 0


if __name__ == '__main__':
    sys.exit(main(sys.argv[1:]))
