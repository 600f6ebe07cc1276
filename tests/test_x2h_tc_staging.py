"""The staged node-plane rows of the wgmma tile kernel (csrc/x2h_tc.cu) against its register-gather path.

By default the attention-weight passes (MODE_K: X2H and H2X) and the H2X value pass (MODE_XV) read the Pi row and half
of the Pj rows of a tile in S1 from shared memory, where bulk copies put them one tile ahead; CBG_X2H_STAGE=0 gathers
all of them into registers instead, as the X2H aggregation pass (MODE_V) always does.  The values and the arithmetic
are the same, so every output must be bit-identical.  The switch is read once per process, so each configuration runs in a child process of
its own (as in test_kernel_variants.py):
- tests/variant_child.py: forwards with -1 neighbour padding (small graphs, k = 8) and partial generation, TargetDiff
  sampling with the pruned node list (eager and CUDA-graph replay), DiffSBDD and DiffBP sampling;
- tests/staging_child.py: six X2H tiles per CTA and five H2X tiles per CTA, both with a ragged last tile and the
  generated-atom count not a multiple of 4.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CHILD_TIMEOUT = 900          # seconds: CUDA start-up plus well under a minute of work on an H100


def _run(script, out_dir, env_add):
    name = os.path.splitext(script)[0] + '_' + ('_'.join(f'{k}={v}' for k, v in sorted(env_add.items())) or 'default')
    out = os.path.join(out_dir, name + '.npz')
    env = {k: v for k, v in os.environ.items() if not k.startswith('CBG_')}
    env.update(env_add)
    cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [os.path.join(HERE, script), out]
    # subprocess.run kills the child when the timeout expires
    res = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=CHILD_TIMEOUT)
    assert res.returncode == 0, f'{name}: child exited with {res.returncode}\n{res.stdout[-4000:]}\n{res.stderr[-4000:]}'
    with np.load(out) as z:
        return {k: z[k] for k in z.files}


def _assert_identical(out, ref, what):
    assert sorted(out) == sorted(ref)
    bad = [k for k in sorted(out) if not np.array_equal(out[k], ref[k])]
    assert not bad, f'{what}: not bit-identical in ' + ', '.join(bad)


@pytest.mark.parametrize('script', ['variant_child.py', 'staging_child.py'])
def test_staged_rows_are_bit_identical_to_register_gathers(script, tmp_path):
    staged = _run(script, str(tmp_path), {})
    gathered = _run(script, str(tmp_path), {'CBG_X2H_STAGE': '0'})
    _assert_identical(staged, gathered, f'{script}: CBG_X2H_STAGE=0')
    if script == 'staging_child.py':
        assert float(staged['moved']) > 1e-3, 'H2X moved nothing'
