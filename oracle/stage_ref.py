"""Recipe that installs the UNMODIFIED reference (EDAPINENUT/CBGBench) into the git-ignored ``oracle/_ref/``.

The reference is pure Python and not pip-installable, so the install is a copy of its ``repo`` package (``*.py`` and
the size-prior table).  ``build()`` runs this where a reference checkout is available (``$CBG_REFERENCE``, default
``/root/reference``); everything that needs the reference at run time (bench.py's reference arms,
tests/test_reference_plugin.py) reads ``oracle/_ref/`` only and reports / skips when it is absent.
"""
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
STAGED = os.path.join(HERE, '_ref')


def stage(force=False):
    """Returns the staged path, or None when there is neither a reference checkout nor an earlier staged copy."""
    live = os.environ.get('CBG_REFERENCE', '/root/reference')
    if not os.path.isdir(os.path.join(live, 'repo')):
        return STAGED if os.path.isdir(os.path.join(STAGED, 'repo')) else None
    marker = os.path.join(STAGED, '.staged')
    if os.path.exists(marker) and not force:
        return STAGED
    if os.path.isdir(STAGED):
        shutil.rmtree(STAGED)
    for dirpath, _, filenames in os.walk(os.path.join(live, 'repo')):
        rel = os.path.relpath(dirpath, live)
        for fn in filenames:
            if fn.endswith(('.py', '.npy')):
                os.makedirs(os.path.join(STAGED, rel), exist_ok=True)
                shutil.copy2(os.path.join(dirpath, fn), os.path.join(STAGED, rel, fn))
    with open(marker, 'w') as f:
        f.write('staged copy of the reference (EDAPINENUT/CBGBench); git-ignored\n')
    return STAGED


if __name__ == '__main__':
    print(stage(force=True))
