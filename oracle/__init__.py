"""CPU oracle for the CBGBench diffusion-sampling hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is product code: only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import it, and only as the checker / the timed CPU
baseline.  The product path (``cbgbench_b200``) never imports this package and
fails loudly when its CUDA library is missing.

What it is: a plain torch-CPU (fp32) restatement, in our own words, of the
reference's per-step E(3)-equivariant denoiser and reverse-diffusion step
(``/root/reference`` = EDAPINENUT/CBGBench @ 983fca2; each function cites the
file:line it follows).  It keeps the reference's *as-written* formulation (the
``[E,340]`` edge input is materialised, k/v are per-edge tensors, scatter ops key
on ``dst``) so that it is an independent check of the algebraically restructured
CUDA path.

Third-party arithmetic that is NOT in ``/root/reference`` (un-vendored, unpinned:
``torch_cluster.knn_graph`` behind ``torch_geometric.nn``, ``torch_scatter``) is
restated from its published semantics in ``oracle/graph_ops.py``.

Pinning status: the reference ships no tests, golden vectors or fixtures for this
path (SURVEY.md section 8c), so the oracle is pinned against outputs of the reference
itself, imported unchanged through the shims in
``tests/golden/ref_shims.py``; the generating script is
``tests/golden/make_golden.py`` and the fixtures live in ``tests/golden/*.npz``.
The two [3P] primitives have no reference-side pin (they are definitions).
"""
