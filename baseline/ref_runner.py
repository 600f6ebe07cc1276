"""The reference arm of bench.py: the UNMODIFIED reference (EDAPINENUT/CBGBench) run through its own public API.

``stage()``   installs the reference's Python package (``$CBG_REFERENCE/repo``, default ``/root/reference``) into the
              git-ignored ``oracle/_ref/`` by the recipe ``oracle/stage_ref.py`` (the reference is pure Python and not
              pip-installable: this copy IS the install; nothing of it enters the git history).
``install()`` puts the staged tree on ``sys.path`` behind the shims of SURVEY.md
              Appendix C: fake ``easydict`` / ``rdkit``, ``torch_scatter`` + ``torch_geometric.nn.knn_graph`` restated with
              plain torch ops (those two packages are un-vendored third-party dependencies of the reference), empty
              package shells so the heavy ``__init__``s (lmdb, BioPython, real rdkit) are not executed.
``time_sample()`` builds ``TargetDiff(cfg)`` with the bench's seeded weights, and times ``TargetDiff.sample(batch)``
              (repo/models/diffusion/targetdiff.py:127-184) - the call the reference's ``sample.py:187`` makes - on the CPU
              (``device='cpu'``: the reference's CPU path on the box's host cores) or eagerly on the GPU
              (``device='cuda'``: how CBGBench is actually run, ``sample.py:107,155``; the same-box GPU comparator).

Nothing of this repo's kernels, models or engine is on that path.  The scatter primitives come from ``oracle/graph_ops``
(device-agnostic torch restatements; bench.py's reference legs are the one place outside tests that may use ``oracle/``);
the neighbour search has a batched on-device variant here so that the eager-GPU arm is not throttled by a host loop.
"""
import os
import sys
import time
import types
from unittest.mock import MagicMock

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle.stage_ref import STAGED, stage  # noqa: E402,F401


def ref_root():
    """The staged reference (oracle/_ref), or None when build() found no reference to stage."""
    return STAGED if os.path.isdir(os.path.join(STAGED, 'repo')) else None


class EasyDict(dict):
    """Attribute dict that wraps nested dicts (what the reference's configs are)."""

    def __init__(self, d=None, **kw):
        super().__init__()
        for k, v in dict(d or {}, **kw).items():
            self[k] = v

    @classmethod
    def _wrap(cls, v):
        if isinstance(v, dict) and not isinstance(v, EasyDict):
            return cls(v)
        if isinstance(v, (list, tuple)):
            return type(v)(cls._wrap(i) for i in v)
        return v

    def __setitem__(self, k, v):
        super().__setitem__(k, self._wrap(v))

    def __setattr__(self, k, v):
        self[k] = v

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


def knn_graph_batched(x, k, batch=None, loop=False, flow='source_to_target', **_):
    """torch_geometric.nn.knn_graph (call site unitransformer.py:79-80) with dense batched torch ops on x's device:
    graphs padded to the largest one, squared distances, top-k smallest per centre.  Same edge set as the oracle's
    definition up to the order of exactly tied distances."""
    import torch
    assert flow == 'source_to_target' and not loop
    n = x.shape[0]
    if batch is None:
        batch = torch.zeros(n, dtype=torch.long, device=x.device)
    counts = torch.bincount(batch)
    B, m = int(counts.numel()), int(counts.max())
    ptr = torch.zeros(B + 1, dtype=torch.long, device=x.device)
    ptr[1:] = torch.cumsum(counts, 0)
    local = torch.arange(n, device=x.device) - ptr[batch]
    xp = torch.zeros(B, m, 3, dtype=x.dtype, device=x.device)
    xp[batch, local] = x
    valid = torch.zeros(B, m, dtype=torch.bool, device=x.device)
    valid[batch, local] = True
    d = xp[:, :, None, :] - xp[:, None, :, :]
    d2 = (d * d).sum(-1)
    big = torch.finfo(d2.dtype).max
    d2 = d2.masked_fill(~valid[:, None, :], big)
    d2 = d2.masked_fill(torch.eye(m, dtype=torch.bool, device=x.device)[None], big)
    kk = min(int(k), m - 1) if m > 1 else 0
    if kk == 0:
        return torch.zeros(2, 0, dtype=torch.long, device=x.device)
    vals, idx = torch.topk(d2, kk, dim=-1, largest=False, sorted=True)       # [B, m, kk]
    centre = (ptr[:-1, None] + torch.arange(m, device=x.device)[None, :])[:, :, None].expand(B, m, kk)
    src = ptr[:-1, None, None] + idx
    keep = valid[:, :, None] & (vals < big)
    return torch.stack([src[keep], centre[keep]], 0)


def install(device_knn=True):
    """Make ``from repo.models.diffusion.targetdiff import TargetDiff`` importable.  Returns the root used."""
    root = ref_root()
    if root is None:
        raise FileNotFoundError('no staged reference: run oracle/stage_ref.py where the reference checkout is available')
    if 'repo.models.diffusion.targetdiff' in sys.modules:
        return root
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import graph_ops
    if root not in sys.path:
        sys.path.insert(0, root)
    ed = types.ModuleType('easydict')
    ed.EasyDict = EasyDict
    sys.modules['easydict'] = ed
    for name in ['rdkit', 'rdkit.Chem', 'rdkit.Chem.rdchem', 'rdkit.Chem.ChemicalFeatures', 'rdkit.RDConfig',
                 'rdkit.Chem.AllChem', 'rdkit.Chem.rdMolTransforms', 'rdkit.Geometry']:
        sys.modules.setdefault(name, MagicMock())
    ts = types.ModuleType('torch_scatter')
    for fn in ['scatter_sum', 'scatter_add', 'scatter_mean', 'scatter_max', 'scatter_softmax']:
        setattr(ts, fn, getattr(graph_ops, fn))
    sys.modules['torch_scatter'] = ts
    tg = types.ModuleType('torch_geometric')
    tgn = types.ModuleType('torch_geometric.nn')
    tgn.knn_graph = knn_graph_batched if device_knn else graph_ops.knn_graph
    tgn.radius_graph = graph_ops.radius_graph
    tgn.knn = MagicMock()
    tgu = types.ModuleType('torch_geometric.utils')
    tgu.coalesce = MagicMock()
    tg.nn, tg.utils = tgn, tgu
    sys.modules['torch_geometric'] = tg
    sys.modules['torch_geometric.nn'] = tgn
    sys.modules['torch_geometric.utils'] = tgu
    for pkg in ['repo', 'repo.models', 'repo.models.diffusion', 'repo.datasets', 'repo.datasets.transforms']:
        m = types.ModuleType(pkg)
        m.__path__ = [os.path.join(root, *pkg.split('.'))]
        sys.modules[pkg] = m
    return root


def targetdiff_cfg(num_steps, **enc_over):
    """configs/denovo/train/targetdiff.yml:1-23 (+ num_atomtype = 13, configuration.py:13-38)."""
    enc = dict(type='unitransformer', node_feat_dim=128, n_heads=16, num_layers=9)
    enc.update({k: v for k, v in enc_over.items() if v is not None})
    return EasyDict(dict(
        type='targetdiff', num_atomtype=13, encoder=enc,
        generator=dict(pos_schedule=dict(type='sigmoid', beta_start=1.e-7, beta_end=2.e-3),
                       atom_schedule=dict(type='cosine', cosine_s=0.01),
                       num_diffusion_timesteps=num_steps, time_sampler='symmetric'),
        embedder=dict(emb_dim=128, atom=dict(type='linear'), residue=dict(type='linear'))))


def build_reference_model(num_steps, enc, device):
    """Reference TargetDiff with this repo's seeded synthetic weights (same state-dict keys)."""
    import torch
    install()
    from repo.models.diffusion.targetdiff import TargetDiff
    from cbgbench_b200 import synthetic
    from cbgbench_b200.targetdiff import TargetDiffB200
    if enc.get('cutoff_mode') == 'radius':
        raise NotImplementedError("the reference's radius branch is dead code (unitransformer.py:76-77: unbound cut_off)")
    ref = TargetDiff(targetdiff_cfg(num_steps, **enc))
    mine = TargetDiffB200(synthetic.targetdiff_config(num_steps=num_steps, **enc))
    ref.load_state_dict(synthetic.seeded_state_dict(mine, seed=0), strict=True)
    torch.set_grad_enabled(False)
    return ref.eval().to(device)


def time_sample(batch, enc, steps, device='cpu', threads=None, quiet=True):
    """Wall-clock seconds of ONE ``TargetDiff.sample(batch)`` call with ``steps`` diffusion steps (T = steps), all
    tensors already on ``device``.  Returns (seconds, traj)."""
    import torch
    if threads:
        torch.set_num_threads(int(threads))
    dev = torch.device(device)
    model = build_reference_model(max(int(steps), 2), enc, dev)
    b = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    if quiet:
        import repo.models.diffusion.targetdiff as tdm
        tdm.tqdm = lambda it, **kw: it                     # progress bar off (it writes to stderr every step)
    if dev.type == 'cuda':
        torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    traj = model.sample(b)
    if dev.type == 'cuda':
        torch.cuda.synchronize(dev)
    return time.perf_counter() - t0, traj


if __name__ == '__main__':
    if len(sys.argv) > 1 and sys.argv[1] == 'stage':
        print(stage(force='--force' in sys.argv))
    else:
        print(ref_root())
