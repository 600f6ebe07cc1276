"""Import the UNMODIFIED reference from its checkout (``REF_ROOT`` below).

Used only by the fixture generators ``tests/golden/make_golden*.py`` (run where the checkout exists).
bench.py's reference arms use the copy that ``oracle/stage_ref.py`` installs into ``oracle/_ref/``, through
``baseline/ref_runner.py``, instead.  Recipe from SURVEY.md Appendix C:

* fake ``easydict`` (attr-dict), ``rdkit*`` (MagicMock: only touched at import time by
  repo/utils/molecule/constants.py:3-19);
* ``torch_scatter`` / ``torch_geometric.nn`` provided by ``oracle.graph_ops`` - these
  two packages are the un-vendored third-party primitives whose semantics the oracle
  defines (see oracle/graph_ops.py);
* empty package shells for ``repo`` etc. so the heavy ``__init__``s (lmdb, BioPython,
  real rdkit) are not executed.
"""
import sys
import types
from unittest.mock import MagicMock

REF_ROOT = '/root/reference'


class EasyDict(dict):
    def __init__(self, d=None, **kw):
        super().__init__()
        d = dict(d or {}, **kw)
        for k, v in d.items():
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


def install():
    import os
    if not os.path.isdir(REF_ROOT):
        raise FileNotFoundError(REF_ROOT)
    if 'repo.models.diffusion.targetdiff' in sys.modules:
        return
    from oracle import graph_ops

    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)

    ed = types.ModuleType('easydict')
    ed.EasyDict = EasyDict
    sys.modules['easydict'] = ed

    for name in ['rdkit', 'rdkit.Chem', 'rdkit.Chem.rdchem', 'rdkit.Chem.ChemicalFeatures',
                 'rdkit.RDConfig', 'rdkit.Chem.AllChem', 'rdkit.Chem.rdMolTransforms',
                 'rdkit.Geometry']:
        sys.modules.setdefault(name, MagicMock())

    ts = types.ModuleType('torch_scatter')
    for fn in ['scatter_sum', 'scatter_add', 'scatter_mean', 'scatter_max', 'scatter_softmax']:
        setattr(ts, fn, getattr(graph_ops, fn))
    sys.modules['torch_scatter'] = ts

    tg = types.ModuleType('torch_geometric')
    tgn = types.ModuleType('torch_geometric.nn')
    tgn.knn_graph = graph_ops.knn_graph
    tgn.radius_graph = graph_ops.radius_graph
    tgn.knn = MagicMock()
    tgu = types.ModuleType('torch_geometric.utils')
    tgu.coalesce = MagicMock()
    tg.nn, tg.utils = tgn, tgu
    sys.modules['torch_geometric'] = tg
    sys.modules['torch_geometric.nn'] = tgn
    sys.modules['torch_geometric.utils'] = tgu

    for pkg in ['repo', 'repo.models', 'repo.models.diffusion', 'repo.datasets',
                'repo.datasets.transforms']:
        m = types.ModuleType(pkg)
        m.__path__ = [os.path.join(REF_ROOT, *pkg.split('.'))]
        sys.modules[pkg] = m


def targetdiff_cfg(num_steps=1000, num_layers=9, k=None, cutoff_mode=None):
    """EasyDict mirroring configs/denovo/train/targetdiff.yml:1-23 (+ num_atomtype=13,
    which configuration.py:13-38 infers from the transform mode)."""
    enc = dict(type='unitransformer', node_feat_dim=128, n_heads=16, num_layers=num_layers)
    if k is not None:
        enc['k'] = k
    if cutoff_mode is not None:
        enc['cutoff_mode'] = cutoff_mode
    return EasyDict(dict(
        type='targetdiff', num_atomtype=13, encoder=enc,
        generator=dict(pos_schedule=dict(type='sigmoid', beta_start=1.e-7, beta_end=2.e-3),
                       atom_schedule=dict(type='cosine', cosine_s=0.01),
                       num_diffusion_timesteps=num_steps, time_sampler='symmetric'),
        embedder=dict(emb_dim=128, atom=dict(type='linear'), residue=dict(type='linear')),
    ))


def load_targetdiff(cfg=None, **kw):
    install()
    import torch
    from repo.models.diffusion.targetdiff import TargetDiff
    model = TargetDiff(cfg or targetdiff_cfg(**kw))
    model.eval()
    torch.set_grad_enabled(False)
    return model
