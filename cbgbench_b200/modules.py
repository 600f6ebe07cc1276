"""Host-side mirror of the reference denoiser's nn.Module tree, backed by the CUDA library.

Drop-in target: ``UniTransformer`` of /root/reference repo/modules/e3nn/unitransformer.py:12-123
(factory ``get_e3_gnn``, repo/modules/e3nn/__init__.py:5-18).  Same constructor argument
(``cfg`` with ``cfg.get(name, default)``), same ``forward(x, h, batch_idx, lig_flag, gen_flag)
-> (x, h, c)`` signature, same state-dict keys (SURVEY.md section 8b) so reference checkpoints
load unchanged.  The sub-modules below only HOLD parameters under the reference's names; all
arithmetic happens in libcbg_b200.so - there is no PyTorch fallback.
"""
import math

import torch
from torch import nn

from . import _lib

HIDDEN = 128
N_HEADS = 16
N_RBF = 20
RBF_OFFSETS = [0, 1, 1.25, 1.5, 1.75, 2, 2.25, 2.5, 2.75, 3, 3.5, 4, 4.5, 5, 5.5, 6, 7, 8, 9, 10]


def cfg_get(cfg, key, default=None):
    if cfg is None:
        return default
    if hasattr(cfg, 'get'):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


class _NoTorchPath(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError(f'{type(self).__name__} is a parameter container; the arithmetic runs in '
                           'libcbg_b200.so through UniTransformerB200.forward (no PyTorch fallback)')


class GaussianSmearing(_NoTorchPath):
    """Parameter container for common.py:114-133 (buffer ``offset``; fixed 20 offsets)."""

    def __init__(self, num_gaussians=N_RBF):
        super().__init__()
        if num_gaussians != N_RBF:
            raise ValueError('num_r_gaussian must be 20 (the reference hard-codes 20 offsets, SURVEY.md A4)')
        self.register_buffer('offset', torch.tensor(RBF_OFFSETS, dtype=torch.float32))

    @property
    def coeff(self):
        o = self.offset
        return -0.5 / float(o[1] - o[0]) ** 2


class MLP(_NoTorchPath):
    """Parameter container for common.py:151-171: net = [Linear, LayerNorm, ReLU, Linear]."""

    def __init__(self, in_dim, out_dim, hidden_dim):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(in_dim, hidden_dim), nn.LayerNorm(hidden_dim), nn.ReLU(),
                                 nn.Linear(hidden_dim, out_dim))


class ShiftedSoftplus(_NoTorchPath):
    pass


class X2HAttention(_NoTorchPath):
    """Parameters of x2h_attention.py:8-41 (ew_net_type='global', out_fc=False)."""

    def __init__(self, hidden=HIDDEN, n_heads=N_HEADS, edge_feat_dim=4, num_r_gaussian=N_RBF):
        super().__init__()
        kv_in = hidden * 2 + edge_feat_dim + num_r_gaussian * 4
        self.distance_expansion = GaussianSmearing(num_r_gaussian)
        self.hk_func = MLP(kv_in, hidden, hidden)
        self.hv_func = MLP(kv_in, hidden, hidden)
        self.hq_func = MLP(hidden, hidden, hidden)


class H2XAttention(_NoTorchPath):
    """Parameters of h2x_attention.py:9-31 (ew_net_type='global')."""

    def __init__(self, hidden=HIDDEN, n_heads=N_HEADS, edge_feat_dim=4, num_r_gaussian=N_RBF):
        super().__init__()
        kv_in = hidden * 2 + edge_feat_dim + num_r_gaussian * 4
        self.distance_expansion = GaussianSmearing(num_r_gaussian)
        self.xk_func = MLP(kv_in, hidden, hidden)
        self.xv_func = MLP(kv_in, n_heads, hidden)
        self.xq_func = MLP(hidden, hidden, hidden)


class E3DualAttentionLayer(_NoTorchPath):
    """unitransformer.py:125-165 with num_x2h = num_h2x = 1."""

    def __init__(self, hidden=HIDDEN, n_heads=N_HEADS, edge_feat_dim=4, num_r_gaussian=N_RBF):
        super().__init__()
        self.x2h_layers = nn.ModuleList([X2HAttention(hidden, n_heads, edge_feat_dim, num_r_gaussian)])
        self.h2x_layers = nn.ModuleList([H2XAttention(hidden, n_heads, edge_feat_dim, num_r_gaussian)])


import itertools
_BLOB_VERSIONS = itertools.count(1)


def _t(w):
    return w.detach().to('cpu', torch.float64)


def _round_tf32(x):
    """cvt.rna.tf32.f32 on the host: round-to-nearest (ties away) to a 10-bit mantissa, fp32 container."""
    import numpy as np
    b = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    b = ((b + 0x1000) & 0xFFFFE000).astype(np.uint32)
    return b.view(np.float32)


def tc_weight_plane(w):
    """[128 n][128 k] weight (natural nn.Linear layout) -> the tensor-core operand image:
    4 K-chunks x (hi | lo) x [128 n][32 k] tf32, each in the canonical K-major / no-swizzle layout
    (8-row x 16-byte core matrices, 128 B apart along K, 1024 B between 8-row groups)."""
    import numpy as np
    w = w.detach().cpu().to(torch.float32).numpy()
    assert w.shape == (128, 128)
    hi = _round_tf32(w)
    lo = _round_tf32(w - hi)
    kc = 32
    out = np.zeros((128 // kc, 2, 16, kc // 4, 8, 4), dtype=np.float32)   # [chunk][hi/lo][n/8][k_local/4][n%8][k%4]
    for c in range(128 // kc):
        for part, src in enumerate((hi, lo)):
            blk = src[:, kc * c: kc * c + kc].reshape(16, 8, kc // 4, 4)    # [n/8][n%8][kl/4][kl%4]
            out[c, part] = blk.transpose(0, 2, 1, 3)
    return torch.from_numpy(out.reshape(-1)).to(torch.float64)


def tc_f16_image(w, what='weight image', scale=1.0):
    """[n][K k] matrix (n = 128, or 16 for the H2X value head; float64, already scaled by ``scale``, its power of two) ->
    the (hi | lo) f16 operand images of the wgmma kernels (csrc/x2h_tc.cu, csrc/node_gemm_f16.cu): w ~= hi + lo, each
    image in the canonical K-major / no-swizzle layout for 16-bit types (8-row x 8-element core matrices, 128 B apart
    along K, K/8 * 128 B between 8-row groups).  Returns the raw bits as an int32 tensor (two f16 per word).
    Raises ValueError (naming ``what``) when a scaled weight leaves the f16 range: hi would be inf and every product
    that reads it NaN."""
    import numpy as np
    w = np.asarray(w, dtype=np.float64)
    n, k = w.shape
    assert n % 8 == 0 and k % 16 == 0
    with np.errstate(over='ignore', invalid='ignore'):
        hi = w.astype(np.float16)
        lo = (w - hi.astype(np.float64)).astype(np.float16)
    if not (np.isfinite(hi).all() and np.isfinite(lo).all()):
        big = float(np.nanmax(np.abs(w))) / scale if np.isfinite(w).any() else float('nan')
        raise ValueError(f'{what}: max |w| = {big:.6g} does not fit the f16 tensor-core image (|w| x {scale:g} must stay '
                         f'below {F16_MAX:g}, i.e. |w| < {F16_MAX / scale:.6g}), or a weight is not finite')
    imgs = [m.reshape(n // 8, 8, k // 8, 8).transpose(0, 2, 1, 3).reshape(-1) for m in (hi, lo)]
    return torch.from_numpy(np.concatenate(imgs).view(np.int32).copy())


def check_ln_activation_bound(ln_params, scale, what):
    """relu(LayerNorm(x) * gamma + beta) over 128 features is bounded by sqrt(127) max|gamma| + max|beta| (no normalised
    feature exceeds sqrt(n - 1)).  The wgmma kernels split these activations into f16 (hi, lo) after multiplying by
    ``scale``; raise ValueError (naming ``what``) when the scaled bound reaches the f16 maximum."""
    g, b = ln_params[:HIDDEN], ln_params[HIDDEN:]
    bound = math.sqrt(HIDDEN - 1) * float(g.abs().max()) + float(b.abs().max())
    if not bound * scale < F16_MAX:
        raise ValueError(f'{what}: LayerNorm activation bound sqrt(127) max|gamma| + max|beta| = {bound:.6g} times '
                         f'{scale:g} reaches the f16 maximum {F16_MAX:g} of the tensor-core operand '
                         f'(the bound must stay below {F16_MAX / scale:.6g})')


# power-of-two scales of the f16 images (must match csrc/x2h_tc.cu)
TC_SCALE_WG = 16.0
TC_SCALE_W1 = 64.0
TC_KG = 96
TC_SCALE_NODE = 256.0       # node GEMM weight planes (csrc/node_gemm_f16.cu)
TC_SCALE_ACT = 64.0         # LayerNorm + ReLU activations of the edge MLPs (csrc/x2h_tc.cu)
TC_SCALE_Q = 16.0           # LayerNorm + ReLU activations of the q MLP (csrc/node_gemm_f16.cu)
F16_MAX = 65504.0


def pack_denoiser_blob(sd, prefix, num_layers, num_classes, com_head=False):
    """Pack a (reference-keyed) state dict into the flat fp32 blob of csrc/cbg_layout.h.

    ``com_head=True`` packs DiffBP's CoMPredictor (diffbp.py:30-57: its own ``dist_emb`` and ``num_layers`` x
    H2XAttention under ``h2xattentions.<l>.``) into the same layout: the gate fields of the global block and the
    H2X fields of every layer block are filled, classifier and X2H fields stay zero."""
    lay = _lib.blob_layout()
    total = lay['global_floats'] + num_layers * lay['layer_floats']
    blob = torch.zeros(total, dtype=torch.float64)
    raw = []      # (offset, int32 bit patterns): fields that are not fp32 values (f16 images), written after the cast

    def put_raw(base, field_map, name, bits):
        off, size = field_map[name]
        assert bits.dtype == torch.int32 and bits.numel() == size, (name, bits.numel(), size)
        raw.append((base + off, bits))

    def put(base, field_map, name, value):
        off, size = field_map[name]
        v = value.reshape(-1)
        assert v.numel() <= size, (name, v.numel(), size)
        blob[base + off: base + off + v.numel()] = v

    def rbf_field(offset_buf, extra=None):
        o = _t(offset_buf)
        assert o.numel() == N_RBF
        v = torch.zeros(32, dtype=torch.float64)
        v[:N_RBF] = o
        v[20] = -0.5 / float(o[1] - o[0]) ** 2
        if extra is not None:
            v[21] = extra
        return v

    def first_layer_split(w0):
        """W0 [128,340] -> (Wrf [4][20][128], c [4][128], W_i^T [128k][128n], W_j^T)."""
        w0 = _t(w0)
        c = w0[:, 0:4].t().contiguous()                                         # [t][f]
        wrf = w0[:, 4:84].reshape(HIDDEN, 4, N_RBF).permute(1, 2, 0).contiguous()  # [t][m][f]
        wi_t = w0[:, 84:212].t().contiguous()                                   # [k][n]
        wj_t = w0[:, 212:340].t().contiguous()
        return wrf, c, wi_t, wj_t

    g = lay['global']
    p = prefix
    put(0, g, 'GATE_W0T', _t(sd[p + 'dist_emb.1.net.0.weight']).t().contiguous())
    put(0, g, 'GATE_B0', _t(sd[p + 'dist_emb.1.net.0.bias']))
    put(0, g, 'GATE_LN', torch.cat([_t(sd[p + 'dist_emb.1.net.1.weight']), _t(sd[p + 'dist_emb.1.net.1.bias'])]))
    put(0, g, 'GATE_W1', _t(sd[p + 'dist_emb.1.net.3.weight']).reshape(-1))
    put(0, g, 'GATE_RBF', rbf_field(sd[p + 'dist_emb.0.offset'], float(sd[p + 'dist_emb.1.net.3.bias'].reshape(-1)[0])))
    if not com_head:
        put(0, g, 'CLS_W0T', _t(sd[p + 'classifier.0.weight']).t().contiguous())
        put(0, g, 'CLS_B0', _t(sd[p + 'classifier.0.bias']))
        w1 = _t(sd[p + 'classifier.2.weight'])
        assert w1.shape == (num_classes, HIDDEN) and num_classes <= 16
        put(0, g, 'CLS_W1', w1)
        put(0, g, 'CLS_B1', _t(sd[p + 'classifier.2.bias']))

    lf = lay['layer']
    inv_sqrt_dh = 1.0 / math.sqrt(HIDDEN // N_HEADS)
    for l in range(num_layers):
        base = lay['global_floats'] + l * lay['layer_floats']
        subs = ((('H2X', f'h2xattentions.{l}.', 'xk_func', 'xv_func', 'xq_func'),) if com_head else
                (('X2H', f'blocks.{l}.x2h_layers.0.', 'hk_func', 'hv_func', 'hq_func'),
                 ('H2X', f'blocks.{l}.h2x_layers.0.', 'xk_func', 'xv_func', 'xq_func')))
        for tag, sub, kname, vname, qname in subs:
            sp = p + sub
            w0k, w0v = _t(sd[sp + kname + '.net.0.weight']), _t(sd[sp + vname + '.net.0.weight'])
            b0k, b0v = _t(sd[sp + kname + '.net.0.bias']), _t(sd[sp + vname + '.net.0.bias'])
            # Centre the first Linear of the edge MLPs (X2H and H2X alike) over the OUTPUT-feature axis: LayerNorm follows
            # it directly (common.py:151-171), so pre - mean_f(pre) is all that is ever used, and with
            # W0 <- W0 - mean_f W0, b0 <- b0 - mean_f b0 every piece (Pi, Pj, Wrf g, c) has zero feature mean by
            # itself.  Exact; the wgmma kernels then need only the sum of squares (the SIMT kernels subtract
            # a mean that is zero up to rounding).
            w0k, w0v = w0k - w0k.mean(0, keepdim=True), w0v - w0v.mean(0, keepdim=True)
            b0k, b0v = b0k - b0k.mean(), b0v - b0v.mean()
            wrf_k, c_k, wi_k, wj_k = first_layer_split(w0k)
            wrf_v, c_v, wi_v, wj_v = first_layer_split(w0v)
            wq0_t = _t(sd[sp + qname + '.net.0.weight']).t().contiguous()
            node_wt = torch.cat([wj_k, wj_v, wi_k, wi_v, wq0_t], dim=1)            # [128 k][640 n]
            node_b = torch.cat([torch.zeros(256, dtype=torch.float64), b0k, b0v, _t(sd[sp + qname + '.net.0.bias'])])
            put(base, lf, f'{tag}_NODE_WT', node_wt)
            tc = [w0k[:, 212:340], w0v[:, 212:340], w0k[:, 84:212], w0v[:, 84:212],
                  _t(sd[sp + qname + '.net.0.weight']), _t(sd[sp + qname + '.net.3.weight']) * inv_sqrt_dh]
            put(base, lf, f'{tag}_NODE_TC', torch.cat([tc_weight_plane(m.to(torch.float32)) for m in tc]))
            where = f'layer {l} {tag}'
            put_raw(base, lf, f'{tag}_NODE_TCH', torch.cat([tc_f16_image((m[:, 64 * c: 64 * c + 64] * TC_SCALE_NODE).numpy(),
                                                                         f'{where}_NODE_TCH', TC_SCALE_NODE)
                                                            for m in tc for c in range(2)]))
            put(base, lf, f'{tag}_NODE_B', node_b)
            q_ln = torch.cat([_t(sd[sp + qname + '.net.1.weight']), _t(sd[sp + qname + '.net.1.bias'])])
            check_ln_activation_bound(q_ln, TC_SCALE_Q, f'{where}_Q_LN')
            put(base, lf, f'{tag}_Q_LN', q_ln)
            put(base, lf, f'{tag}_Q_W1T', (_t(sd[sp + qname + '.net.3.weight']) * inv_sqrt_dh).t().contiguous())
            put(base, lf, f'{tag}_Q_B1', _t(sd[sp + qname + '.net.3.bias']) * inv_sqrt_dh)
            rbf = rbf_field(sd[sp + 'distance_expansion.offset'])
            put(base, lf, f'{tag}_K_WRF', wrf_k)
            put(base, lf, f'{tag}_K_C', c_k)
            k_ln = torch.cat([_t(sd[sp + kname + '.net.1.weight']), _t(sd[sp + kname + '.net.1.bias'])])
            v_ln = torch.cat([_t(sd[sp + vname + '.net.1.weight']), _t(sd[sp + vname + '.net.1.bias'])])
            check_ln_activation_bound(k_ln, TC_SCALE_ACT, f'{where}_K_LN')
            check_ln_activation_bound(v_ln, TC_SCALE_ACT, f'{where}_V_LN')
            put(base, lf, f'{tag}_K_LN', k_ln)
            put(base, lf, f'{tag}_K_W1', _t(sd[sp + kname + '.net.3.weight']))
            put(base, lf, f'{tag}_V_WRF', wrf_v)
            put(base, lf, f'{tag}_V_C', c_v)
            put(base, lf, f'{tag}_V_LN', v_ln)
            put(base, lf, f'{tag}_V_W1', _t(sd[sp + vname + '.net.3.weight']))
            put(base, lf, f'{tag}_V_B1', _t(sd[sp + vname + '.net.3.bias']))
            if tag == 'X2H':
                put(base, lf, 'X2H_K_RBF', rbf)
                put(base, lf, 'X2H_V_RBF', rbf)
            else:
                put(base, lf, 'H2X_RBF', rbf)
            # operand images of the wgmma edge kernels (H2X: xv's second Linear has one output per head -> 16 rows)
            for kv, w0, w1 in (('K', w0k, _t(sd[sp + kname + '.net.3.weight'])),
                               ('V', w0v, _t(sd[sp + vname + '.net.3.weight']))):
                wg = torch.zeros(HIDDEN, TC_KG, dtype=torch.float64)     # [f][k]: k = 20 t + m | 80 + t | Pi columns
                wg[:, 0:80] = w0[:, 4:84]
                wg[:, 80:84] = w0[:, 0:4]
                put_raw(base, lf, f'{tag}_{kv}_TCWG', tc_f16_image((wg * TC_SCALE_WG).numpy(), f'{where}_{kv}_TCWG', TC_SCALE_WG))
                put_raw(base, lf, f'{tag}_{kv}_TCW1', tc_f16_image((w1 * TC_SCALE_W1).numpy(), f'{where}_{kv}_TCW1', TC_SCALE_W1))
    blob32 = blob.to(torch.float32)
    bits = blob32.view(torch.int32)
    for off, b in raw:
        bits[off: off + b.numel()] = b
    return blob32


class _Workspace:
    """Grow-only device scratch shared by the calls of one module."""

    def __init__(self):
        self.buf = None

    def get(self, nbytes, device):
        if self.buf is None or self.buf.numel() < nbytes or self.buf.device != device:
            self.buf = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=device)
        off = (-self.buf.data_ptr()) % 256
        return self.buf.data_ptr() + off, self.buf.numel() - off


def graph_ptr_from_batch(batch_idx):
    """Sorted PyG batch vector -> (graph_ptr int32 [B+1] on the same device, B, max nodes per graph).
    One host sync (the reference's ``batch_idx.max() + 1`` does the same, targetdiff.py:146)."""
    if batch_idx.numel() == 0:
        raise ValueError('empty batch')
    counts = torch.bincount(batch_idx)
    ptr = torch.zeros(counts.numel() + 1, dtype=torch.int32, device=batch_idx.device)
    ptr[1:] = torch.cumsum(counts, 0).to(torch.int32)
    if not bool((batch_idx[1:] >= batch_idx[:-1]).all()):
        raise ValueError('batch_idx must be sorted (graphs must be contiguous)')
    return ptr, int(counts.numel()), int(counts.max())


class UniTransformerB200(nn.Module):
    """CUDA (H100) drop-in for the reference's ``UniTransformer`` (unitransformer.py:12-123)."""

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        self.num_classes = cfg_get(cfg, 'num_classes', None)
        self.out_classes = cfg_get(cfg, 'out_classes', self.num_classes)
        self.num_blocks = cfg_get(cfg, 'num_blocks', 1)
        self.num_layers = cfg_get(cfg, 'num_layers', 6)
        self.hidden_dim = cfg_get(cfg, 'node_feat_dim', 128)
        self.n_heads = cfg_get(cfg, 'n_heads', 16)
        self.edge_feat_dim = cfg_get(cfg, 'edge_feat_dim', 4)
        self.cutoff_mode = cfg_get(cfg, 'cutoff_mode', 'knn')
        self.cut_off = int(cfg_get(cfg, 'k', 32))
        self.r_max = float(cfg_get(cfg, 'r_max', 10.0))
        self.ew_net_type = cfg_get(cfg, 'ew_type', 'global')
        self.num_r_gaussian = cfg_get(cfg, 'num_r_gaussian', 20)
        unsupported = []
        if self.hidden_dim != HIDDEN or cfg_get(cfg, 'pair_feat_dim', 128) != 128:
            unsupported.append('node_feat_dim/pair_feat_dim != 128')
        if self.n_heads != N_HEADS:
            unsupported.append('n_heads != 16')
        if self.num_blocks != 1:
            unsupported.append('num_blocks != 1')
        if self.ew_net_type != 'global':
            unsupported.append("ew_type != 'global'")
        if cfg_get(cfg, 'act_fn', 'relu') != 'relu' or not cfg_get(cfg, 'norm', True):
            unsupported.append('act_fn/norm')
        if cfg_get(cfg, 'num_x2h', 1) != 1 or cfg_get(cfg, 'num_h2x', 1) != 1 or cfg_get(cfg, 'x2h_out_fc', False):
            unsupported.append('num_x2h/num_h2x/x2h_out_fc')
        if cfg_get(cfg, 'dist_emb_type', 'gaussian_exp') != 'gaussian_exp':
            unsupported.append('dist_emb_type')
        if self.cutoff_mode not in ('knn', 'radius'):
            unsupported.append(f'cutoff_mode={self.cutoff_mode}')
        if not (1 <= self.cut_off <= 32):
            unsupported.append('k outside [1,32]')
        if self.num_classes is None or not (1 <= self.out_classes <= 16):
            unsupported.append('num_classes must be in [1,16]')
        if unsupported:
            raise NotImplementedError('UniTransformerB200 covers the configuration every shipped CBGBench '
                                      'config uses (SURVEY.md); unsupported: ' + ', '.join(unsupported))

        self.dist_emb = nn.Sequential(GaussianSmearing(self.num_r_gaussian),
                                      MLP(self.num_r_gaussian, 1, self.num_r_gaussian * 8))
        self.blocks = nn.ModuleList([E3DualAttentionLayer(self.hidden_dim, self.n_heads, self.edge_feat_dim,
                                                          self.num_r_gaussian) for _ in range(self.num_layers)])
        self.classifier = nn.Sequential(nn.Linear(self.hidden_dim, self.hidden_dim), ShiftedSoftplus(),
                                        nn.Linear(self.hidden_dim, self.out_classes))
        self._blob = None
        self._blob_key = None
        self._ws = _Workspace()

    def __repr__(self):
        return (f'UniTransformerB200(num_layers={self.num_layers}, n_heads={self.n_heads}, '
                f'cutoff_mode={self.cutoff_mode}, k={self.cut_off}, r_max={self.r_max})')

    # ---- weights -------------------------------------------------------------------------
    def _state_key(self, device):
        return (str(device),) + tuple((t.data_ptr(), t._version) for t in self.state_dict(keep_vars=True).values())

    def packed_blob(self, device):
        """Flat fp32 weight blob on ``device`` (re-packed when any parameter changed)."""
        key = self._state_key(device)
        if self._blob is None or key != self._blob_key:
            sd = {k: v for k, v in self.state_dict().items()}
            self._blob = pack_denoiser_blob(sd, '', self.num_layers, self.out_classes).to(device)
            self._blob_key = key
            self._blob_version = next(_BLOB_VERSIONS)       # process-unique: the C side keys its device copy on it
        return self._blob

    @property
    def mode_id(self):
        return 0 if self.cutoff_mode == 'knn' else 1

    # ---- the reference-facing call -------------------------------------------------------
    @torch.no_grad()
    def forward(self, x, h, batch_idx, lig_flag, gen_flag, stop_after_layers=-1):
        if not x.is_cuda:
            raise RuntimeError('UniTransformerB200 runs on a CUDA device only (no CPU fallback); '
                               'for host buffers use forward_host()')
        dev = x.device
        L = _lib.lib()
        N = x.shape[0]
        x32 = x.detach().to(torch.float32).contiguous()
        h32 = h.detach().to(torch.float32).contiguous()
        gptr, B, max_n = graph_ptr_from_batch(batch_idx)
        lig8 = lig_flag.to(torch.uint8).contiguous()
        gen8 = gen_flag.to(torch.uint8).contiguous()
        gen_idx = torch.nonzero(gen8, as_tuple=False).flatten().to(torch.int32).contiguous()
        n_gen = int(gen_idx.numel())
        blob = self.packed_blob(dev)
        x_out = torch.empty_like(x32)
        h_out = torch.empty_like(h32)
        c_out = torch.empty((N, self.out_classes), dtype=torch.float32, device=dev)
        ws_bytes = L.cbg_workspace_bytes(N, n_gen)
        ws_ptr, ws_have = self._ws.get(ws_bytes, dev)
        with torch.cuda.device(dev):
            _lib.check(L.cbg_denoiser_forward_f32(
                blob.data_ptr(), self.num_layers, self.out_classes, x32.data_ptr(), h32.data_ptr(),
                gptr.data_ptr(), B, max_n, lig8.data_ptr(), gen8.data_ptr(),
                gen_idx.data_ptr() if n_gen else None, n_gen, None, 0, N, self.mode_id, self.cut_off,
                self.r_max, int(stop_after_layers), x_out.data_ptr(), h_out.data_ptr(), c_out.data_ptr(),
                ws_ptr, ws_have, _lib.stream_ptr(dev)))
        return x_out, h_out, c_out

    @torch.no_grad()
    def forward_host(self, x, h, batch_idx, lig_flag, gen_flag):
        """Same contract with HOST tensors in and out (H2D/D2H inside the C-ABI call)."""
        L = _lib.lib()
        N = x.shape[0]
        x32 = x.detach().to('cpu', torch.float32).contiguous()
        h32 = h.detach().to('cpu', torch.float32).contiguous()
        b = batch_idx.detach().cpu()
        counts = torch.bincount(b)
        gptr = torch.zeros(counts.numel() + 1, dtype=torch.int32)
        gptr[1:] = torch.cumsum(counts, 0).to(torch.int32)
        lig8 = lig_flag.detach().cpu().to(torch.uint8).contiguous()
        gen8 = gen_flag.detach().cpu().to(torch.uint8).contiguous()
        blob = self.packed_blob(torch.device('cpu'))
        x_out, h_out = torch.empty_like(x32), torch.empty_like(h32)
        c_out = torch.empty((N, self.out_classes), dtype=torch.float32)
        _lib.check(L.cbg_denoiser_forward_host_f32(
            blob.data_ptr(), blob.numel(), self._blob_version, self.num_layers, self.out_classes,
            x32.data_ptr(), h32.data_ptr(), gptr.data_ptr(), int(counts.numel()), lig8.data_ptr(), gen8.data_ptr(),
            N, self.mode_id, self.cut_off, self.r_max, x_out.data_ptr(), h_out.data_ptr(), c_out.data_ptr()))
        return x_out, h_out, c_out


def get_e3_gnn(cfg, num_classes=None, num_edge_classes=None):
    """Mirror of repo/modules/e3nn/__init__.py:5-18 for the encoder types built here."""
    if num_classes is not None:
        cfg.num_classes = num_classes
    if num_edge_classes is not None:
        cfg.num_edge_classes = num_edge_classes
    if cfg_get(cfg, 'type') == 'unitransformer':
        return UniTransformerB200(cfg)
    if cfg_get(cfg, 'type') in ('ipatransformer', 'itatransformer'):      # row f4; the shipped D3FG config spells it 'itatransformer'
        from .ipatransformer import IPATransformerB200
        return IPATransformerB200(cfg)
    raise ValueError(f"cbgbench_b200 implements encoder types 'unitransformer' and 'ipatransformer', got {cfg_get(cfg, 'type')}")
