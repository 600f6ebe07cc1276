// Packed-weight blob layout shared by the CUDA kernels and (through the C-ABI layout
// queries in include/cbg_b200.h) by the Python packer.  Single source of truth.
//
// All sizes are in floats and multiples of 4 so every field is 16-byte aligned when the
// blob base is.  Field order inside a layer is the order in which each edge kernel
// stages its weights into shared memory, so one contiguous float4 copy loads a kernel's
// whole working set.
//
// Notation (reference state-dict names, SURVEY.md section 8b):
//   W0k = blocks.l.x2h_layers.0.hk_func.net.0.weight [128,340]  (cols: 0:4 edge type,
//         4:84 type(x)RBF with index 20*type+m, 84:212 h_dst ("i"), 212:340 h_src ("j"))
//   "Note D" split: W0*[ type | rfeat | h_i | h_j ] = c[type] + Wrf[type]*g(d) + Pi[i] + Pj[j]
#pragma once

#define CBG_H        128   // node_feat_dim (only value the reference's configs use)
#define CBG_HEADS     16   // n_heads
#define CBG_DH         8   // head dim
#define CBG_NRBF      20   // num_r_gaussian (only valid value, SURVEY.md A4)
#define CBG_NTYPE      4   // edge types
#define CBG_KMAX      32   // neighbour-table width (k <= 32)
#define CBG_GATE_H   160   // dist_emb MLP hidden = 8 * num_r_gaussian
#define CBG_MAXCLS    16   // classifier rows are padded to 16 (num_classes <= 16)
#define CBG_IPA_MAXCLS 32  // IPATransformer type head (csrc/ipa.cu): rows padded to 32 (D3FG: 28 functional-group types)
#define CBG_NPLANES    5   // node projection planes per sub-layer: Pj_k, Pj_v, Pi_k, Pi_v, q_hidden
#define CBG_NODE_SRC_PLANES 2   // the first two are gathered by edges from the SOURCE node, the rest belong to the destination

// ---- per-layer fields -------------------------------------------------------------------
// X(name, floats)
#define CBG_LAYER_FIELDS(X)                                                              \
  /* X2H node GEMM: Wt[k=128][n=640], n-planes = [Pj_k | Pj_v | Pi_k | Pi_v | q_hidden] */ \
  X(X2H_NODE_WT, 128 * 640)                                                              \
  X(X2H_NODE_B, 640)        /* [0|0|b0k|b0v|bq0] */                                      \
  X(X2H_Q_LN, 256)          /* gamma[128], beta[128] of hq_func.net.1 */                 \
  X(X2H_Q_W1T, 128 * 128)   /* (hq_func.net.3.weight / sqrt(8))^T  [k][n] */             \
  X(X2H_Q_B1, 128)          /* hq_func.net.3.bias / sqrt(8) */                           \
  /* x2h_k edge kernel working set (contiguous) */                                       \
  X(X2H_K_WRF, 4 * 20 * 128) /* [type][m][f] = W0k[f, 4+20*type+m] */                    \
  X(X2H_K_C, 4 * 128)        /* [type][f]    = W0k[f, type] */                           \
  X(X2H_K_LN, 256)           /* gamma, beta of hk_func.net.1 */                          \
  X(X2H_K_W1, 128 * 128)     /* hk_func.net.3.weight natural [f_out][f_in] */            \
  X(X2H_K_RBF, 32)           /* offsets[20], coeff at [20] */                            \
  /* x2h_v edge kernel working set (contiguous) */                                       \
  X(X2H_V_WRF, 4 * 20 * 128)                                                             \
  X(X2H_V_C, 4 * 128)                                                                    \
  X(X2H_V_LN, 256)                                                                       \
  X(X2H_V_W1, 128 * 128)     /* hv_func.net.3.weight natural [f_out][f_in] */            \
  X(X2H_V_B1, 128)           /* hv_func.net.3.bias */                                    \
  X(X2H_V_RBF, 32)                                                                       \
  /* X2H node GEMM weights for the 3xTF32 wgmma path: 6 planes [Pj_k,Pj_v,Pi_k,Pi_v,q_hidden,q_out],   \
     each = 4 K-chunks x (hi | lo) x [128 n][32 k] tf32 in the canonical K-major layout  */       \
  X(X2H_NODE_TC, 6 * 32768)                                                              \
  /* H2X node GEMM */                                                                    \
  X(H2X_NODE_WT, 128 * 640)                                                              \
  X(H2X_NODE_B, 640)                                                                     \
  X(H2X_Q_LN, 256)                                                                       \
  X(H2X_Q_W1T, 128 * 128)                                                                \
  X(H2X_Q_B1, 128)                                                                       \
  X(H2X_NODE_TC, 6 * 32768)                                                              \
  /* h2x edge kernel working set (contiguous) */                                         \
  X(H2X_K_WRF, 4 * 20 * 128)                                                             \
  X(H2X_K_C, 4 * 128)                                                                    \
  X(H2X_K_LN, 256)                                                                       \
  X(H2X_K_W1, 128 * 128)     /* xk_func.net.3.weight natural */                          \
  X(H2X_V_WRF, 4 * 20 * 128)                                                             \
  X(H2X_V_C, 4 * 128)                                                                    \
  X(H2X_V_LN, 256)                                                                       \
  X(H2X_V_W1, 16 * 128)      /* xv_func.net.3.weight [head][f_in] */                     \
  X(H2X_V_B1, 32)            /* xv_func.net.3.bias[16], zero padded */                   \
  X(H2X_RBF, 32)                                                                         \
  /* wgmma X2H kernels (x2h_tc.cu): f16 (hi | lo) operand images in the canonical K-major no-swizzle layout.   \
     TCW1 = 64 * W1 [128 n][128 k]; TCWG = [128 n][96 k] with k < 80: 16 * Wrf[t][m] at k = 20 t + m,           \
     k = 80 + t: 16 * c[t], k >= 84: zero padding to K = 96.  Sizes in floats. */                       \
  X(X2H_K_TCW1, 2 * 128 * 128 / 2)                                                       \
  X(X2H_K_TCWG, 2 * 128 * 96 / 2)                                                        \
  X(X2H_V_TCW1, 2 * 128 * 128 / 2)                                                       \
  X(X2H_V_TCWG, 2 * 128 * 96 / 2)                                                        \
  /* node GEMM weights for the f16 wgmma path   (node_gemm_f16.cu): the 6 planes of X2H_NODE_TC / H2X_NODE_TC, each as   \
     2 K-chunks x (hi | lo) x [128 n][64 k] f16 of 256 * W in the canonical K-major layout.  Sizes in floats. */        \
  X(X2H_NODE_TCH, 6 * 2 * 2 * 128 * 64 / 2)                                              \
  X(H2X_NODE_TCH, 6 * 2 * 2 * 128 * 64 / 2)                                              \
  /* wgmma   H2X kernels (x2h_tc.cu, modes H2X-k / H2X-v): same images for the xk / xv edge MLPs of H2XAttention; the    \
     second Linear of xv has 16 outputs (one per head): TCW1 = 64 * W1xv as a [16 n][128 k] (hi | lo) image */          \
  X(H2X_K_TCW1, 2 * 128 * 128 / 2)                                                       \
  X(H2X_K_TCWG, 2 * 128 * 96 / 2)                                                        \
  X(H2X_V_TCW1, 2 * 16 * 128 / 2)                                                        \
  X(H2X_V_TCWG, 2 * 128 * 96 / 2)

// ---- global (per-denoiser) fields -------------------------------------------------------
#define CBG_GLOBAL_FIELDS(X)                                                             \
  /* edge gate (dist_emb) working set (contiguous) */                                    \
  X(GATE_W0T, 20 * 160)      /* dist_emb.1.net.0.weight^T [m][u] */                      \
  X(GATE_B0, 160)                                                                        \
  X(GATE_LN, 320)            /* gamma[160], beta[160] */                                 \
  X(GATE_W1, 160)            /* dist_emb.1.net.3.weight[0,:] */                          \
  X(GATE_RBF, 32)            /* offsets[20], coeff at [20], net.3.bias at [21] */        \
  /* classifier working set (contiguous) */                                              \
  X(CLS_W0T, 128 * 128)      /* classifier.0.weight^T [k][n] */                          \
  X(CLS_B0, 128)                                                                         \
  X(CLS_W1, 16 * 128)        /* classifier.2.weight [class][f], zero padded to 16 rows */\
  X(CLS_B1, 32)              /* classifier.2.bias, zero padded */

enum CbgLayerField {
#define X(name, n) CBG_LF_##name,
  CBG_LAYER_FIELDS(X)
#undef X
  CBG_LF_COUNT
};

enum CbgGlobalField {
#define X(name, n) CBG_GF_##name,
  CBG_GLOBAL_FIELDS(X)
#undef X
  CBG_GF_COUNT
};

#ifdef __cplusplus
namespace cbg_layout {
constexpr long long kLayerSizes[] = {
#define X(name, n) (long long)(n),
    CBG_LAYER_FIELDS(X)
#undef X
};
constexpr long long kGlobalSizes[] = {
#define X(name, n) (long long)(n),
    CBG_GLOBAL_FIELDS(X)
#undef X
};
constexpr long long layer_offset(int f) {
  long long o = 0;
  for (int i = 0; i < f; ++i) o += kLayerSizes[i];
  return o;
}
constexpr long long global_offset(int f) {
  long long o = 0;
  for (int i = 0; i < f; ++i) o += kGlobalSizes[i];
  return o;
}
constexpr long long kLayerFloats = layer_offset(CBG_LF_COUNT);
constexpr long long kGlobalFloats = global_offset(CBG_GF_COUNT);
}  // namespace cbg_layout
#endif
