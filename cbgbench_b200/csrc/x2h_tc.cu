// X2H attention on the Hopper tensor cores (wgmma): one CTA tile = 4 destination nodes x 32 in-edges = 128 edge rows,
// two warpgroups of 64 rows (2 nodes) each.
//
// Reference semantics: repo/modules/attention/x2h_attention.py:43-97 (per edge e = (j -> i):
//   kv = [onehot(type) | onehot(type) (x) g(d) | h_i | h_j], k = MLP_k(kv), v = MLP_v(kv) * e_w,
//   alpha = softmax_j(<q_i, k_ij>/sqrt(8)) per head, h_i += sum_j alpha_ij v_ij).
//
// Both edge MLPs are 340 -> 128 -> LayerNorm -> ReLU -> 128.  Per 64-row half tile a warpgroup runs two GEMMs:
//   MMA1  pre[64 x 128] = G[64 x 96] * Wg[96 x 128]        G = [onehot(t) (x) g(d) | onehot(t)], Wg = [Wrf[t] ; c[t]]
//         (the type-dependent RBF mat-vec and the type bias in one K = 96 product, A and B from shared memory; the
//          node planes Pi[i] and Pj[j] are added to the accumulator fragment straight from global memory / L2)
//   MMA2  out[64 x 128] = relu(LN(pre + Pi + Pj)) * W1^T   (A from REGISTERS: the fp32 accumulator fragment of MMA1,
//         packed to f16 pairs, is exactly the A fragment wgmma expects - the activations never touch shared memory)
// fp32 accuracy comes from the split x = hi + lo into two f16 values (scaled by powers of two so lo stays normal)
// and the three products hi*hi + hi*lo + lo*hi accumulated in fp32 (cbg_tc.cuh): same error class as 3xTF32
// at twice the tensor-core rate and half the operand bytes.
//
// B operands (weight images, pre-split and pre-laid-out by the host packer) stay resident in shared memory for the whole
// persistent CTA (bulk copies, mbarrier).  Nothing of size [E, 128] touches HBM and no R-cache is needed: the only
// per-edge gather is the 512-byte Pj row, read in the accumulator layout (a quad of lanes = one 32-byte sector of a row).
// In that layout a row's 128 columns live in the 4 lanes of a quad, so LayerNorm is two shuffles, and a head's 8 columns
// are one quad's registers, so <q_i, k> per head is a reduction over the quad as well; the softmax over a node's 32
// edges (2 warps) and the sum over them go through a small shared-memory buffer.  The two warpgroups only share the
// weights: each walks its own 2 nodes of every tile, and while one waits on its MMAs or gathers the other one computes.
//
// H2X (repo/modules/attention/h2x_attention.py:34-73) runs on the same kernel over the list of generated nodes:
//   launch 1  MODE_K with the xk / xq weights -> w = alpha * e_w (compact buffer, indexed by list position)
//   launch 2  MODE_XV with the xv weights: the second Linear has one output per head (N = 16 MMA), and the epilogue forms
//             dx_i = (1/16) sum_e (sum_hd w_e,hd (v_e,hd + b1_hd)) (x_i - x_j)     (mean over heads of alpha * v * e_w * rel_x)
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <type_traits>
#include "cbg_kernels.cuh"
#include "cbg_tc.cuh"

using namespace cbg_tc;

namespace {

// ---- blob fields ------------------------------------------------------------------------------------------------
constexpr long long kOffKW1 = cbg_layout::layer_offset(CBG_LF_X2H_K_TCW1);
constexpr long long kOffKWg = cbg_layout::layer_offset(CBG_LF_X2H_K_TCWG);
constexpr long long kOffVW1 = cbg_layout::layer_offset(CBG_LF_X2H_V_TCW1);
constexpr long long kOffVWg = cbg_layout::layer_offset(CBG_LF_X2H_V_TCWG);
constexpr long long kOffKLn = cbg_layout::layer_offset(CBG_LF_X2H_K_LN);
constexpr long long kOffVLn = cbg_layout::layer_offset(CBG_LF_X2H_V_LN);
constexpr long long kOffVB1 = cbg_layout::layer_offset(CBG_LF_X2H_V_B1);
constexpr long long kOffRbf = cbg_layout::layer_offset(CBG_LF_X2H_K_RBF);
constexpr long long kOffXKW1 = cbg_layout::layer_offset(CBG_LF_H2X_K_TCW1);
constexpr long long kOffXKWg = cbg_layout::layer_offset(CBG_LF_H2X_K_TCWG);
constexpr long long kOffXVW1 = cbg_layout::layer_offset(CBG_LF_H2X_V_TCW1);
constexpr long long kOffXVWg = cbg_layout::layer_offset(CBG_LF_H2X_V_TCWG);
constexpr long long kOffXKLn = cbg_layout::layer_offset(CBG_LF_H2X_K_LN);
constexpr long long kOffXVLn = cbg_layout::layer_offset(CBG_LF_H2X_V_LN);
constexpr long long kOffXVB1 = cbg_layout::layer_offset(CBG_LF_H2X_V_B1);
constexpr long long kOffXRbf = cbg_layout::layer_offset(CBG_LF_H2X_RBF);

// what a launch computes; the weight fields it uses travel in TcWeights (filled by the launcher)
enum { MODE_K = 0, MODE_V = 1, MODE_XV = 2 };
struct TcWeights {
  const float* w1;     // (hi | lo) image of the second Linear: [128 n][128 k], MODE_XV [16 n][128 k]
  const float* wg;     // (hi | lo) image of [Wrf ; c ; Pi columns]
  const float* ln;     // gamma[128], beta[128]
  const float* b1;     // second-Linear bias (MODE_V: 128, MODE_XV: 16; unused by MODE_K - it cancels in the softmax)
  const float* rbf;    // Gaussian offsets [20], coefficient at [20]
};

// ---- scales (exact powers of two; must match modules.py: tc_f16_image) ----------------------------------------
// Wrf, c in Wg are scaled by 16 (packer)                       -> pre accumulates at 2^14
constexpr float kInvPre = 1.f / 16384.f;
constexpr uint32_t kHalfTypeOne = 0x6400u;   // f16 1024
constexpr float kScaleA = 64.f;          // activations
constexpr float kInvOut = 1.f / 4096.f;  // W1 image is scaled by 64 -> out accumulates at 2^12

// ---- shapes -----------------------------------------------------------------------------------------------------
constexpr int KG = 96;                   // K of MMA1 (84 used: the packer leaves k >= 84 of the Wg images zero)
constexpr int KG_LO = 80;                // the lo part of G is non-zero only in the RBF columns
constexpr uint32_t W1_IMG = 128 * 128 * 2;            // one (hi | lo) image, bytes
constexpr uint32_t W1X_IMG = 16 * 128 * 2;            // MODE_XV: 16 output rows
constexpr uint32_t WG_IMG = 128 * KG * 2;
constexpr uint32_t G_IMG = 64 * KG * 2;               // one warpgroup's G rows (hi or lo), same layout as the weight images
constexpr uint32_t W1_SBO = (128 / 8) * 128, WG_SBO = (KG / 8) * 128, LBO = 128;
constexpr uint32_t SM_W1 = 0;                         // hi | lo
constexpr uint32_t SM_WG = SM_W1 + 2 * W1_IMG;
constexpr uint32_t SM_G = SM_WG + 2 * WG_IMG;         // [warpgroup][hi | lo]
constexpr uint32_t SM_LN = SM_G + 4 * G_IMG;          // gamma * 64 [128] | beta * 64 [128]
constexpr uint32_t SM_B1 = SM_LN + 1024;              // b1v [128]
constexpr uint32_t SM_RBF = SM_B1 + 512;              // Gaussian offsets [20] + coeff
constexpr uint32_t SM_EPI = SM_RBF + 128;             // k: [node slot][32 edges][17] logits; v: [slot][warp][128] partial sums; xv: [slot][warp][4]
// Staged node-plane rows of the tile in flight, per warp: the Pi row of its node, then the Pj rows of its accumulator
// rows e0 (row r = lane / 4).  The Pj rows are 512 + 32 bytes apart, so that the 64-bit accumulator-layout reads of a
// half-warp (rows r .. r + 3) fall on 32 different banks.
constexpr uint32_t P_ROW = CBG_H * 4;                 // one fp32 node-plane row, bytes
constexpr uint32_t STG_WARP = P_ROW + 8 * (P_ROW + 32);
constexpr uint32_t SM_BAR = SM_EPI + 4 * 32 * 17 * 4;
constexpr uint32_t SM_STG = SM_BAR + 128;             // [warp][Pi | Pj rows 0 .. 7]
// STAGE: the whole layout; !STAGE ends before the staging slots, so its shared-memory carve-out (and L1) stays as it was
constexpr uint32_t sm_total(bool stage) { return stage ? SM_STG + 8 * STG_WARP : SM_STG; }
static_assert(sm_total(true) <= 232448, "shared memory budget");
static_assert(SM_STG % 16 == 0 && STG_WARP % 16 == 0, "bulk-copy destinations are 16-byte aligned");
enum { B_WFULL = 0 /* Wg images */, B_W1FULL /* W1 images */, B_STG /* + warp: staged rows of the warp */ };
__host__ __device__ constexpr uint32_t stg_pj_row(int r) { return P_ROW + (P_ROW + 32u) * (uint32_t)r; }

__device__ __forceinline__ int list_len(const EdgeArgs& p) {
  int n = p.n_nodes;
  if (p.n_nodes_dev) { const int nd = *p.n_nodes_dev; n = nd < n ? nd : n; }
  return n;
}
__device__ __forceinline__ int node_of(const EdgeArgs& p, int n, int n_list) {
  const int nc = n < n_list ? n : n_list - 1;
  return p.node_idx ? p.node_idx[nc] : nc;
}
__device__ __forceinline__ float quad_sum(float v) {        // fixed butterfly order: deterministic
  v += __shfl_xor_sync(CBG_FULL, v, 1);
  return v + __shfl_xor_sync(CBG_FULL, v, 2);
}
__device__ __forceinline__ float rows_sum(float v) {        // over the 8 row groups of a warp (lanes with equal lane % 4)
  v += __shfl_xor_sync(CBG_FULL, v, 4);
  v += __shfl_xor_sync(CBG_FULL, v, 8);
  return v + __shfl_xor_sync(CBG_FULL, v, 16);
}
// Reduce-scatter of a[0 .. N) over the lanes that differ in lane bits LB .. LB + LEVELS - 1, for epilogues where each
// sum is stored by one lane only.  Level l pairs the lanes as the butterfly's xor (1 << (LB + l)) does; each lane sends
// the half of its values whose index bit IB differs from its lane bit LB + l and adds the partner's copy of the half it
// keeps, own + partner as in the butterfly.  So every kept value is the same fp32 sum tree, bit for bit, that
// quad_sum / rows_sum leave in every lane; which lane keeps which value only decides where its store comes from.  The kept
// values are compacted in place (index bit IB removed, higher bits shift down): afterwards a lane holds a[0 .. N >> LEVELS),
// the values whose original index bits IB .. IB + LEVELS - 1 equal its lane bits LB .. LB + LEVELS - 1.
// N (1 - 2^-LEVELS) shuffles instead of the butterfly's N LEVELS; fully unrolled, constant indices: registers only.
// (One level per instantiation, so that every loop has a constant trip count and the array stays in registers.)
template <int IB, int LB, int LEVELS, int N, int LIVE = N>
__device__ __forceinline__ void reduce_scatter(float (&a)[N], int lane) {
  static_assert((LIVE >> LEVELS) << LEVELS == LIVE && (LIVE >> LEVELS) >= (1 << IB), "reduce_scatter shape");
  const bool up = (lane >> LB) & 1;
#pragma unroll
  for (int o = 0; o < LIVE / 2; ++o) {      // o <= i0 < i1: the in-place write never clobbers a later read
    const int i0 = ((o >> IB) << (IB + 1)) | (o & ((1 << IB) - 1)), i1 = i0 | (1 << IB);
    const float give = up ? a[i0] : a[i1];
    const float keep = up ? a[i1] : a[i0];
    a[o] = keep + __shfl_xor_sync(CBG_FULL, give, 1 << LB);
  }
  if constexpr (LEVELS > 1) reduce_scatter<IB, LB + 1, LEVELS - 1, N, LIVE / 2>(a, lane);
}
__device__ __forceinline__ float2 ldg2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }

// pipeline event stamps of warpgroup 0 of CTA 0 (debugging; p.trace == nullptr in production: one predicated-off branch per
// event).  Events of tile k, in loop order: 0 MMA1(k) complete, 1 MMA2(k) issued (S1 done), 2 MMA2(k) complete (G(k+1)
// built meanwhile), 3 MMA1(k+1) issued (G(k+1) handed over; not stamped on the last tile), 4 epilogue(k) done
#define TC_STAMP(k, ev)                                                                                  \
  do {                                                                                                   \
    if (p.trace != nullptr && blockIdx.x == 0 && tid == 0 && (k) < p.trace_tiles) p.trace[(k) * 16 + (ev)] = clock64(); \
  } while (0)

// =================================================================================================================
// STAGE: the Pi row and the Pj rows of accumulator row e0 reach S1 through shared memory (bulk copies issued one tile
// ahead); the Pj rows of e0 + 8 through registers.  !STAGE (MODE_V, or any mode under CBG_X2H_STAGE=0): Pi + Pj of both
// rows gathered into registers during the previous epilogue.  Same values, same arithmetic: bit-identical results.
template <int MODE, bool STAGE>
__global__ void __launch_bounds__(256, 1) x2h_tc_kernel(EdgeArgs p, TcWeights W) {
  constexpr bool IS_V = MODE == MODE_V, IS_XV = MODE == MODE_XV;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t sbase = smem_u32(smem);
  constexpr uint32_t W1B = IS_XV ? W1X_IMG : W1_IMG;      // bytes of one second-Linear image
  const uint32_t bars = sbase + SM_BAR;
  auto bar = [&](int i) { return bars + 8u * (uint32_t)i; };

  // ---- prologue: nothing here reads what the previous kernel of the stream produces (weights are constants), so with a
  // programmatic dependent launch it overlaps that kernel's tail; pdl_wait() below is the dependency
  pdl_launch_dependents();
  // debugging: CTA 0 stamps kernel entry / end of prologue / exit into the row behind the per-tile rows of the trace buffer
#define TC_STAMP_CTA(ev) do { if (p.trace != nullptr && blockIdx.x == 0 && tid == 0) p.trace[p.trace_tiles * 16 + (ev)] = clock64(); } while (0)
  TC_STAMP_CTA(0);
  if (tid == 32) {
    mbar_init(bar(B_WFULL), 1);
    mbar_init(bar(B_W1FULL), 1);
    if constexpr (STAGE) {
      for (int w = 0; w < 8; ++w) mbar_init(bar(B_STG + w), 1);
    }
    fence_mbar_init();
    // Resident weight images by bulk (TMA) copies.  Wg first on its own barrier: MMA1 of the first tile needs only Wg,
    // W1 is not read before MMA2.  Every CTA of the grid reads the same 112 KB at the same moment, so each image goes
    // in four pieces whose order is rotated by the CTA index: at any time the CTAs pull different L2 lines.
    mbar_expect_tx(bar(B_WFULL), 2 * WG_IMG);
    mbar_expect_tx(bar(B_W1FULL), 2 * W1B);
    const uint32_t rot = blockIdx.x & 3u;
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i) {
      const uint32_t pc = (i + rot) & 3u, nb = (2 * WG_IMG) / 4;
      bulk_g2s(sbase + SM_WG + pc * nb, reinterpret_cast<const uint8_t*>(W.wg) + pc * nb, nb, bar(B_WFULL));
    }
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i) {
      const uint32_t pc = (i + rot) & 3u, nb = (2 * W1B) / 4;
      bulk_g2s(sbase + SM_W1 + pc * nb, reinterpret_cast<const uint8_t*>(W.w1) + pc * nb, nb, bar(B_W1FULL));
    }
  }
  {   // LayerNorm affine (pre-multiplied by the activation scale), the value bias and the Gaussian table
    float* s_ln = reinterpret_cast<float*>(smem + SM_LN);
    float* s_b1 = reinterpret_cast<float*>(smem + SM_B1);
    s_ln[tid] = W.ln[tid] * kScaleA;
    if (tid < 128) s_b1[tid] = (IS_V || (IS_XV && tid < CBG_HEADS)) ? W.b1[tid] : 0.f;
    else if (tid < 128 + 24) reinterpret_cast<float*>(smem + SM_RBF)[tid - 128] = W.rbf[tid - 128];
  }
  pdl_wait();
  const int n_list = list_len(p);
  const int n_tiles = (n_list + 3) >> 2;
  const bool has_work = (int)blockIdx.x < n_tiles;
  const int n_my = has_work ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;     // tiles of this CTA: blockIdx.x + k * gridDim.x
  // node of slot `slot` of this CTA's kk-th tile (clamped to the list: surplus slots of the last tile redo the last node)
  auto tile_node = [&](int kk, int slot) { return node_of(p, 4 * ((int)blockIdx.x + kk * (int)gridDim.x) + slot, n_list); };
  __syncthreads();
  TC_STAMP_CTA(1);
  // the bulk copies must land before the CTA reads the images - or exits (device-side list shorter than the grid)
  mbar_wait(bar(B_WFULL), 0u);
  mbar_wait(bar(B_W1FULL), 0u);

  // ---- thread roles ------------------------------------------------------------------------------------------------
  const int wg = warp >> 2, w4 = warp & 3, qg = lane >> 2, qt = lane & 3;
  // G build: thread = (row of the warpgroup's half tile, hi | lo image)
  const int g_row = tid & 63, g_part = (tid >> 6) & 1;
  const int g_slot = 2 * wg + (g_row >> 5);
  // MMA fragments / epilogue: node slot of this warp, its two edge rows e0 and e0 + 8 of the node's 32
  const int slot = 2 * wg + (w4 >> 1), wp = w4 & 1, e0 = 16 * wp + qg;
  const float* rbf = reinterpret_cast<const float*>(smem + SM_RBF);
  const float c2 = rbf[20] * 1.4426950408889634f;      // exp(c u^2) = 2^(c log2(e) u^2)
  const float* s_ln = reinterpret_cast<const float*>(smem + SM_LN);
  const float* s_b1 = reinterpret_cast<const float*>(smem + SM_B1);
  float* s_epi = reinterpret_cast<float*>(smem + SM_EPI);
  const float* pj_plane = MODE != MODE_K ? p.pj_v : p.pj_k;
  const float* pi_plane = MODE != MODE_K ? p.pi_v : p.pi_k;
  const uint32_t g_base = sbase + SM_G + (uint32_t)wg * 2u * G_IMG;
  const uint64_t dg_hi = smem_desc(g_base, LBO, WG_SBO), dg_lo = smem_desc(g_base + G_IMG, LBO, WG_SBO);
  const uint64_t dw_hi = smem_desc(sbase + SM_WG, LBO, WG_SBO), dw_lo = smem_desc(sbase + SM_WG + WG_IMG, LBO, WG_SBO);
  const uint64_t d1_hi = smem_desc(sbase + SM_W1, LBO, W1_SBO), d1_lo = smem_desc(sbase + SM_W1 + W1B, LBO, W1_SBO);

  // ---- stages of a tile ----------------------------------------------------------------------------------------------
  // Index loads of tile kk: the node and neighbour of this thread's G row, the node and the two neighbours of its two
  // accumulator rows
  auto load_idx = [&](int kk, int& gi, int& gjn, int& ti, int& tj0, int& tj1) {
    gi = tile_node(kk, g_slot);
    gjn = p.nbr[(size_t)gi * CBG_KMAX + (g_row & 31)];
    ti = tile_node(kk, slot);
    const size_t eoff = (size_t)ti * CBG_KMAX + e0;
    tj0 = p.nbr[eoff];
    tj1 = p.nbr[eoff + 8];
  };
  // G row of this thread's edge into the warpgroup's G buffer (x2h_attention.py:46-52, unitransformer.py:88-99; explicit
  // operation order: position-independent results; the factor 1024 of the G scale rides in the exponent).  Type block tb
  // occupies k = 20 tb .. 20 tb + 19, the type one-hot k = 80 .. 83 of G_hi.
  auto build_g = [&](const float4 xi, const float4 xj) {
    const float rx = xi.x - xj.x, ry = xi.y - xj.y, rz = xi.z - xj.z;
    const float d = sqrtf(__fmaf_rn(rz, rz, __fmaf_rn(ry, ry, __fmul_rn(rx, rx))));
    const int fi = node_flags(xi), fj = node_flags(xj);
    const int t_e = ((fj & 1) ? 0 : 2) + ((fi & 1) ? 0 : 1);
    uint32_t gv[10];
#pragma unroll
    for (int mp = 0; mp < 10; ++mp) {
      const float u0 = d - rbf[2 * mp], u1 = d - rbf[2 * mp + 1];
      float g0, g1;
      asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(g0) : "f"(fmaf(c2 * u0, u0, 10.f)));
      asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(g1) : "f"(fmaf(c2 * u1, u1, 10.f)));
      uint32_t hi, lo;
      split_pair(g0, g1, hi, lo);
      gv[mp] = g_part ? lo : hi;
    }
    uint8_t* grow = smem + SM_G + (uint32_t)(2 * wg + g_part) * G_IMG + (uint32_t)(g_row >> 3) * WG_SBO + (uint32_t)(g_row & 7) * 16u;
#pragma unroll
    for (int c = 0; c < KG_LO / 8; ++c) {        // 16-byte core-matrix rows: f16 pairs 4 c .. 4 c + 3
      uint4 w;
      w.x = (t_e == (4 * c) / 10) ? gv[(4 * c) % 10] : 0u;
      w.y = (t_e == (4 * c + 1) / 10) ? gv[(4 * c + 1) % 10] : 0u;
      w.z = (t_e == (4 * c + 2) / 10) ? gv[(4 * c + 2) % 10] : 0u;
      w.w = (t_e == (4 * c + 3) / 10) ? gv[(4 * c + 3) % 10] : 0u;
      *reinterpret_cast<uint4*>(grow + 128u * c) = w;
    }
    if (g_part == 0) {        // k = 80 .. 95 exist in G_hi only: the type one-hot, then zeros
      uint4 w = make_uint4(0u, 0u, 0u, 0u);
      w.x = (t_e == 0) ? kHalfTypeOne : ((t_e == 1) ? (kHalfTypeOne << 16) : 0u);
      w.y = (t_e == 2) ? kHalfTypeOne : ((t_e == 3) ? (kHalfTypeOne << 16) : 0u);
      *reinterpret_cast<uint4*>(grow + 128u * 10) = w;
      *reinterpret_cast<uint4*>(grow + 128u * 11) = make_uint4(0u, 0u, 0u, 0u);
    }
  };
  // MMA1, issued and committed, not waited for: small terms first
  auto issue_mma1 = [&](float (&d)[64]) {
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < KG_LO / 16; ++ks) {
      if (ks == 0) wgmma_f16_ss_first(d, dg_lo, dw_hi);
      else wgmma_f16_ss(d, dg_lo + 16u * ks, dw_hi + 16u * ks, 1u);
    }
#pragma unroll
    for (int ks = 0; ks < KG / 16; ++ks) wgmma_f16_ss(d, dg_hi + 16u * ks, dw_lo + 16u * ks, 1u);
#pragma unroll
    for (int ks = 0; ks < KG / 16; ++ks) wgmma_f16_ss(d, dg_hi + 16u * ks, dw_hi + 16u * ks, 1u);
    wgmma_commit();
    wgmma_settle(d);
  };
  // Pi[i] + Pj[j] of this thread's two accumulator rows in the accumulator layout, columns 8 j + 2 qt, + 1
  auto gather_p = [&](float (&v)[64], int j, int ti, int tj0, int tj1) {
    const float2 a = ldg2(pi_plane + (size_t)ti * CBG_H + 2 * qt + 8 * j);
    const float2 b0 = ldg2(pj_plane + (size_t)(tj0 >= 0 ? tj0 : ti) * CBG_H + 2 * qt + 8 * j);
    const float2 b1 = ldg2(pj_plane + (size_t)(tj1 >= 0 ? tj1 : ti) * CBG_H + 2 * qt + 8 * j);
    v[4 * j] = a.x + b0.x; v[4 * j + 1] = a.y + b0.y; v[4 * j + 2] = a.x + b1.x; v[4 * j + 3] = a.y + b1.y;
  };
  // STAGE: bulk copies of a tile's Pi row and the warp's eight e0 Pj rows into the warp's staging slot, completing on
  // the warp's barrier (one phase per tile).  The caller guarantees that every lane has read the slot's previous rows.
  const uint32_t stg = sbase + SM_STG + (uint32_t)warp * STG_WARP;
  const uint8_t* s_stg = smem + SM_STG + (uint32_t)warp * STG_WARP;
  auto stage_rows = [&](int sti, int stj0) {
    __syncwarp();
    if (lane == 0) mbar_expect_tx(bar(B_STG + warp), 9 * P_ROW);
    if (qt == 0) bulk_g2s(stg + stg_pj_row(qg), pj_plane + (size_t)(stj0 >= 0 ? stj0 : sti) * CBG_H, P_ROW, bar(B_STG + warp));
    else if (lane == 1) bulk_g2s(stg, pi_plane + (size_t)sti * CBG_H, P_ROW, bar(B_STG + warp));
  };
  // STAGE: Pj of accumulator row e0 + 8 into registers, columns 8 j + 2 qt, + 1 (S1 adds Pi)
  auto gather_pj1 = [&](float (&b)[32], int sti, int stj1) {
    const float* r = pj_plane + (size_t)(stj1 >= 0 ? stj1 : sti) * CBG_H + 2 * qt;
#pragma unroll
    for (int j = 0; j < 16; ++j) { const float2 t = ldg2(r + 8 * j); b[2 * j] = t.x; b[2 * j + 1] = t.y; }
  };

  // ---- software pipeline over this CTA's tiles.  Per warpgroup, tile k:
  //   wait MMA1(k), S1(k), issue MMA2(k) | load the coordinates of k+1, build G(k+1) while MMA2(k) runs | wait MMA2(k),
  //   issue MMA1(k+1) | epilogue(k) while MMA1(k+1) runs (it issues the Pi + Pj gathers of k+1 as it frees registers)
  // The G buffer is free once every warp of the warpgroup has completed MMA1(k) (MMA2 reads no G), and the s_epi slots once
  // every warp has finished epilogue(k-1): one warpgroup barrier after the MMA2 issue orders both.
  // STAGE: the staged rows of tile k+1 are copied as soon as S1(k) has read those of tile k, and the e0 + 8 Pj row is
  // loaded behind MMA2(k): each gets most of a tile period to land.
  float d[64];               // MMA1 accumulator of the tile in flight
  float v[64];               // Pi + Pj of the tile in flight
  float pj1[32];             // STAGE: Pj of row e0 + 8 of the tile in flight
  int ti = 0, tj0 = 0, tj1 = 0;                        // node / neighbours of this thread's accumulator rows, tile k
  int ngi = 0, ngjn = 0, nti = 0, ntj0 = 0, ntj1 = 0;  // the same of tile k+1, and its G-row node / neighbour
  if (n_my > 0) {          // prologue: tile 0 up to its MMA1 issue
    int gi, gjn;
    load_idx(0, gi, gjn, ti, tj0, tj1);
    if constexpr (STAGE) {
      stage_rows(ti, tj0);
      gather_pj1(pj1, ti, tj1);
    }
    build_g(p.x4[gi], p.x4[gjn >= 0 ? gjn : gi]);
    fence_proxy_async();
    warpgroup_sync(wg);
    issue_mma1(d);
    if constexpr (!STAGE) {
#pragma unroll
      for (int j = 0; j < 16; ++j) gather_p(v, j, ti, tj0, tj1);
    }
  }
  // one tile; `more` (a compile-time constant: the last tile is peeled) says whether a tile k+1 follows, so the compiler
  // sees exactly where d and v are redefined and keeps neither live across the drain
  auto tile = [&](const int k, auto more_c) {
    constexpr bool more = decltype(more_c)::value;
    if constexpr (more) load_idx(k + 1, ngi, ngjn, nti, ntj0, ntj1);     // dependent index loads: their latency hides behind MMA1(k)
    wgmma_wait0();
    wgmma_settle(d);
    TC_STAMP(k, 0);
    // ---- inputs of this thread's two accumulator rows
    const int n = 4 * ((int)blockIdx.x + k * (int)gridDim.x) + slot;
    const bool live = n < n_list;
    const int i = ti;
    const int w_row = p.w_compact ? (n < n_list ? n : n_list - 1) : i;       // row of the w buffer: list position (H2X) or node id
    // ---- S1: pre = acc + Pi + Pj -> LayerNorm -> ReLU -> (hi, lo) f16 A fragments.  The first Linear is centred over
    // the feature axis by the packer, so pre has zero mean and LayerNorm needs only the sum of squares.
    uint32_t a_hi[8][4], a_lo[8][4];
    {
      float q0 = 0.f, q1 = 0.f;
      if constexpr (STAGE) {     // Pi + Pj from the staged rows and pj1, added as gather_p adds them
        mbar_wait(bar(B_STG + warp), (uint32_t)k & 1u);
        const float* s_pi = reinterpret_cast<const float*>(s_stg) + 2 * qt;
        const float* s_pj = reinterpret_cast<const float*>(s_stg + stg_pj_row(qg)) + 2 * qt;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float2 a = *reinterpret_cast<const float2*>(s_pi + 8 * j);
          const float2 b0 = *reinterpret_cast<const float2*>(s_pj + 8 * j);
          v[4 * j] = a.x + b0.x; v[4 * j + 1] = a.y + b0.y; v[4 * j + 2] = a.x + pj1[2 * j]; v[4 * j + 3] = a.y + pj1[2 * j + 1];
        }
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        v[4 * j] = fmaf(d[4 * j], kInvPre, v[4 * j]);
        v[4 * j + 1] = fmaf(d[4 * j + 1], kInvPre, v[4 * j + 1]);
        v[4 * j + 2] = fmaf(d[4 * j + 2], kInvPre, v[4 * j + 2]);
        v[4 * j + 3] = fmaf(d[4 * j + 3], kInvPre, v[4 * j + 3]);
        q0 = fmaf(v[4 * j], v[4 * j], q0); q0 = fmaf(v[4 * j + 1], v[4 * j + 1], q0);
        q1 = fmaf(v[4 * j + 2], v[4 * j + 2], q1); q1 = fmaf(v[4 * j + 3], v[4 * j + 3], q1);
      }
      float rs[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float var = quad_sum(h ? q1 : q0) * (1.f / 128.f) + 1e-5f;
        const float r = rsqrtf(var);                      // MUFU.RSQ + one Newton step: < 1 ulp
        rs[h] = r * (1.5f - 0.5f * var * r * r);
      }
      // relu((pre * rstd) * gamma + beta) * 64; accumulator columns 16 s .. 16 s + 15 are the A fragment of K step s
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 ga = *reinterpret_cast<const float2*>(s_ln + 8 * j + 2 * qt);
        const float2 be = *reinterpret_cast<const float2*>(s_ln + 128 + 8 * j + 2 * qt);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float y0 = fmaf(v[4 * j + 2 * h] * rs[h], ga.x, be.x), y1 = fmaf(v[4 * j + 2 * h + 1] * rs[h], ga.y, be.y);
          split_pair_relu(y0, y1, a_hi[j >> 1][2 * (j & 1) + h], a_lo[j >> 1][2 * (j & 1) + h]);
        }
      }
    }
    // ---- MMA2 (A from REGISTERS: a_hi / a_lo stay untouched until it completes), issued and committed
    auto issue_mma2 = [&](auto& o) {
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        if constexpr (IS_XV) wgmma_f16_rs_n16(o, a_lo[ks], d1_hi + 16u * ks, ks > 0 ? 1u : 0u);
        else wgmma_f16_rs(o, a_lo[ks], d1_hi + 16u * ks, ks > 0 ? 1u : 0u);
      }
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        if constexpr (IS_XV) wgmma_f16_rs_n16(o, a_hi[ks], d1_lo + 16u * ks, 1u);
        else wgmma_f16_rs(o, a_hi[ks], d1_lo + 16u * ks, 1u);
      }
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        if constexpr (IS_XV) wgmma_f16_rs_n16(o, a_hi[ks], d1_hi + 16u * ks, 1u);
        else wgmma_f16_rs(o, a_hi[ks], d1_hi + 16u * ks, 1u);
      }
      wgmma_commit();
      wgmma_settle(o);
      TC_STAMP(k, 1);
    };
    // ---- while MMA2(k) runs: G(k+1); then MMA2(k) complete, MMA1(k+1) issued
    auto advance = [&](auto& o) {
      if constexpr (more && STAGE) {
        stage_rows(nti, ntj0);                         // S1(k) has read the slot: the __syncwarp in stage_rows orders it
        gather_pj1(pj1, nti, ntj1);
      }
      if constexpr (more) {
        const float4 xi = p.x4[ngi], xj = p.x4[ngjn >= 0 ? ngjn : ngi];
        warpgroup_sync(wg);                            // MMA1(k) complete and epilogue(k-1) done in every warp
        build_g(xi, xj);
        fence_proxy_async();
      } else {
        warpgroup_sync(wg);                            // epilogue(k-1) done in every warp
      }
      wgmma_wait0();
      wgmma_settle(o);
      TC_STAMP(k, 2);
      if constexpr (more) {
        warpgroup_sync(wg);                            // G(k+1) complete
        issue_mma1(d);
        TC_STAMP(k, 3);
      }
    };
    // ---- epilogue(k) from the MMA2 fragment, while MMA1(k+1) runs.  The Pi + Pj gathers of k+1 are issued column
    // group by column group as the epilogue frees the fragment registers of the same group: they start early, and o and
    // v are never both live in full
    auto gather_next = [&](int j) { if constexpr (more && !STAGE) gather_p(v, j, nti, ntj0, ntj1); };
    if constexpr (MODE == MODE_K) {
      // attention weights: <q_i, k> per head (a head's 8 columns = one quad's registers), softmax over the node's 32
      // edges through shared memory, w = alpha * e_w
      float qv[32];
      {
        const float* qr = p.q + (size_t)i * CBG_H + 2 * qt;
#pragma unroll
        for (int j = 0; j < 16; ++j) { const float2 t = ldg2(qr + 8 * j); qv[2 * j] = t.x; qv[2 * j + 1] = t.y; }
      }
      // softmax role: lane = (head, half of the edges); this warp stores edges 16 half + 8 wp .. + 7
      const int hd = lane & 15, eh = 16 * (lane >> 4);
      float sc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const size_t eo = (size_t)i * CBG_KMAX + eh + 8 * wp + j;
        sc[j] = p.nbr[eo] >= 0 ? p.ew[eo] : 0.f;
      }
      float o[64];
      issue_mma2(o);
      advance(o);
      float* s_sm = s_epi + slot * (32 * 17);              // [edge][17]: the softmax reads it without bank conflicts
      // heads 4 m .. 4 m + 3 at a time: the quad's partial dot products are reduce-scattered over the quad, lane qt keeps
      // head 4 m + qt of both rows (these stores have two-way bank conflicts; the rows stay padded to 17 for the softmax)
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        float lg[8];                                       // [head 4 m + jj][row e0 | e0 + 8]
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = 4 * m + jj;
          lg[2 * jj] = fmaf(o[4 * j + 1], qv[2 * j + 1], o[4 * j] * qv[2 * j]);
          lg[2 * jj + 1] = fmaf(o[4 * j + 3], qv[2 * j + 1], o[4 * j + 2] * qv[2 * j]);
          gather_next(j);
        }
        reduce_scatter<1, 0, 2>(lg, lane);                 // xor 1, xor 2: quad_sum's tree
        s_sm[e0 * 17 + 4 * m + qt] = tj0 >= 0 ? lg[0] * kInvOut : -INFINITY;
        s_sm[(e0 + 8) * 17 + 4 * m + qt] = tj1 >= 0 ? lg[1] * kInvOut : -INFINITY;
      }
      warpgroup_sync(wg);
      {
        float l[16];
        float mx = -INFINITY;
#pragma unroll
        for (int j = 0; j < 16; ++j) { l[j] = s_sm[(eh + j) * 17 + hd]; mx = fmaxf(mx, l[j]); }
        mx = fmaxf(mx, __shfl_xor_sync(CBG_FULL, mx, 16));
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) { l[j] = (mx == -INFINITY) ? 0.f : __expf(l[j] - mx); sum += l[j]; }
        sum += __shfl_xor_sync(CBG_FULL, sum, 16);
        const float inv = 1.f / ((sum > 0.f) ? sum : 1.f);
        if (live) {      // 16 lanes = the 16 heads of one edge: 64-byte rows
          float* wo = p.w + ((size_t)w_row * CBG_KMAX + eh + 8 * wp) * CBG_HEADS + hd;
#pragma unroll
          for (int j = 0; j < 8; ++j) wo[j * CBG_HEADS] = (wp ? l[8 + j] : l[j]) * inv * sc[j];
        }
      }
    } else if constexpr (IS_V) {
      // aggregation: (v + b1v) * w summed over the node's 32 edges, h_i +=
      float wv[2][CBG_HEADS];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float* wi = p.w + ((size_t)w_row * CBG_KMAX + e0 + 8 * h) * CBG_HEADS;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float4 t = ld4(wi + 4 * j);
          wv[h][4 * j] = t.x; wv[h][4 * j + 1] = t.y; wv[h][4 * j + 2] = t.z; wv[h][4 * j + 3] = t.w;
        }
      }
      // this thread's two h_i values, read early: every node is listed once and no other thread writes its row
      const int c = 2 * (32 * wp + lane);
      float2* hp = reinterpret_cast<float2*>(p.h + (size_t)i * CBG_H + c);
      const float2 hv = *hp;
      float o[64];
      issue_mma2(o);
      advance(o);
      float* s_vr = s_epi + (slot * 2 + wp) * CBG_H;       // this warp's 16-edge partial sums
      // columns 64 b .. 64 b + 63 at a time: the per-row terms are reduce-scattered over the warp's 8 row groups, lane qg
      // keeps column group 8 b + qg (one conflict-free float2 row store per half)
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        float s[16];                                       // [column group 8 b + jj][column 2 qt | 2 qt + 1]
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = 8 * b + jj;
          const float2 b1 = *reinterpret_cast<const float2*>(s_b1 + 8 * j + 2 * qt);
          s[2 * jj] = fmaf(fmaf(o[4 * j + 2], kInvOut, b1.x), wv[1][j], fmaf(o[4 * j], kInvOut, b1.x) * wv[0][j]);
          s[2 * jj + 1] = fmaf(fmaf(o[4 * j + 3], kInvOut, b1.y), wv[1][j], fmaf(o[4 * j + 1], kInvOut, b1.y) * wv[0][j]);
          gather_next(j);
        }
        reduce_scatter<1, 2, 3>(s, lane);                  // xor 4, 8, 16: rows_sum's tree
        *reinterpret_cast<float2*>(s_vr + 64 * b + 8 * qg + 2 * qt) = make_float2(s[0], s[1]);
      }
      warpgroup_sync(wg);
      if (live) {
        const float* s0 = s_epi + (slot * 2) * CBG_H + c;
        *hp = make_float2(hv.x + (s0[0] + s0[CBG_H]), hv.y + (s0[1] + s0[CBG_H + 1]));
      }
    } else {
      // H2X coordinate update: s_e = sum_hd w_e,hd (v_e,hd + b1_hd), dx_i = (1/16) sum_e s_e (x_i - x_j)
      float2 wx[2][2];
      float rel[2][3];
      {
        const float4 xi = p.x4[i];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float* wi = p.w + ((size_t)w_row * CBG_KMAX + e0 + 8 * h) * CBG_HEADS + 2 * qt;
          wx[h][0] = *reinterpret_cast<const float2*>(wi);
          wx[h][1] = *reinterpret_cast<const float2*>(wi + 8);
          const int jn = h ? tj1 : tj0;       // padded slots: j = i, and their w is zero
          const float4 xj = p.x4[jn >= 0 ? jn : i];
          rel[h][0] = xi.x - xj.x; rel[h][1] = xi.y - xj.y; rel[h][2] = xi.z - xj.z;
        }
      }
      float o[8];
      issue_mma2(o);
      advance(o);
#pragma unroll
      for (int j = 0; j < 16; ++j) gather_next(j);
      float se[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float2 b1 = *reinterpret_cast<const float2*>(s_b1 + 8 * j + 2 * qt);
          acc = fmaf(fmaf(o[4 * j + 2 * h], kInvOut, b1.x), wx[h][j].x, acc);
          acc = fmaf(fmaf(o[4 * j + 2 * h + 1], kInvOut, b1.y), wx[h][j].y, acc);
        }
        se[h] = quad_sum(acc);
      }
      float* s_dx = s_epi + (slot * 2 + wp) * 4;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float a = rows_sum(fmaf(se[1], rel[1][c], se[0] * rel[0][c]));
        if (lane == 0) s_dx[c] = a;
      }
      warpgroup_sync(wg);
      if (live && wp == 0 && lane == 0) {
        const float* s0 = s_epi + slot * 8;
        st4(p.dx + 4 * (size_t)n, make_float4((s0[0] + s0[4]) * (1.f / 16.f), (s0[1] + s0[5]) * (1.f / 16.f), (s0[2] + s0[6]) * (1.f / 16.f), 0.f));
      }
    }
    TC_STAMP(k, 4);
    ti = nti; tj0 = ntj0; tj1 = ntj1;
  };
  for (int k = 0; k + 1 < n_my; ++k) tile(k, std::true_type{});
  if (n_my > 0) tile(n_my - 1, std::false_type{});
  TC_STAMP_CTA(2);
}

// =================================================================================================================
// Hardware self-test of the operand conventions the kernels rely on (B in the canonical K-major no-swizzle layout, A
// through a shared-memory descriptor in the same layout or from registers in the accumulator-compatible fragment layout,
// fp32 accumulator fragment).  D[128 x 128] = A[128 x 32] * B[128 x 32]^T, one warpgroup, two 64-row halves.
// a, b: f16 row-major [128][32]; d: fp32 [128][128].
__global__ void __launch_bounds__(128, 1) wgmma_selftest_kernel(const __half* a, const __half* b, float* d, int a_from_smem) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, qg = lane >> 2, qt = lane & 3;
  constexpr uint32_t SBO = (32 / 8) * 128;        // K = 32: 4 core matrices per 8-row group
  const uint32_t sbase = smem_u32(smem);
  const uint32_t sb_b = sbase, sb_a = sbase + 128 * 32 * 2;
  for (int e = tid; e < 128 * 32; e += 128) {
    const int r = e >> 5, kk = e & 31;
    const uint32_t off = (uint32_t)(r >> 3) * SBO + (uint32_t)(kk >> 3) * 128u + (uint32_t)(r & 7) * 16u + (uint32_t)(kk & 7) * 2u;
    *reinterpret_cast<__half*>(smem + off) = b[e];
    *reinterpret_cast<__half*>(smem + 128 * 32 * 2 + off) = a[e];
  }
  fence_proxy_async();
  __syncthreads();
#pragma unroll 1
  for (int half = 0; half < 2; ++half) {
    const int r0 = 64 * half + 16 * warp + qg;
    float acc[64];
    uint32_t af[2][4];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      af[ks][0] = *reinterpret_cast<const uint32_t*>(a + (size_t)r0 * 32 + 16 * ks + 2 * qt);
      af[ks][1] = *reinterpret_cast<const uint32_t*>(a + (size_t)(r0 + 8) * 32 + 16 * ks + 2 * qt);
      af[ks][2] = *reinterpret_cast<const uint32_t*>(a + (size_t)r0 * 32 + 16 * ks + 8 + 2 * qt);
      af[ks][3] = *reinterpret_cast<const uint32_t*>(a + (size_t)(r0 + 8) * 32 + 16 * ks + 8 + 2 * qt);
    }
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      if (a_from_smem) wgmma_f16_ss(acc, smem_desc(sb_a + (uint32_t)(8 * half) * SBO + 256u * ks, 128, SBO), smem_desc(sb_b + 256u * ks, 128, SBO), ks > 0);
      else wgmma_f16_rs(acc, af[ks], smem_desc(sb_b + 256u * ks, 128, SBO), ks > 0);
    }
    wgmma_commit();
    wgmma_wait0();
    wgmma_settle(acc);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      *reinterpret_cast<float2*>(d + (size_t)r0 * 128 + 8 * j + 2 * qt) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(d + (size_t)(r0 + 8) * 128 + 8 * j + 2 * qt) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
}

int g_tc_sms = 0;
bool g_tc_stage = true;      // CBG_X2H_STAGE=0: the register-gather path in every mode
long long* g_tc_trace = nullptr;
int g_tc_trace_tiles = 0;

// MODE_V always gathers into registers: staging measured slower there on H100 (DESIGN §5.2), faster in MODE_K
template <int MODE>
void launch_tc(int grid, cudaStream_t st, const EdgeArgs& a, const TcWeights& w) {
  if constexpr (MODE != MODE_V) {
    if (g_tc_stage) {
      cbg_launch_pdl(x2h_tc_kernel<MODE, true>, dim3(grid), dim3(256), sm_total(true), st, a, w);
      return;
    }
  }
  cbg_launch_pdl(x2h_tc_kernel<MODE, false>, dim3(grid), dim3(256), sm_total(false), st, a, w);
}

int tc_init() {
  static bool done_dev[CBG_MAX_DEVICES] = {};
  bool& done = cbg_dev_flag(done_dev);
  if (done) return 0;
  int dev = 0;
  CBG_CUDA_OK(cudaGetDevice(&dev));
  CBG_CUDA_OK(cudaDeviceGetAttribute(&g_tc_sms, cudaDevAttrMultiProcessorCount, dev));
  if (const char* e = getenv("CBG_X2H_STAGE")) g_tc_stage = strcmp(e, "0") != 0;
#define TC_ATTR(MODE, STAGE) CBG_CUDA_OK(cudaFuncSetAttribute(x2h_tc_kernel<MODE, STAGE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_total(STAGE)))
  TC_ATTR(MODE_K, true); TC_ATTR(MODE_XV, true);
  TC_ATTR(MODE_K, false); TC_ATTR(MODE_V, false); TC_ATTR(MODE_XV, false);
#undef TC_ATTR
  done = true;
  return 0;
}

}  // namespace

int cbg_launch_x2h_tc(const EdgeArgs& a, cudaStream_t st) {
  if (a.n_nodes <= 0) return 0;
  if (int rc = tc_init()) return rc;
  const int tiles = (a.n_nodes + 3) / 4;
  const int grid = tiles < g_tc_sms ? tiles : g_tc_sms;
  EdgeArgs ak = a;
  ak.w_compact = 0;
  EdgeArgs av = a;
  av.w_compact = 0;
  // debugging hook: one-shot, the next attention-weight launch (max_tiles > 0) or aggregation launch (max_tiles < 0) only
  if (g_tc_trace_tiles >= 0) { ak.trace = g_tc_trace; ak.trace_tiles = g_tc_trace_tiles; }
  else { av.trace = g_tc_trace; av.trace_tiles = -g_tc_trace_tiles; }
  g_tc_trace = nullptr;
  const float* L = a.layer;
  const TcWeights wk{L + kOffKW1, L + kOffKWg, L + kOffKLn, nullptr, L + kOffRbf};
  const TcWeights wv{L + kOffVW1, L + kOffVWg, L + kOffVLn, L + kOffVB1, L + kOffRbf};
  CBG_PROF_BEGIN(CBG_K_X2H_K, st);
  launch_tc<MODE_K>(grid, st, ak, wk);
  CBG_LAUNCHED(CBG_K_X2H_K, st);
  CBG_PROF_BEGIN(CBG_K_X2H_V, st);
  launch_tc<MODE_V>(grid, st, av, wv);
  CBG_LAUNCHED(CBG_K_X2H_V, st);
  return 0;
}

// H2X for the listed (generated) nodes: attention weights with the xk / xq weights into the compact buffer a.w
// ([n_nodes, 32, 16]), then the value head + coordinate update into a.dx ([n_nodes, 4])
int cbg_launch_h2x_tc(const EdgeArgs& a, cudaStream_t st) {
  if (a.n_nodes <= 0) return 0;
  if (int rc = tc_init()) return rc;
  if (a.node_idx == nullptr || a.w == nullptr || a.dx == nullptr) { cbg_set_error("h2x_tc: node list, w and dx buffers are required"); return 1; }
  const int tiles = (a.n_nodes + 3) / 4;
  const int grid = tiles < g_tc_sms ? tiles : g_tc_sms;
  EdgeArgs ax = a;
  ax.w_compact = 1; ax.trace = nullptr; ax.trace_tiles = 0;
  const float* L = a.layer;
  const TcWeights wk{L + kOffXKW1, L + kOffXKWg, L + kOffXKLn, nullptr, L + kOffXRbf};
  const TcWeights wv{L + kOffXVW1, L + kOffXVWg, L + kOffXVLn, L + kOffXVB1, L + kOffXRbf};
  CBG_PROF_BEGIN(CBG_K_H2X, st);
  launch_tc<MODE_K>(grid, st, ax, wk);
  CBG_LAUNCHED(CBG_K_H2X, st);
  CBG_PROF_BEGIN(CBG_K_H2X, st);
  launch_tc<MODE_XV>(grid, st, ax, wv);
  CBG_LAUNCHED(CBG_K_H2X, st);
  return 0;
}

void cbg_x2h_tc_set_trace(long long* buf, int max_tiles) { g_tc_trace = buf; g_tc_trace_tiles = buf ? max_tiles : 0; }

int cbg_launch_umma_selftest(const void* a, const void* b, float* d, int a_from_smem, cudaStream_t st) {
  const int smem_bytes = 2 * 128 * 32 * 2;
  wgmma_selftest_kernel<<<1, 128, smem_bytes, st>>>((const __half*)a, (const __half*)b, d, a_from_smem);
  CBG_CUDA_OK(cudaGetLastError());
  return 0;
}
