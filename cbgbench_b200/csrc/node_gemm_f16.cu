// Node-level projections on the Hopper tensor cores (wgmma) with the f16 (hi, lo) split (three products per K step, fp32
// accumulate in registers): same contract as node_gemm_tc.cu (planes Pj_k, Pj_v, Pi_k, Pi_v, q of one attention
// sub-layer; reference: x2h_attention.py:58-83, h2x_attention.py:42-62, common.py:151-171), half the tensor-core time
// and half the operand bytes of the 3xTF32 version at the same accuracy class (cbg_tc.cuh).
//
// One CTA = one 128-row tile = two consumer warpgroups of 64 rows (wgmma M = 64) + a copy warp.  A (rows of h, each
// scaled by its own power of two) is split once per CTA into hi/lo f16 tiles in shared memory (canonical K-major layout,
// read through wgmma descriptors); the weight planes (scaled by 256) are pre-split and pre-laid-out by the packer in 64-wide K chunks
// (hi | lo = 32 KB) and stream through a 3-stage ring with cp.async.bulk + mbarrier.  Each warpgroup holds the
// 64 x 128 fp32 accumulator of its rows in registers and runs the epilogue from them: a quad of lanes owns 8 consecutive
// columns of a row, so the plane rows go to global memory as full 32-byte sectors with no staging.  LayerNorm + ReLU
// of the q MLP is done in registers (row sums over the quad) and written to a second (hi | lo) A tile for the second
// Linear; only the owning warpgroup reads those rows back, so that hand-over is a warpgroup barrier.
//
// Operand windows.  The split keeps ~2^-22 relative accuracy only while hi stays below the f16 maximum (65504) and lo
// stays a normal f16 (>= 2^-14), so every operand is scaled by a power of two into that window:
//   - W (packer, x256): |W| < 256 is checked when the blob is packed (modules.py raises ValueError above it).
//   - q hidden after LayerNorm + ReLU (x16): bounded by sqrt(127) max|gamma| + max|beta|, checked by the packer.
//   - h (run time, per row): h is data, so no fixed scale fits every input.  Row r is scaled by 2^e_r with
//     max|h_r| 2^e_r in [2^10, 2^11) (e_r clamped to [-126, 118] so that both 2^e_r and 2^(-8 - e_r) are normal fp32,
//     e_r = 0 for a zero row), and the epilogue of the GEMMs that read this tile multiplies by 2^(-8 - e_r).  Both
//     scales are powers of two, so the scaling adds no rounding.  The staging threads r and r + 128 each reduce the
//     max over their half of row r and exchange it through shared memory behind a named barrier of the 256 threads.
#include "cbg_kernels.cuh"
#include "cbg_tc.cuh"

using namespace cbg_tc;

namespace {

constexpr int TM = 128;                        // rows per CTA (2 x wgmma M)
constexpr int KC = 64;                         // K elements per weight chunk
constexpr int NKC = CBG_H / KC;                // 2 chunks per plane
constexpr int STAGES = 3;
constexpr uint32_t A_TILE = TM * CBG_H * 2;                // 32 KB per (hi | lo)
constexpr uint32_t B_CHUNK = 128 * KC * 2;                 // 16 KB per (hi | lo)
constexpr uint32_t B_STAGE = 2 * B_CHUNK;
constexpr uint32_t SM_A_HI = 0;                            // rows of h (hi at +0, lo at +A_TILE)
constexpr uint32_t SM_Q = 2 * A_TILE;                      // relu(LN(q hidden)), same (hi | lo) layout
constexpr uint32_t SM_B0 = 4 * A_TILE;
constexpr uint32_t SM_ROWMAX = SM_B0 + STAGES * B_STAGE;   // [2][128] fp32: max|h| over each half of a row of the tile
constexpr uint32_t SM_BARS = SM_ROWMAX + 2 * TM * 4;
constexpr uint32_t SM_TOTAL = SM_BARS + 64;
static_assert(SM_TOTAL <= 232448, "shared memory budget");
constexpr uint32_t A_SBO = (CBG_H / 8) * 128, B_SBO = (KC / 8) * 128, LBO = 128;
constexpr float kScaleQ = 16.f;                // the LayerNorm'ed q hidden in its A tile (bounded by the packer)
constexpr float kInvAcc = 1.f / 4096.f;        // q tile x16, weights x256 (packer): accumulator at 2^12
constexpr int kBarStage = 3;                   // named barrier of the 256 A-staging threads (1, 2: warpgroup_sync)

// e_r of a row whose max |h| is m: m 2^e_r in [2^10, 2^11), clamped to [-126, 118] (2^e_r and 2^(-8 - e_r) normal
// fp32; this clamp also covers subnormal, inf and NaN maxima), 0 for a zero row
__device__ __forceinline__ int row_exp(float m) {
  if (m == 0.f) return 0;
  const int e = 137 - (int)((__float_as_uint(m) >> 23) & 0xffu);
  return e < -126 ? -126 : (e > 118 ? 118 : e);
}
__device__ __forceinline__ float exp2i(int e) { return __uint_as_float((uint32_t)(e + 127) << 23); }   // normal range only

// byte offset of elements (row, k .. k+7) inside an A tile (k a multiple of 8: one 16-byte core-matrix row)
__device__ __forceinline__ uint32_t a_off8(int row, int k8) {
  return (uint32_t)(row >> 3) * A_SBO + (uint32_t)k8 * 128u + (uint32_t)(row & 7) * 16u;
}
__device__ __forceinline__ void store_split8(uint8_t* tile, int row, int k8, const float4 a, const float4 b, float sc) {
  uint4 hi, lo;
  split_pair(a.x * sc, a.y * sc, hi.x, lo.x);
  split_pair(a.z * sc, a.w * sc, hi.y, lo.y);
  split_pair(b.x * sc, b.y * sc, hi.z, lo.z);
  split_pair(b.z * sc, b.w * sc, hi.w, lo.w);
  const uint32_t off = a_off8(row, k8);
  *reinterpret_cast<uint4*>(tile + off) = hi;
  *reinterpret_cast<uint4*>(tile + A_TILE + off) = lo;
}

// The GEMMs of one CTA, in issue order.  With the q MLP the hidden plane goes FIRST and its second Linear LAST, so the
// LayerNorm epilogue (the only serial dependency) hides behind the other planes.  kind: 0 plane -> global, 1 q hidden
// (-> LN -> ReLU -> A tile of the second Linear), 2 q second Linear.
struct Sched {
  int n_gemm, n_norm, has_q;
  __device__ __forceinline__ Sched(const NodeGemmArgs& p, bool cta_dst) {
    has_q = (p.has_q && cta_dst) ? 1 : 0;
    if (cta_dst) n_norm = p.n_planes - (p.has_q ? 1 : 0);
    else { n_norm = CBG_NODE_SRC_PLANES - p.tc_first_plane; n_norm = n_norm < 0 ? 0 : (n_norm > p.n_planes ? p.n_planes : n_norm); }
    n_gemm = n_norm + 2 * has_q;
  }
  __device__ __forceinline__ int kind(int g) const { return has_q ? (g == 0 ? 1 : (g == n_gemm - 1 ? 2 : 0)) : 0; }
  // plane relative to the launch's first plane (bias / out index); q second Linear: -1
  // The plain planes are visited in an order rotated by the CTA index: every CTA streams the same weight images from L2,
  // and without the rotation all of them pull the same lines at the same moment.
  __device__ __forceinline__ int rel(const NodeGemmArgs& p, int g) const {
    if (has_q && g == 0) return p.n_planes - 1;
    if (has_q && g == n_gemm - 1) return -1;
    const int idx = has_q ? g - 1 : g;
    return n_norm > 1 ? (idx + (int)(blockIdx.x % (unsigned)n_norm)) % n_norm : idx;
  }
};
// weight image of GEMM g: NKC chunks x (hi | lo) x [128 n][64 k] f16; image 5 = q second Linear
__device__ __forceinline__ const float* chunk_src(const NodeGemmArgs& p, const Sched& sc, int i) {
  const int g = i / NKC, c = i % NKC;
  const int r = sc.rel(p, g);
  const int plane = r < 0 ? 5 : p.tc_first_plane + r;
  return p.tch_planes + (size_t)plane * (NKC * B_STAGE / 4) + (size_t)c * (B_STAGE / 4);
}

__device__ __forceinline__ void stamp(long long* trace, int slot) {
  if (trace && blockIdx.x == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    trace[slot] = (long long)t;
  }
}

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(CBG_FULL, v, 1);
  return v + __shfl_xor_sync(CBG_FULL, v, 2);
}

__global__ void __launch_bounds__(288, 1) node_gemm_f16_kernel(const __grid_constant__ NodeGemmArgs p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  int n_rows = p.n_rows;
  if (p.n_rows_dev) { const int nd = *p.n_rows_dev; n_rows = nd < n_rows ? nd : n_rows; }
  // merged launch: planes >= CBG_NODE_SRC_PLANES (destination planes, q) only for the first n_dst rows of the list
  int n_dst = n_rows;
  if (p.n_dst_dev) { const int nd = *p.n_dst_dev; n_dst = nd < n_dst ? nd : n_dst; }
  const int row0 = blockIdx.x * TM;
  if (row0 >= n_rows) return;
  const Sched sc(p, row0 < n_dst);
  if (sc.n_gemm == 0) return;
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar_full = sbase + SM_BARS;                  // [STAGES]
  const uint32_t bar_empty = bar_full + 8 * STAGES;           // [STAGES]: one arrival per consumer warpgroup
  const int total_chunks = sc.n_gemm * NKC;
  if (tid == 0) stamp(p.trace, 0);

  if (tid == 256) {
    // barriers + the first weight chunks: nothing here depends on the A tile, so the copies fly during its staging
    for (int s = 0; s < STAGES; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 2); }
    fence_mbar_init();
    for (int i = 0; i < STAGES && i < total_chunks; ++i) {
      mbar_expect_tx(bar_full + 8 * i, B_STAGE);
      bulk_g2s(sbase + SM_B0 + i * B_STAGE, chunk_src(p, sc, i), B_STAGE, bar_full + 8 * i);
    }
  }
  if (warp < 8) {
    // A tile: rows of h -> (hi, lo) f16 tiles; lane <-> row keeps the 16-byte shared stores conflict free
    const int r = tid & (TM - 1);
    const int row = row0 + r;
    const bool live = row < n_rows;
    const float* arow = p.a + (size_t)(live ? (p.row_idx ? p.row_idx[row] : row) : 0) * CBG_H;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 v[16];                                  // thread handles k8 = (tid >> 7) + 2 * j, j < 8: all 16 loads in flight
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k8 = (tid >> 7) + 2 * j;
      v[2 * j] = live ? ldg4(arow + 8 * k8) : z;
      v[2 * j + 1] = live ? ldg4(arow + 8 * k8 + 4) : z;
    }
    // per-row scale: max |h| over this thread's half of the row, combined with the other half's through shared memory
    float m = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) m = fmaxf(m, fmaxf(fmaxf(fabsf(v[j].x), fabsf(v[j].y)), fmaxf(fabsf(v[j].z), fabsf(v[j].w))));
    float* rowmax = reinterpret_cast<float*>(smem + SM_ROWMAX);
    rowmax[tid] = m;
    asm volatile("bar.sync %0, 256;" ::"r"(kBarStage) : "memory");
    const float sc = exp2i(row_exp(fmaxf(rowmax[r], rowmax[r + TM])));
#pragma unroll
    for (int j = 0; j < 8; ++j) store_split8(smem + SM_A_HI, r, (tid >> 7) + 2 * j, v[2 * j], v[2 * j + 1], sc);
    fence_proxy_async();
  }
  __syncthreads();
  if (tid == 0) stamp(p.trace, 1);

  if (warp == 8) {
    // ===== weight-chunk producer (chunks 0 .. STAGES-1 are already in flight) =====
    if (lane == 0) {
      for (int i = STAGES; i < total_chunks; ++i) {
        const int s = i % STAGES;
        mbar_wait(bar_empty + 8 * s, (uint32_t)(((i / STAGES) - 1) & 1));
        mbar_expect_tx(bar_full + 8 * s, B_STAGE);
        bulk_g2s(sbase + SM_B0 + s * B_STAGE, chunk_src(p, sc, i), B_STAGE, bar_full + 8 * s);
      }
    }
    return;
  }
  // ===== consumer warpgroups: MMAs and epilogue of rows 64 wg .. 64 wg + 63 =====
  const int wg = warp >> 2, qg = lane >> 2, qt = lane & 3;
  const int r_lo = 64 * wg + 16 * (warp & 3) + qg;            // this thread's accumulator rows: r_lo and r_lo + 8
  int node[2];
  float inv_acc_h[2];                                           // 2^(-8 - e_r): accumulators of the GEMMs that read h
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int grow = row0 + r_lo + 8 * h;
    node[h] = (grow < n_rows) ? (p.row_idx ? p.row_idx[grow] : grow) : -1;
    const float* rowmax = reinterpret_cast<const float*>(smem + SM_ROWMAX);
    inv_acc_h[h] = exp2i(-8 - row_exp(fmaxf(rowmax[r_lo + 8 * h], rowmax[r_lo + 8 * h + TM])));
  }
  for (int g = 0; g < sc.n_gemm; ++g) {
    const int kind = sc.kind(g), rel = sc.rel(p, g);
    const uint32_t a_base = sbase + (kind == 2 ? SM_Q : SM_A_HI) + (uint32_t)(8 * wg) * A_SBO;
    const uint64_t da_hi = smem_desc(a_base, LBO, A_SBO), da_lo = smem_desc(a_base + A_TILE, LBO, A_SBO);
    float d[64];
#pragma unroll
    for (int c = 0; c < NKC; ++c) {
      const int i = g * NKC + c, s = i % STAGES;
      mbar_wait(bar_full + 8 * s, (uint32_t)((i / STAGES) & 1));
      const uint64_t db_hi = smem_desc(sbase + SM_B0 + s * B_STAGE, LBO, B_SBO);
      const uint64_t db_lo = smem_desc(sbase + SM_B0 + s * B_STAGE + B_CHUNK, LBO, B_SBO);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < KC / 16; ++ks) {
        const uint64_t ka = (uint64_t)(16 * (c * (KC / 16) + ks)), kb = (uint64_t)(16 * ks);   // 256 bytes per K step
        wgmma_f16_ss(d, da_lo + ka, db_hi + kb, (c == 0 && ks == 0) ? 0u : 1u);                // small terms first
        wgmma_f16_ss(d, da_hi + ka, db_lo + kb, 1u);
        wgmma_f16_ss(d, da_hi + ka, db_hi + kb, 1u);
      }
      wgmma_commit();
      wgmma_wait0();
      if ((tid & 127) == 0) mbar_arrive(bar_empty + 8 * s);      // this warpgroup is done with the ring stage
    }
    wgmma_settle(d);
    if (tid == 0) stamp(p.trace, 2 + g);
    if (kind != 1) {
      const float* bias = kind == 2 ? p.q_b1 : p.bias + rel * CBG_H;
      float* out = kind == 2 ? p.out_q : p.out[rel];
      // destination planes / q of a merged launch stop at n_dst
      const bool dst_plane = kind == 2 || p.tc_first_plane + rel >= CBG_NODE_SRC_PLANES;
      const int row_lim = dst_plane ? n_dst : n_rows;      // rows of this tile that exist for this plane
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (node[h] < 0 || row0 + r_lo + 8 * h >= row_lim) continue;
        float* o = out + (size_t)node[h] * CBG_H + 2 * qt;
        const float inv = kind == 2 ? kInvAcc : inv_acc_h[h];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float2 b = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + 2 * qt));
          *reinterpret_cast<float2*>(o + 8 * j) = make_float2(fmaf(d[4 * j + 2 * h], inv, b.x), fmaf(d[4 * j + 2 * h + 1], inv, b.y));
        }
      }
    } else {
      // q hidden: + bias, LayerNorm over the row (a row's 128 columns live in the 4 lanes of a quad; mean first, then
      // the squared deviations), ReLU, (hi, lo) split into the A tile of the second Linear
      const float* bias = p.bias + rel * CBG_H;
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + 2 * qt));
        d[4 * j] = fmaf(d[4 * j], inv_acc_h[0], b.x);
        d[4 * j + 1] = fmaf(d[4 * j + 1], inv_acc_h[0], b.y);
        d[4 * j + 2] = fmaf(d[4 * j + 2], inv_acc_h[1], b.x);
        d[4 * j + 3] = fmaf(d[4 * j + 3], inv_acc_h[1], b.y);
        s0 += d[4 * j] + d[4 * j + 1];
        s1 += d[4 * j + 2] + d[4 * j + 3];
      }
      const float mean0 = quad_sum(s0) * (1.f / 128.f), mean1 = quad_sum(s1) * (1.f / 128.f);
      float q0 = 0.f, q1 = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        d[4 * j] -= mean0; d[4 * j + 1] -= mean0; d[4 * j + 2] -= mean1; d[4 * j + 3] -= mean1;
        q0 = fmaf(d[4 * j], d[4 * j], q0); q0 = fmaf(d[4 * j + 1], d[4 * j + 1], q0);
        q1 = fmaf(d[4 * j + 2], d[4 * j + 2], q1); q1 = fmaf(d[4 * j + 3], d[4 * j + 3], q1);
      }
      const float rstd0 = 1.f / sqrtf(quad_sum(q0) * (1.f / 128.f) + 1e-5f);
      const float rstd1 = 1.f / sqrtf(quad_sum(q1) * (1.f / 128.f) + 1e-5f);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 gm = __ldg(reinterpret_cast<const float2*>(p.q_ln + 8 * j + 2 * qt));
        const float2 bt = __ldg(reinterpret_cast<const float2*>(p.q_ln + 128 + 8 * j + 2 * qt));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float rs = h ? rstd1 : rstd0;
          const float a0 = fmaxf(fmaf(d[4 * j + 2 * h] * rs, gm.x, bt.x), 0.f);
          const float a1 = fmaxf(fmaf(d[4 * j + 2 * h + 1] * rs, gm.y, bt.y), 0.f);
          uint32_t hi, lo;
          split_pair(a0 * kScaleQ, a1 * kScaleQ, hi, lo);
          const uint32_t off = a_off8(r_lo + 8 * h, j) + 4u * (uint32_t)qt;
          *reinterpret_cast<uint32_t*>(smem + SM_Q + off) = hi;
          *reinterpret_cast<uint32_t*>(smem + SM_Q + A_TILE + off) = lo;
        }
      }
      fence_proxy_async();
      warpgroup_sync(wg);      // the second Linear of this warpgroup reads exactly the rows it has just written
    }
    if (tid == 0) stamp(p.trace, 10 + g);
  }
  if (tid == 0) stamp(p.trace, 20);
}

}  // namespace

static long long* g_trace_buf = nullptr;
void cbg_node_gemm_f16_set_trace(long long* buf_dev) { g_trace_buf = buf_dev; }

int cbg_launch_node_gemm_f16(const NodeGemmArgs& a, cudaStream_t st) {
  if (a.n_rows <= 0) return 0;
  if (!a.tch_planes) { cbg_set_error("f16 tensor-core node GEMM needs the f16 weight images (tch_planes)"); return 1; }
  static bool attr_dev[CBG_MAX_DEVICES] = {};
  bool& attr_set = cbg_dev_flag(attr_dev);
  if (!attr_set) {
    CBG_CUDA_OK(cudaFuncSetAttribute(node_gemm_f16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SM_TOTAL));
    attr_set = true;
  }
  NodeGemmArgs args = a;
  args.trace = g_trace_buf;
  CBG_PROF_BEGIN(CBG_K_NODE_GEMM, st);
  node_gemm_f16_kernel<<<(a.n_rows + TM - 1) / TM, 288, SM_TOTAL, st>>>(args);
  CBG_LAUNCHED(CBG_K_NODE_GEMM, st);
  return 0;
}
