// Node-level projections on the Hopper tensor cores (wgmma, sm_90a) in 3xTF32.
//
// Same contract as node_gemm.cu (planes Pj_k, Pj_v, Pi_k, Pi_v, q of one attention sub-layer;
// reference: x2h_attention.py:58-83, h2x_attention.py:42-62, common.py:151-171), but the
// [rows,128] x [128,128] products run as wgmma m64n128k8 tf32 with the 3xTF32 error-compensated
// split  a*b ~= a_hi*b_hi + a_hi*b_lo + a_lo*b_hi  (a_hi = rna_tf32(a), a_lo = rna_tf32(a - a_hi)),
// fp32 accumulation in registers => fp32-class accuracy (needed for the 1e-4 parity bar; single-pass
// TF32 is ~1e-3 after 9 residual layers, SURVEY.md section 7 hard part 1).
//
// One CTA = one 128-row tile = two consumer warpgroups of 64 rows + a copy warp.  A (rows of h) is converted once
// per CTA into hi/lo tf32 tiles in shared memory in the canonical K-major no-swizzle layout (8 x 16 B core matrices);
// B (the weight plane) is pre-split and pre-laid-out on the host (packer) so a plain 1-D bulk
// async copy (cp.async.bulk + mbarrier complete_tx) stages each 32 KB K-chunk into a 3-stage ring,
// optionally multicast across a thread-block cluster of CL row tiles: every CTA copies 1/CL of a chunk into all CL
// shared memories, and a ring stage is refilled once the consumers of all CL CTAs have released it.
// Each warpgroup keeps the 64 x 128 fp32 accumulator in registers for the epilogue (+bias -> global, or
// LayerNorm+ReLU -> A tiles for the second Linear of the q MLP).
#include "cbg_kernels.cuh"
#include "cbg_tc.cuh"

using namespace cbg_tc;

namespace {

constexpr int TM = 128;                        // rows per CTA (2 x wgmma M)
constexpr int KC = 32;                         // K elements per weight chunk
constexpr int NKC = CBG_H / KC;                // 4 chunks per plane
constexpr int NSTAGE = 3;                      // weight-chunk ring depth
constexpr uint32_t A_TILE_BYTES = TM * CBG_H * 4;          // 64 KB per (hi | lo)
constexpr uint32_t B_CHUNK_BYTES = 128 * KC * 4;           // 16 KB per (hi | lo)
constexpr uint32_t B_STAGE_BYTES = 2 * B_CHUNK_BYTES;      // hi + lo, contiguous in the blob
constexpr uint32_t SMEM_A_HI = 0;
constexpr uint32_t SMEM_A_LO = A_TILE_BYTES;
constexpr uint32_t SMEM_B0 = 2 * A_TILE_BYTES;
constexpr uint32_t SMEM_BAR = SMEM_B0 + NSTAGE * B_STAGE_BYTES;
constexpr uint32_t SMEM_TOTAL = SMEM_BAR + 64;
static_assert(SMEM_TOTAL <= 232448, "shared memory budget");
constexpr uint32_t A_SBO = (CBG_H / 4) * 128;   // byte stride between 8-row groups of an A tile
constexpr uint32_t B_SBO = (KC / 4) * 128;      // same for a B chunk
constexpr uint32_t LBO = 128;                   // byte stride between core matrices along K

__device__ __forceinline__ float to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
// byte offset of element (row, k) inside an A tile (canonical K-major, no swizzle)
__device__ __forceinline__ uint32_t a_off(int row, int k) {
  return (uint32_t)(row >> 3) * A_SBO + (uint32_t)(k >> 2) * 128u + (uint32_t)(row & 7) * 16u + (uint32_t)(k & 3) * 4u;
}
__device__ __forceinline__ void store_split(uint8_t* smem, int row, int k4, float4 v) {
  float4 hi = make_float4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w));
  float4 lo = make_float4(to_tf32(v.x - hi.x), to_tf32(v.y - hi.y), to_tf32(v.z - hi.z), to_tf32(v.w - hi.w));
  const uint32_t off = a_off(row, 4 * k4);
  *reinterpret_cast<float4*>(smem + SMEM_A_HI + off) = hi;
  *reinterpret_cast<float4*>(smem + SMEM_A_LO + off) = lo;
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(CBG_FULL, v, 1);
  return v + __shfl_xor_sync(CBG_FULL, v, 2);
}

// weight chunk i lives at: plane(i / NKC) -> tc plane index, chunk (i % NKC)
__device__ __forceinline__ const float* chunk_src_ptr(const NodeGemmArgs& p, int i) {
  const int g = i / NKC, c = i % NKC;
  const int plane = (g < p.n_planes) ? (p.tc_first_plane + g) : 5;       // plane 5 = q second Linear
  return p.tc_planes + (size_t)plane * (NKC * 2 * 128 * KC) + (size_t)c * (2 * 128 * KC);
}

// CL = CTAs per cluster sharing every weight chunk through multicast bulk copies (1 = no cluster).
// Every CTA needs all 6 x 128 KB of weight images, so a cluster of CL row tiles cuts the L2 -> SM weight traffic by CL.
template <int CL>
__global__ void __launch_bounds__(288, 1) node_gemm_tc_kernel(NodeGemmArgs p) {
  constexpr uint16_t kMask = (uint16_t)((1u << CL) - 1u);
  const uint32_t crank = (CL > 1) ? cluster_rank() : 0u;
  if (p.n_rows_dev) {                 // list length lives on the device (receptive-field pruning)
    const int nd = *p.n_rows_dev;
    p.n_rows = nd < p.n_rows ? nd : p.n_rows;
  }
  if ((int)(blockIdx.x / CL) * CL * TM >= p.n_rows) return;   // whole cluster beyond the list: nothing to do
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int row0 = blockIdx.x * TM;
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar_full = sbase + SMEM_BAR;                 // [NSTAGE]
  const uint32_t bar_empty = bar_full + 8 * NSTAGE;           // [NSTAGE]: one arrival per consumer warpgroup of every CTA

  if (tid == 256) {
    for (int s = 0; s < NSTAGE; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 2 * CL); }
    fence_mbar_init();
  }
  if (warp < 8) {
    // A tile: rows of h -> (hi, lo) tf32 tiles; lanes <-> rows keeps the 16 B shared stores conflict free
    const int r = tid & (TM - 1);
    const int row = row0 + r;
    const bool live = row < p.n_rows;
    const float* arow = p.a + (size_t)(live ? (p.row_idx ? p.row_idx[row] : row) : 0) * CBG_H;
#pragma unroll
    for (int it = 0; it < 16; it += 8) {          // thread handles k4 = (tid>>7) + 2*j, j < 16
      float4 v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        v[j] = live ? ldg4(arow + 4 * ((tid >> 7) + 2 * (it + j))) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int j = 0; j < 8; ++j) store_split(smem, r, (tid >> 7) + 2 * (it + j), v[j]);
    }
    fence_proxy_async();
  }
  __syncthreads();
  if (CL > 1) cluster_sync_all();      // every CTA's barriers exist before any peer copy / arrive targets them

  const int n_gemm = p.n_planes + (p.has_q ? 1 : 0);      // + the second Linear of the q MLP
  const int total_chunks = n_gemm * NKC;

  if (warp == 8) {
    // ===== weight-chunk producer: own slice only when clustered =====
    if (lane == 0) {
      for (int i = 0; i < total_chunks; ++i) {
        const int s = i % NSTAGE;
        if (i >= NSTAGE) mbar_wait(bar_empty + 8 * s, (uint32_t)(((i / NSTAGE) - 1) & 1));   // all CL CTAs released the stage
        const uint32_t bf = bar_full + 8 * s;
        mbar_expect_tx(bf, B_STAGE_BYTES);                       // the whole chunk lands here (all slices)
        if (CL > 1) {
          constexpr uint32_t slice = B_STAGE_BYTES / CL;
          bulk_g2s_mcast(sbase + SMEM_B0 + s * B_STAGE_BYTES + crank * slice,
                         reinterpret_cast<const char*>(chunk_src_ptr(p, i)) + crank * slice, slice, bf, kMask);
        } else {
          bulk_g2s(sbase + SMEM_B0 + s * B_STAGE_BYTES, chunk_src_ptr(p, i), B_STAGE_BYTES, bf);
        }
      }
    }
  } else {
    // ===== consumer warpgroups: MMAs and epilogue of rows 64 wg .. 64 wg + 63 =====
    const int wg = warp >> 2, qg = lane >> 2, qt = lane & 3;
    const int r_lo = 64 * wg + 16 * (warp & 3) + qg;          // this thread's accumulator rows: r_lo and r_lo + 8
    int dst[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int grow = row0 + r_lo + 8 * h;
      dst[h] = (grow < p.n_rows) ? (p.row_idx ? p.row_idx[grow] : grow) : -1;
    }
    const uint32_t a_base = sbase + (uint32_t)(8 * wg) * A_SBO;
    const uint64_t da_hi = smem_desc(a_base + SMEM_A_HI, LBO, A_SBO), da_lo = smem_desc(a_base + SMEM_A_LO, LBO, A_SBO);
    for (int g = 0; g < n_gemm; ++g) {
      float d[64];
#pragma unroll
      for (int c = 0; c < NKC; ++c) {
        const int i = g * NKC + c, s = i % NSTAGE;
        mbar_wait(bar_full + 8 * s, (uint32_t)((i / NSTAGE) & 1));
        const uint64_t db_hi = smem_desc(sbase + SMEM_B0 + s * B_STAGE_BYTES, LBO, B_SBO);
        const uint64_t db_lo = smem_desc(sbase + SMEM_B0 + s * B_STAGE_BYTES + B_CHUNK_BYTES, LBO, B_SBO);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < KC / 8; ++ks) {
          const uint64_t ka = (uint64_t)(16 * (c * (KC / 8) + ks)), kb = (uint64_t)(16 * ks);   // 2 core matrices = 256 bytes per K = 8 step
          wgmma_tf32_ss(d, da_lo + ka, db_hi + kb, (c == 0 && ks == 0) ? 0u : 1u);              // small terms first
          wgmma_tf32_ss(d, da_hi + ka, db_lo + kb, 1u);
          wgmma_tf32_ss(d, da_hi + ka, db_hi + kb, 1u);
        }
        wgmma_commit();
        wgmma_wait0();
        if ((tid & 127) == 0) {        // this warpgroup is done with the ring stage: tell the producer of every CTA
          if (CL > 1) { for (uint32_t r = 0; r < (uint32_t)CL; ++r) mbar_arrive_cluster(bar_empty + 8 * s, r); }
          else mbar_arrive(bar_empty + 8 * s);
        }
      }
      wgmma_settle(d);
      const bool is_qhid = p.has_q && (g == p.n_planes - 1);
      const bool is_q2 = p.has_q && (g == p.n_planes);
      if (!is_qhid) {
        const float* bias = is_q2 ? p.q_b1 : (p.bias + g * CBG_H);
        float* out = is_q2 ? p.out_q : p.out[g];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (dst[h] < 0) continue;
          float* o = out + (size_t)dst[h] * CBG_H + 2 * qt;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const float2 b = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + 2 * qt));
            *reinterpret_cast<float2*>(o + 8 * j) = make_float2(d[4 * j + 2 * h] + b.x, d[4 * j + 2 * h + 1] + b.y);
          }
        }
      } else {
        // q hidden: + bias, LayerNorm(128) + ReLU per row (a row's columns live in the 4 lanes of a quad), then back
        // into this warpgroup's rows of the A tiles as the operand of the second Linear
        const float* bias = p.bias + g * CBG_H;
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float2 b = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + 2 * qt));
          d[4 * j] += b.x; d[4 * j + 1] += b.y; d[4 * j + 2] += b.x; d[4 * j + 3] += b.y;
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
          const float2 ga = __ldg(reinterpret_cast<const float2*>(p.q_ln + 8 * j + 2 * qt));
          const float2 be = __ldg(reinterpret_cast<const float2*>(p.q_ln + 128 + 8 * j + 2 * qt));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float rs = h ? rstd1 : rstd0;
            const float a0 = fmaxf(fmaf(d[4 * j + 2 * h] * rs, ga.x, be.x), 0.f);
            const float a1 = fmaxf(fmaf(d[4 * j + 2 * h + 1] * rs, ga.y, be.y), 0.f);
            const float h0 = to_tf32(a0), h1 = to_tf32(a1);
            const uint32_t off = a_off(r_lo + 8 * h, 8 * j + 2 * qt);
            *reinterpret_cast<float2*>(smem + SMEM_A_HI + off) = make_float2(h0, h1);
            *reinterpret_cast<float2*>(smem + SMEM_A_LO + off) = make_float2(to_tf32(a0 - h0), to_tf32(a1 - h1));
          }
        }
        fence_proxy_async();
        warpgroup_sync(wg);      // the second Linear of this warpgroup reads exactly the rows it has just rewritten
      }
    }
  }
  if (CL > 1) cluster_sync_all();      // no CTA may exit while peers can still write its smem / signal its barriers
}

template <int CL>
int launch_tc(const NodeGemmArgs& a, cudaStream_t st) {
  static bool attr_dev[CBG_MAX_DEVICES] = {};
  bool& attr_set = cbg_dev_flag(attr_dev);
  if (!attr_set) {
    CBG_CUDA_OK(cudaFuncSetAttribute(node_gemm_tc_kernel<CL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_TOTAL));
    attr_set = true;
  }
  const int tiles = (a.n_rows + TM - 1) / TM;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)((tiles + CL - 1) / CL * CL));   // padded tiles run the protocol with zero rows
  cfg.blockDim = dim3(288);
  cfg.dynamicSmemBytes = SMEM_TOTAL;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = (CL > 1) ? 1 : 0;
  CBG_PROF_BEGIN(CBG_K_NODE_GEMM, st);
  CBG_CUDA_OK(cudaLaunchKernelEx(&cfg, node_gemm_tc_kernel<CL>, a));
  CBG_LAUNCHED(CBG_K_NODE_GEMM, st);
  return 0;
}

}  // namespace

int cbg_launch_node_gemm_tc(const NodeGemmArgs& a, cudaStream_t st, int cluster) {
  if (a.n_rows <= 0) return 0;
  if (!a.tc_planes) { cbg_set_error("tensor-core node GEMM needs the pre-split weight planes"); return 1; }
  // the merged source/destination launch (n_dst_dev) is an f16-kernel feature: run_denoiser gives this kernel two launches
  if (a.n_dst_dev) { cbg_set_error("3xTF32 node GEMM: n_dst_dev is not supported"); return 1; }
  static int cl_env = -1;
  if (cl_env < 0) {
    const char* e = getenv("CBG_GEMM_CLUSTER");
    cl_env = e ? atoi(e) : 1;
    if (cl_env != 1 && cl_env != 2 && cl_env != 4) cl_env = 1;
  }
  switch ((cluster == 1 || cluster == 2 || cluster == 4) ? cluster : cl_env) {
    case 2: return launch_tc<2>(a, st);
    case 4: return launch_tc<4>(a, st);
    default: return launch_tc<1>(a, st);
  }
}
