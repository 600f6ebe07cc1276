// Node-level projections of one attention sub-layer (fp32 SIMT tile GEMM, K = 128).
//
// "Note D" split of the reference's 340-wide first edge Linear (SURVEY.md section 8a):
//   W0 . [type | rfeat | h_i | h_j] = c[type] + Wrf[type] g(d) + (W_i h)_i + (W_j h)_j
// so the h-dependent part is computed ONCE PER NODE here instead of once per edge:
//   planes Pj_k, Pj_v = h W_j^T ; Pi_k, Pi_v = h W_i^T + b0 ; q = MLP_q(h) / sqrt(8)
// Reference: repo/modules/attention/x2h_attention.py:58-83, h2x_attention.py:42-62,
//            repo/modules/common.py:151-171 (MLP = Linear -> LayerNorm -> ReLU -> Linear).
#include "cbg_kernels.cuh"

namespace {

constexpr int BM = 64;                               // rows per CTA
constexpr int kSmemFloats = 128 * BM + 128 * 128;    // A tile (k-major) + W tile
constexpr int kSmemBytes = kSmemFloats * 4;          // 96 KB

// acc[r][c]: rows ty*4+r ; cols c<4 -> tx*4+c , c>=4 -> 64+tx*4+(c-4)
__device__ __forceinline__ void tile_mma(const float* __restrict__ As, const float* __restrict__ Ws,
                                         int tx, int ty, float (&acc)[4][8]) {
#pragma unroll 8
  for (int k = 0; k < 128; ++k) {
    const float4 a = ld4(As + k * BM + ty * 4);
    const float4 b0 = ld4(Ws + k * 128 + tx * 4);
    const float4 b1 = ld4(Ws + k * 128 + 64 + tx * 4);
    const float av[4] = {a.x, a.y, a.z, a.w};
    const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[r][c] = fmaf(av[r], bv[c], acc[r][c]);
  }
}

__global__ void __launch_bounds__(256, 2) node_gemm_kernel(NodeGemmArgs p) {
  extern __shared__ __align__(16) float smem[];
  float* As = smem;              // [128][BM]
  float* Ws = smem + 128 * BM;   // [128][128]
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int row0 = blockIdx.x * BM;
  if (p.n_rows_dev) {
    const int nd = *p.n_rows_dev;
    p.n_rows = nd < p.n_rows ? nd : p.n_rows;
  }
  if (row0 >= p.n_rows) return;

  // A tile, transposed to k-major; lanes <-> rows so the shared stores are conflict-free
  for (int idx = tid; idx < BM * 32; idx += 256) {
    const int r = idx % BM, kq = idx / BM;
    const int row = row0 + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row < p.n_rows) {
      const int src = p.row_idx ? p.row_idx[row] : row;
      v = ldg4(p.a + (size_t)src * 128 + kq * 4);
    }
    As[(kq * 4 + 0) * BM + r] = v.x;
    As[(kq * 4 + 1) * BM + r] = v.y;
    As[(kq * 4 + 2) * BM + r] = v.z;
    As[(kq * 4 + 3) * BM + r] = v.w;
  }
  // destination node ids of this thread's 4 rows
  int dst[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int row = row0 + ty * 4 + r;
    dst[r] = (row < p.n_rows) ? (p.row_idx ? p.row_idx[row] : row) : -1;
  }

  float acc[4][8];
  for (int plane = 0; plane < p.n_planes; ++plane) {
    __syncthreads();   // previous plane's readers of Ws are done (and As is complete on plane 0)
    for (int idx = tid; idx < 128 * 32; idx += 256) {
      const int k = idx >> 5, c4 = idx & 31;
      st4(Ws + k * 128 + c4 * 4, ldg4(p.wt + (size_t)k * p.ldw + plane * 128 + c4 * 4));
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[r][c] = 0.f;
    tile_mma(As, Ws, tx, ty, acc);
    const float4 bl = ldg4(p.bias + plane * 128 + tx * 4);
    const float4 bh = ldg4(p.bias + plane * 128 + 64 + tx * 4);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      acc[r][0] += bl.x; acc[r][1] += bl.y; acc[r][2] += bl.z; acc[r][3] += bl.w;
      acc[r][4] += bh.x; acc[r][5] += bh.y; acc[r][6] += bh.z; acc[r][7] += bh.w;
    }
    if (p.has_q && plane == p.n_planes - 1) break;   // q_hidden stays in registers
    float* out = p.out[plane];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      if (dst[r] < 0) continue;
      float* o = out + (size_t)dst[r] * 128;
      st4(o + tx * 4, make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]));
      st4(o + 64 + tx * 4, make_float4(acc[r][4], acc[r][5], acc[r][6], acc[r][7]));
    }
  }
  if (!p.has_q) return;

  // q = W1 . relu(LN(q_hidden)) + b1   (weights pre-scaled by 1/sqrt(head_dim))
  __syncthreads();   // everyone is done reading As / Ws
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int col = (c < 4) ? (tx * 4 + c) : (64 + tx * 4 + (c - 4));
    st4(As + col * BM + ty * 4, make_float4(acc[0][c], acc[1][c], acc[2][c], acc[3][c]));
  }
  for (int idx = tid; idx < 128 * 32; idx += 256) {
    const int k = idx >> 5, c4 = idx & 31;
    st4(Ws + k * 128 + c4 * 4, ldg4(p.q_w1t + (size_t)k * 128 + c4 * 4));
  }
  __syncthreads();
  {
    const int warp = tid >> 5, lane = tid & 31;
    float ga[4], be[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) { ga[c] = __ldg(p.q_ln + lane + 32 * c); be[c] = __ldg(p.q_ln + 128 + lane + 32 * c); }
    for (int r = warp * 8; r < warp * 8 + 8; ++r) {
      float v[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) v[c] = As[(lane + 32 * c) * BM + r];
      const float mean = warp_sum((v[0] + v[1]) + (v[2] + v[3])) * (1.f / 128.f);
#pragma unroll
      for (int c = 0; c < 4; ++c) v[c] -= mean;
      const float var = warp_sum((v[0] * v[0] + v[1] * v[1]) + (v[2] * v[2] + v[3] * v[3])) * (1.f / 128.f);
      const float rstd = 1.f / sqrtf(var + 1e-5f);
#pragma unroll
      for (int c = 0; c < 4; ++c) As[(lane + 32 * c) * BM + r] = fmaxf(fmaf(v[c] * rstd, ga[c], be[c]), 0.f);
    }
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[r][c] = 0.f;
  tile_mma(As, Ws, tx, ty, acc);
  const float4 bl = ldg4(p.q_b1 + tx * 4);
  const float4 bh = ldg4(p.q_b1 + 64 + tx * 4);
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    if (dst[r] < 0) continue;
    float* o = p.out_q + (size_t)dst[r] * 128;
    st4(o + tx * 4, make_float4(acc[r][0] + bl.x, acc[r][1] + bl.y, acc[r][2] + bl.z, acc[r][3] + bl.w));
    st4(o + 64 + tx * 4, make_float4(acc[r][4] + bh.x, acc[r][5] + bh.y, acc[r][6] + bh.z, acc[r][7] + bh.w));
  }
}

}  // namespace

int cbg_launch_node_gemm(const NodeGemmArgs& a, cudaStream_t st) {
  if (a.n_rows <= 0) return 0;
  // the merged source/destination launch (n_dst_dev) is an f16-kernel feature: run_denoiser gives this kernel two launches
  if (a.n_dst_dev) { cbg_set_error("fp32 SIMT node GEMM: n_dst_dev is not supported"); return 1; }
  static bool attr_dev[CBG_MAX_DEVICES] = {};
  bool& attr_set = cbg_dev_flag(attr_dev);
  if (!attr_set) {
    CBG_CUDA_OK(cudaFuncSetAttribute(node_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    attr_set = true;
  }
  CBG_PROF_BEGIN(CBG_K_NODE_GEMM, st);
  node_gemm_kernel<<<(a.n_rows + BM - 1) / BM, 256, kSmemBytes, st>>>(a);
  CBG_LAUNCHED(CBG_K_NODE_GEMM, st);
  return 0;
}
