// Shared device helpers for the cbg_b200 kernels (sm_90a).
#pragma once
#include <stdlib.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "cbg_layout.h"

#define CBG_FULL 0xffffffffu

// error plumbing (api.cu owns the storage)
void cbg_set_error(const char* fmt, ...);
#define CBG_CUDA_OK(expr)                                                        \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess) {                                                     \
      cbg_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return 2;                                                                  \
    }                                                                            \
  } while (0)

// One-time per-DEVICE setup guards: kernel attributes (opt-in shared memory) belong to a device's context, so a
// process that drives several GPUs must set them once on each.
constexpr int CBG_MAX_DEVICES = 64;
inline bool& cbg_dev_flag(bool (&flags)[CBG_MAX_DEVICES]) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= CBG_MAX_DEVICES) dev = 0;
  return flags[dev];
}

extern long long g_cbg_launches;
extern int g_cbg_prof_on;
// kernel families for the optional per-kernel CUDA-event profile (bench.py roofline)
enum CbgKernelFamily {
  CBG_K_KNN = 0, CBG_K_GATE, CBG_K_NODE_GEMM, CBG_K_X2H_K, CBG_K_X2H_V, CBG_K_H2X, CBG_K_CLASSIFIER,
  CBG_K_STEP_INIT, CBG_K_REVERSE, CBG_K_MISC, CBG_K_COUNT
};
void cbg_prof_mark(int family, int is_end, cudaStream_t st);
// bracket a kernel launch: PROF_BEGIN before it, LAUNCHED after it (surfaces launch errors,
// counts the launch, closes the profile bracket)
#define CBG_PROF_BEGIN(family, st) \
  do { if (g_cbg_prof_on) cbg_prof_mark((family), 0, (st)); } while (0)
#define CBG_LAUNCHED(family, st)                              \
  do {                                                        \
    CBG_CUDA_OK(cudaGetLastError());                          \
    g_cbg_launches += 1;                                      \
    if (g_cbg_prof_on) cbg_prof_mark((family), 1, (st));      \
  } while (0)

// Launch with (or without) programmatic stream serialization: the kernel may be scheduled before the previous kernel of
// the stream has finished; it must execute griddepcontrol.wait (cbg_tc.cuh: pdl_wait) before touching anything that
// kernel produces or still reads.  Off unless CBG_PDL=1 (DESIGN.md section 5.3).
inline bool cbg_pdl_enabled() {
  static int on = -1;
  if (on < 0) { const char* e = getenv("CBG_PDL"); on = (e && e[0] == '1') ? 1 : 0; }
  return on != 0;
}
template <typename... KArgs, typename... Args>
inline cudaError_t cbg_launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = cbg_pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// workspace carves: every region starts on a 256-byte boundary
inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v += __shfl_xor_sync(CBG_FULL, v, m);
  return v;
}

// ---- per-graph kernels (reverse steps, validation losses): one CTA of kGraphThreads threads per graph ----------------
constexpr int kGraphThreads = 128, kGraphWarps = kGraphThreads / 32;
static_assert(kGraphWarps == 4, "block_sum adds exactly four warp partials: (w0 + w1) + (w2 + w3)");

// first index of the ascending a[0, n) whose value is >= key (n if none)
__device__ __forceinline__ int lower_bound(const int* __restrict__ a, int n, int key) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// Graph g's ligand atoms [lo, hi), returned to every thread of the CTA: lig_node holds the ascending composed node index
// of every ligand atom and graph g owns the nodes [graph_ptr[g], graph_ptr[g + 1]).  Thread 0 searches, a barrier
// publishes the result.
__device__ __forceinline__ int2 graph_ligand_range(const int* __restrict__ lig_node, int n_lig,
                                                   const int* __restrict__ graph_ptr, int g) {
  __shared__ int s_rng[2];
  if (threadIdx.x == 0) {
    s_rng[0] = lower_bound(lig_node, n_lig, graph_ptr[g]);
    s_rng[1] = lower_bound(lig_node, n_lig, graph_ptr[g + 1]);
  }
  __syncthreads();
  return make_int2(s_rng[0], s_rng[1]);
}

// Sum of N per-thread values over the kGraphThreads threads of the CTA into out[N] (shared memory, read by any thread
// after the call), in a fixed order: warp_sum, then (w0 + w1) + (w2 + w3).  s_red is [kGraphWarps][N] shared scratch.
template <int N>
__device__ __forceinline__ void block_sum(float (&v)[N], float (*s_red)[N], float* out) {
#pragma unroll
  for (int c = 0; c < N; ++c) v[c] = warp_sum(v[c]);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int c = 0; c < N; ++c) s_red[threadIdx.x >> 5][c] = v[c];
  }
  __syncthreads();
  if (threadIdx.x < N) out[threadIdx.x] = (s_red[0][threadIdx.x] + s_red[1][threadIdx.x]) + (s_red[2][threadIdx.x] + s_red[3][threadIdx.x]);
  __syncthreads();
}

// Reduce NV per-lane values across the 32 lanes of a warp with a halving butterfly.
// On return lane l holds in v[0 .. NV/32) the full (all-lane) sums of the original
// indices l*(NV/32) + i.  NV must be a power of two >= 32; 2*NV-64 shuffles... (NV-NV/32).
template <int NV>
__device__ __forceinline__ void warp_transpose_reduce(float (&v)[NV], int lane) {
#pragma unroll
  for (int s = 0; s < 5; ++s) {
    const int mask = 16 >> s;
    const int n = NV >> (s + 1);
    const bool upper = (lane & mask) != 0;
#pragma unroll
    for (int i = 0; i < n; ++i) {
      const float send = upper ? v[i] : v[i + n];
      const float keep = upper ? v[i + n] : v[i];
      v[i] = keep + __shfl_xor_sync(CBG_FULL, send, mask);
    }
  }
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// Pairwise fp32 helpers: two IEEE-rn operations on the halves of a float2 (Hopper has no packed fp32 instruction:
// these compile to two scalar FFMA / FMUL / FADD and are bit-identical to the scalar forms).
__device__ __forceinline__ float2 ffma2(const float2 a, const float2 b, const float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(const float2 a, const float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(const float2 a, const float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ void fma4(float4& acc, const float4 w, const float s) {
  const float2 ss = make_float2(s, s);
  const float2 lo = ffma2(make_float2(w.x, w.y), ss, make_float2(acc.x, acc.y));
  const float2 hi = ffma2(make_float2(w.z, w.w), ss, make_float2(acc.z, acc.w));
  acc = make_float4(lo.x, lo.y, hi.x, hi.y);
}
__device__ __forceinline__ float4 add4(const float4 a, const float4 b) {
  const float2 lo = fadd2(make_float2(a.x, a.y), make_float2(b.x, b.y));
  const float2 hi = fadd2(make_float2(a.z, a.w), make_float2(b.z, b.w));
  return make_float4(lo.x, lo.y, hi.x, hi.y);
}
__device__ __forceinline__ float4 add4s(const float4 a, const float s) {
  const float2 ss = make_float2(s, s);
  const float2 lo = fadd2(make_float2(a.x, a.y), ss);
  const float2 hi = fadd2(make_float2(a.z, a.w), ss);
  return make_float4(lo.x, lo.y, hi.x, hi.y);
}
// a.x*b.x + a.y*b.y + a.z*b.z + a.w*b.w as (x,z | y,w) packed partial sums
__device__ __forceinline__ float dot4(const float4 a, const float4 b) {
  float2 t = fmul2(make_float2(a.x, a.y), make_float2(b.x, b.y));
  t = ffma2(make_float2(a.z, a.w), make_float2(b.z, b.w), t);
  return t.x + t.y;
}
// relu((a * rstd) * gamma + beta)
__device__ __forceinline__ float4 ln_relu4(const float4 a, const float rstd, const float4 gamma, const float4 beta) {
  const float2 rr = make_float2(rstd, rstd);
  float2 lo = fmul2(make_float2(a.x, a.y), rr), hi = fmul2(make_float2(a.z, a.w), rr);
  lo = ffma2(lo, make_float2(gamma.x, gamma.y), make_float2(beta.x, beta.y));
  hi = ffma2(hi, make_float2(gamma.z, gamma.w), make_float2(beta.z, beta.w));
  return make_float4(fmaxf(lo.x, 0.f), fmaxf(lo.y, 0.f), fmaxf(hi.x, 0.f), fmaxf(hi.y, 0.f));
}

// cooperative contiguous copy global -> shared, n floats (multiple of 4), both 16B aligned
__device__ __forceinline__ void block_copy_f4(float* dst, const float* __restrict__ src, int n_floats) {
  const int n4 = n_floats >> 2;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) st4(dst + 4 * i, ldg4(src + 4 * i));
}

// node flags are stored as a float in x4.w: 0/1 = ligand bit, +2 = generate bit
__device__ __forceinline__ int node_flags(const float4 x) { return (int)x.w; }
