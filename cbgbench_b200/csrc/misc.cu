// Small kernels around the message-passing layers: coordinate packing, per-step node-state
// initialisation (ligand embedding), masked coordinate update, classifier head and the
// fused reverse-diffusion step.
#include <math.h>
#include "cbg_kernels.cuh"

namespace {

__global__ void pack_x4_kernel(const float* __restrict__ x, const unsigned char* __restrict__ lig,
                               const unsigned char* __restrict__ gen, long long n, float4* __restrict__ x4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = (lig[i] ? 1 : 0) | (gen[i] ? 2 : 0);
  x4[i] = make_float4(x[3 * i], x[3 * i + 1], x[3 * i + 2], (float)f);
}

__global__ void unpack_x_kernel(const float4* __restrict__ x4, long long n, float* __restrict__ x) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 v = x4[i];
  x[3 * i] = v.x; x[3 * i + 1] = v.y; x[3 * i + 2] = v.z;
}

__global__ void gather_x_kernel(const float4* __restrict__ x4, const int* __restrict__ idx, int n,
                                float* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const float4 v = x4[idx[k]];
  out[3 * k] = v.x; out[3 * k + 1] = v.y; out[3 * k + 2] = v.z;
}

// x[node_idx[n]] += dx[n]   (x += delta_x * gen_flag, unitransformer.py:182; node_idx lists
// exactly the nodes whose gen_flag is set)
__global__ void apply_dx_kernel(float4* __restrict__ x4, const int* __restrict__ node_idx,
                                const float* __restrict__ dx, int n) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int i = node_idx[k];
  float4 v = x4[i];
  const float4 d = ld4(dx + 4 * (size_t)k);
  v.x += d.x; v.y += d.y; v.z += d.z;
  x4[i] = v;
}

// classifier head: Linear(128,128) -> softplus - ln2 -> Linear(128,K)   (unitransformer.py:46-51,119-121)
// one warp per row; lane owns hidden units 4*lane..4*lane+3
constexpr int kClsFloats = 128 * 128 + 128 + 16 * 128 + 32;

__global__ void __launch_bounds__(256) classifier_kernel(const float* __restrict__ cw, const float* __restrict__ h,
                                                         const int* __restrict__ row_idx, int n_rows,
                                                         int num_classes, float* __restrict__ logits) {
  extern __shared__ __align__(16) float sm[];
  block_copy_f4(sm, cw, kClsFloats);
  __syncthreads();
  const float* w0t = sm;                  // [k][n]
  const float* b0 = sm + 128 * 128;
  const float* w1 = b0 + 128;             // [16][128]
  const float* b1 = w1 + 16 * 128;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = blockIdx.x * 8 + warp; r < n_rows; r += gridDim.x * 8) {
    const int i = row_idx ? row_idx[r] : r;
    const float* hi = h + (size_t)i * CBG_H;
    float4 acc = ld4(b0 + 4 * lane);
#pragma unroll 4
    for (int k4 = 0; k4 < 32; ++k4) {
      const float4 hv = ldg4(hi + 4 * k4);
      fma4(acc, ld4(w0t + (4 * k4 + 0) * 128 + 4 * lane), hv.x);
      fma4(acc, ld4(w0t + (4 * k4 + 1) * 128 + 4 * lane), hv.y);
      fma4(acc, ld4(w0t + (4 * k4 + 2) * 128 + 4 * lane), hv.z);
      fma4(acc, ld4(w0t + (4 * k4 + 3) * 128 + 4 * lane), hv.w);
    }
    // F.softplus (beta=1, threshold=20) minus ln 2   (common.py:174-180)
    const float ln2 = 0.693147180559945f;
    float a[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
    for (int c = 0; c < 4; ++c) a[c] = ((a[c] > 20.f) ? a[c] : log1pf(expf(a[c]))) - ln2;
    float part[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) part[c] = 0.f;
#pragma unroll
    for (int c = 0; c < CBG_MAXCLS; ++c) {
      const float4 wv = ld4(w1 + c * 128 + 4 * lane);
      part[c] = fmaf(a[3], wv.w, fmaf(a[2], wv.z, fmaf(a[1], wv.y, a[0] * wv.x)));
    }
    warp_transpose_reduce<32>(part, lane);   // lane c holds class c
    if (lane < num_classes) logits[(size_t)r * num_classes + lane] = part[0] + b1[lane];
  }
}

// Per-step node state: ligand rows get coordinates from x_lig and features
//   h = W_atom c_lig + (b_atom + indicator)   (PLContextEmbedder.forward, context_emb.py:201-222;
// the c_lig-independent part is precomputed per atom in h_lig_bias); other rows copy the
// step-invariant protein embedding h_static (SURVEY.md A7).
__device__ __forceinline__ void step_init_body(const float* __restrict__ x_lig, const float* __restrict__ c_lig,
                                               const int* __restrict__ lig_node, int n_lig, int num_classes,
                                               const float* __restrict__ emb_wt,   // [K][128]
                                               const float* __restrict__ h_lig_bias,  // [n_lig][128]
                                               float4* __restrict__ x4, float* __restrict__ h) {
  const int a = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (a >= n_lig) return;
  const int i = lig_node[a];
  float4 acc = ldg4(h_lig_bias + (size_t)a * CBG_H + 4 * lane);
  for (int c = 0; c < num_classes; ++c) fma4(acc, ldg4(emb_wt + c * CBG_H + 4 * lane), __ldg(c_lig + (size_t)a * num_classes + c));
  st4(h + (size_t)i * CBG_H + 4 * lane, acc);
  if (lane == 0) {
    float4 v = x4[i];
    v.x = x_lig[3 * a]; v.y = x_lig[3 * a + 1]; v.z = x_lig[3 * a + 2];
    x4[i] = v;
  }
}
__global__ void __launch_bounds__(256) step_init_kernel(const float* __restrict__ x_lig, const float* __restrict__ c_lig,
                                                        const int* __restrict__ lig_node, int n_lig, int num_classes,
                                                        const float* __restrict__ emb_wt, const float* __restrict__ h_lig_bias,
                                                        float4* __restrict__ x4, float* __restrict__ h) {
  step_init_body(x_lig, c_lig, lig_node, n_lig, num_classes, emb_wt, h_lig_bias, x4, h);
}
// graph replay: the step's x_t / c_t pointers come from device memory
__global__ void __launch_bounds__(256) step_init_io_kernel(const StepIO* __restrict__ io, const int* __restrict__ lig_node,
                                                           int n_lig, int num_classes, const float* __restrict__ emb_wt,
                                                           const float* __restrict__ h_lig_bias, float4* __restrict__ x4,
                                                           float* __restrict__ h) {
  step_init_body(io->x_t, io->c_t, lig_node, n_lig, num_classes, emb_wt, h_lig_bias, x4, h);
}

// Fused reverse step for one ligand atom per thread.
//   positions: CTNVPScheduler.backward_remove_noise(type='denoise') diffusion_scheduler.py:144-165
//   types:     TypeVPScheduler.backward_remove_noise                diffusion_scheduler.py:367-378
//              (q_v_posterior :407-418, q_v_pred :420-429, q_v_pred_one_timestep :431-441,
//               log_sample_categorical / log_add_exp categorical.py:26-37)
__device__ __forceinline__ void reverse_body(const ReverseArgs& p, float logvar, float nonzero) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= p.n_lig) return;
  const int K = p.num_classes;
  const bool gen = p.gen[a] != 0;
  const float* x0p = p.x0 + (size_t)(p.x0_idx ? p.x0_idx[a] : a) * p.x0_stride;
  const float x0v[3] = {x0p[0], x0p[1], x0p[2]};
  const float sigma = expf(0.5f * logvar);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float xt = p.x_t[3 * a + c];
    const float mean = __fadd_rn(__fmul_rn(p.c0, x0v[c]), __fmul_rn(p.ct, xt));
    const float xs = __fadd_rn(mean, __fmul_rn(__fmul_rn(nonzero, sigma), p.pos_noise[3 * a + c]));
    p.x_next[3 * a + c] = gen ? xs : xt;
  }
  float lg[CBG_MAXCLS], un[CBG_MAXCLS];
  float mx = -INFINITY;
  for (int c = 0; c < K; ++c) { lg[c] = p.logits[(size_t)a * K + c]; mx = fmaxf(mx, lg[c]); }
  float se = 0.f;
  for (int c = 0; c < K; ++c) se += expf(lg[c] - mx);
  const float lse = mx + logf(se);
  const float logK = logf((float)K);
  float m2 = -INFINITY;
  int arg_ct = 0;
  float best_ct = -INFINITY;
  for (int c = 0; c < K; ++c) {
    const float ctv = p.c_t[(size_t)a * K + c];
    if (ctv > best_ct) { best_ct = ctv; arg_ct = c; }
    const float log_c_pred = lg[c] - lse;
    const float log_ct = logf(ctv + 1e-8f);
    const float A = log_add_exp(log_c_pred + p.lac_prev, p.l1mac_prev - logK);
    const float B = log_add_exp(log_ct + p.la, p.l1ma - logK);
    un[c] = A + B;
    m2 = fmaxf(m2, un[c]);
  }
  float s2 = 0.f;
  for (int c = 0; c < K; ++c) s2 += expf(un[c] - m2);
  const float lse2 = m2 + logf(s2);
  int arg = 0;
  float best = -INFINITY;
  for (int c = 0; c < K; ++c) {
    const float u = p.type_u[(size_t)a * K + c];
    const float gumbel = -logf(-logf(u + 1e-30f) + 1e-30f);
    const float score = gumbel + (un[c] - lse2);
    if (score > best) { best = score; arg = c; }
  }
  const int v = gen ? arg : arg_ct;
  p.v_next[a] = v;
  for (int c = 0; c < K; ++c) p.c_next[(size_t)a * K + c] = (c == v) ? 1.f : 0.f;
}

__global__ void __launch_bounds__(128) reverse_kernel(ReverseArgs p, float logvar, float nonzero) { reverse_body(p, logvar, nonzero); }
// graph replay: per-step pointers and schedule coefficients come from device memory
__global__ void __launch_bounds__(128) reverse_io_kernel(ReverseArgs p, const StepIO* __restrict__ io) {
  p.x_t = io->x_t; p.c_t = io->c_t; p.pos_noise = io->pos_noise; p.type_u = io->type_u;
  p.x_next = io->x_next; p.c_next = io->c_next; p.v_next = io->v_next;
  p.c0 = io->c0; p.ct = io->ct; p.lac_prev = io->lac_prev; p.l1mac_prev = io->l1mac_prev; p.la = io->la; p.l1ma = io->l1ma;
  reverse_body(p, io->logvar, io->nonzero);
}

// DiffSBDD reverse step + COM projection, one CTA per graph (see SbddArgs)
__global__ void __launch_bounds__(kGraphThreads) sbdd_reverse_kernel(SbddArgs p) {
  __shared__ float s_red[kGraphWarps][3];
  __shared__ float s_mean[3];
  const int g = blockIdx.x;
  const int ns = p.graph_ptr[g], ne = p.graph_ptr[g + 1];
  const int2 rng = graph_ligand_range(p.lig_node, p.n_lig, p.graph_ptr, g);
  const int lo = rng.x, hi = rng.y;
  float sum[3] = {0.f, 0.f, 0.f};
  for (int a = lo + threadIdx.x; a < hi; a += blockDim.x) {
    const float4 pr = p.x4[p.lig_node[a]];
    const float pred[3] = {pr.x, pr.y, pr.z};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float zt = p.x_t[3 * a + c], nz = __fmul_rn(p.s, p.x_noise[3 * a + c]);
      const float mu = p.mode == 0 ? __fsub_rn(__fdiv_rn(zt, p.a), __fmul_rn(p.b, pred[c]))
                                   : __fmul_rn(p.a, __fsub_rn(zt, __fmul_rn(p.b, pred[c])));
      const float zs = __fadd_rn(mu, nz);
      p.x_next[3 * a + c] = zs;
      sum[c] += zs;
    }
  }
  block_sum<3>(sum, s_red, s_mean);
  if (threadIdx.x < 3) s_mean[threadIdx.x] = __fdiv_rn(s_mean[threadIdx.x], (float)(hi > lo ? hi - lo : 1));   // scatter_mean
  __syncthreads();
  const float m[3] = {s_mean[0], s_mean[1], s_mean[2]};
  for (int a = lo + threadIdx.x; a < hi; a += blockDim.x) {          // same thread wrote these entries
#pragma unroll
    for (int c = 0; c < 3; ++c) p.x_next[3 * a + c] = __fsub_rn(p.x_next[3 * a + c], m[c]);
  }
  for (int i = ns + threadIdx.x; i < ne; i += blockDim.x) {
    float4 v = p.x4[i];
    if ((node_flags(v) & 1) == 0) {                                    // pocket atom
      v.x = __fsub_rn(v.x, m[0]); v.y = __fsub_rn(v.y, m[1]); v.z = __fsub_rn(v.z, m[2]);
      p.x4[i] = v;
    }
  }
  const int K = p.num_classes;
  for (long long e = (long long)lo * K + threadIdx.x; e < (long long)hi * K; e += blockDim.x) {
    const float ct = p.c_t[e];
    p.c_next[e] = p.mode == 0
        ? __fadd_rn(__fsub_rn(__fdiv_rn(ct, p.a), __fmul_rn(p.b, p.logits[e])), __fmul_rn(p.s, p.c_noise[e]))
        : __fmul_rn(ct, 4.f);
  }
}

__global__ void scatter_x_kernel(const float* __restrict__ x, const int* __restrict__ idx, int n,
                                 float4* __restrict__ x4) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n) return;
  float4 v = x4[idx[a]];
  v.x = x[3 * a]; v.y = x[3 * a + 1]; v.z = x[3 * a + 2];
  x4[idx[a]] = v;
}

// DiffBP reverse step, one CTA per graph (see BpArgs)
__global__ void __launch_bounds__(kGraphThreads) bp_reverse_kernel(BpArgs p) {
  __shared__ float s_red[kGraphWarps][6];
  __shared__ float s_mean[6];
  const int2 rng = graph_ligand_range(p.lig_node, p.n_lig, p.graph_ptr, blockIdx.x);
  const int lo = rng.x, hi = rng.y;
  float sum[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int a = lo + threadIdx.x; a < hi; a += blockDim.x) {
    const float4 xc = p.x4[p.lig_node[a]];
    const float com[3] = {xc.x, xc.y, xc.z};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float xt = p.x_t[3 * a + c];
      sum[c] += __fsub_rn(p.x_pred[3 * a + c], xt);
      sum[3 + c] += __fsub_rn(com[c], xt);
    }
  }
  block_sum<6>(sum, s_red, s_mean);
  if (threadIdx.x < 6) s_mean[threadIdx.x] = __fdiv_rn(s_mean[threadIdx.x], (float)(hi > lo ? hi - lo : 1));
  __syncthreads();
  const int K = p.num_classes;
  const float sigma = __fsqrt_rn(__fsub_rn(1.f, p.abar));
  const float denom = __fsqrt_rn(__fsub_rn(1.f, p.beta));
  const float nscale = __fmul_rn(p.nonzero, __fsqrt_rn(p.beta));
  for (int a = lo + threadIdx.x; a < hi; a += blockDim.x) {
    const bool gen = p.gen[a] != 0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float xt = p.x_t[3 * a + c];
      const float eps = __fadd_rn(__fsub_rn(__fsub_rn(p.x_pred[3 * a + c], xt), s_mean[c]), s_mean[3 + c]);
      const float score = -__fdiv_rn(eps, sigma);
      float xs = __fdiv_rn(__fadd_rn(xt, __fmul_rn(p.beta, score)), denom);
      xs = __fadd_rn(xs, __fmul_rn(nscale, p.pos_noise[3 * a + c]));
      p.x_next[3 * a + c] = gen ? xs : xt;
      if (p.eps_out) p.eps_out[3 * a + c] = eps;
    }
    // types: argmax of the softmax probabilities (first maximum), change only absorbing-state atoms
    float mx = -INFINITY;
    for (int c = 0; c < K; ++c) mx = fmaxf(mx, p.logits[(size_t)a * K + c]);
    float se = 0.f;
    for (int c = 0; c < K; ++c) se += expf(p.logits[(size_t)a * K + c] - mx);
    int v_pred = 0, vt = 0;
    float best = -INFINITY, best_ct = -INFINITY;
    for (int c = 0; c < K; ++c) {
      const float pr = __fdiv_rn(expf(p.logits[(size_t)a * K + c] - mx), se);
      if (pr > best) { best = pr; v_pred = c; }
      const float ctv = p.c_t[(size_t)a * K + c];
      if (ctv > best_ct) { best_ct = ctv; vt = c; }
    }
    const bool change = (p.type_u[a] < p.prob) && gen && vt == 0;
    const int v = change ? v_pred : vt;
    p.v_next[a] = v;
    for (int c = 0; c < K; ++c) p.c_next[(size_t)a * K + c] = (c == v) ? 1.f : 0.f;
  }
}

}  // namespace

int cbg_launch_scatter_x(const float* x, const int* idx, int n, float4* x4, cudaStream_t st) {
  if (n <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_MISC, st);
  scatter_x_kernel<<<(n + 255) / 256, 256, 0, st>>>(x, idx, n, x4);
  CBG_LAUNCHED(CBG_K_MISC, st);
  return 0;
}

int cbg_launch_bp_reverse(const BpArgs& a, cudaStream_t st) {
  if (a.n_graphs <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_REVERSE, st);
  bp_reverse_kernel<<<a.n_graphs, kGraphThreads, 0, st>>>(a);
  CBG_LAUNCHED(CBG_K_REVERSE, st);
  return 0;
}

int cbg_launch_sbdd_reverse(const SbddArgs& a, cudaStream_t st) {
  if (a.n_graphs <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_REVERSE, st);
  sbdd_reverse_kernel<<<a.n_graphs, kGraphThreads, 0, st>>>(a);
  CBG_LAUNCHED(CBG_K_REVERSE, st);
  return 0;
}

int cbg_launch_pack_x4(const float* x, const unsigned char* lig_flag, const unsigned char* gen_flag,
                       long long n, float4* x4, cudaStream_t st) {
  if (n <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_MISC, st);
  pack_x4_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, lig_flag, gen_flag, n, x4);
  CBG_LAUNCHED(CBG_K_MISC, st);
  return 0;
}

int cbg_launch_unpack_x(const float4* x4, long long n, float* x, cudaStream_t st) {
  if (n <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_MISC, st);
  unpack_x_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x4, n, x);
  CBG_LAUNCHED(CBG_K_MISC, st);
  return 0;
}

int cbg_launch_gather_x(const float4* x4, const int* idx, int n, float* out, cudaStream_t st) {
  if (n <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_MISC, st);
  gather_x_kernel<<<(n + 255) / 256, 256, 0, st>>>(x4, idx, n, out);
  CBG_LAUNCHED(CBG_K_MISC, st);
  return 0;
}

int cbg_launch_apply_dx(float4* x4, const int* node_idx, const float* dx, int n, cudaStream_t st) {
  if (n <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_MISC, st);
  apply_dx_kernel<<<(n + 255) / 256, 256, 0, st>>>(x4, node_idx, dx, n);
  CBG_LAUNCHED(CBG_K_MISC, st);
  return 0;
}

int cbg_launch_classifier(const float* blob_global, const float* h, const int* row_idx, int n_rows,
                          int num_classes, float* logits, cudaStream_t st) {
  if (n_rows <= 0) return 0;
  if (num_classes < 1 || num_classes > CBG_MAXCLS) { cbg_set_error("num_classes=%d outside [1,%d]", num_classes, CBG_MAXCLS); return 1; }
  static bool attr_dev[CBG_MAX_DEVICES] = {};
  bool& attr_set = cbg_dev_flag(attr_dev);
  if (!attr_set) {
    CBG_CUDA_OK(cudaFuncSetAttribute(classifier_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kClsFloats * 4));
    attr_set = true;
  }
  int grid = (n_rows + 7) / 8;
  if (grid > 2 * 132) grid = 2 * 132;
  CBG_PROF_BEGIN(CBG_K_CLASSIFIER, st);
  classifier_kernel<<<grid, 256, kClsFloats * 4, st>>>(blob_global + cbg_layout::global_offset(CBG_GF_CLS_W0T), h,
                                                       row_idx, n_rows, num_classes, logits);
  CBG_LAUNCHED(CBG_K_CLASSIFIER, st);
  return 0;
}

int cbg_launch_step_init(const float* x_lig, const float* c_lig, const int* lig_node, int n_lig,
                         int num_classes, const float* emb_wt, const float* h_lig_bias,
                         const float* h_static, long long n_nodes, float4* x4, float* h, cudaStream_t st) {
  CBG_CUDA_OK(cudaMemcpyAsync(h, h_static, (size_t)n_nodes * CBG_H * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (n_lig <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_STEP_INIT, st);
  step_init_kernel<<<(n_lig + 7) / 8, 256, 0, st>>>(x_lig, c_lig, lig_node, n_lig, num_classes, emb_wt,
                                                    h_lig_bias, x4, h);
  CBG_LAUNCHED(CBG_K_STEP_INIT, st);
  return 0;
}

int cbg_launch_step_init_io(const StepIO* io, const int* lig_node, int n_lig, int num_classes, const float* emb_wt,
                            const float* h_lig_bias, const float* h_static, long long n_nodes, float4* x4, float* h,
                            cudaStream_t st) {
  CBG_CUDA_OK(cudaMemcpyAsync(h, h_static, (size_t)n_nodes * CBG_H * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (n_lig <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_STEP_INIT, st);
  step_init_io_kernel<<<(n_lig + 7) / 8, 256, 0, st>>>(io, lig_node, n_lig, num_classes, emb_wt, h_lig_bias, x4, h);
  CBG_LAUNCHED(CBG_K_STEP_INIT, st);
  return 0;
}

int cbg_launch_reverse_io(const ReverseArgs& a, const StepIO* io, cudaStream_t st) {
  if (a.n_lig <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_REVERSE, st);
  reverse_io_kernel<<<(a.n_lig + 127) / 128, 128, 0, st>>>(a, io);
  CBG_LAUNCHED(CBG_K_REVERSE, st);
  return 0;
}

int cbg_launch_reverse(const ReverseArgs& a, float logvar, float nonzero, cudaStream_t st) {
  if (a.n_lig <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_REVERSE, st);
  reverse_kernel<<<(a.n_lig + 127) / 128, 128, 0, st>>>(a, logvar, nonzero);
  CBG_LAUNCHED(CBG_K_REVERSE, st);
  return 0;
}
