// DiffSBDD validation loss (DiffSBDD.forward with self.training == False, diffsbdd.py:48-191) on a plan whose graphs
// are 2 n_t replicas of one batch: replica 2j is timestep j noised at t_j, replica 2j+1 the same timestep noised at 0.
//   sbdd_eval_noise_kernel   per replicated graph: remove_mean_batch of the clean ligand (the pocket moves with it),
//                            forward_pos_center_noise (zero_center=False: the noisy ligand's mean over ALL its atoms is
//                            removed from the generated atoms and from the pocket) and forward_type_add_noise on the
//                            continuous types onehot / 4 (diffusion_scheduler.py:706-710, 734-775), plus the ligand rows
//                            of the node state (bias + W c, like step_init)
//   sbdd_eval_loss_kernel    per (timestep, graph): the six terms of get_score_loss in eval mode (:897-920) - loss_t with
//                            the SNR weight, loss_0 of the t = 0 copy (continuous for positions, the discretised
//                            likelihood log_ph_given_z0_discrete for types), the KL of the clean state to the prior at T
//   sbdd_eval_reduce_kernel  per timestep: mean of the per-graph sums over the graphs below the last ligand graph
// Sums run in a fixed order and there are no atomics: repeated calls are bit-identical.
#include <math.h>
#include "cbg_kernels.cuh"

namespace {

// scatter_mean of the batch's clean ligand coordinates over atoms [lo, hi) (one-batch indices) into s_mean[3]
__device__ __forceinline__ void clean_mean(const float* __restrict__ x0, int lo, int hi, float (*s_red)[3], float* s_mean) {
  float s[3] = {0.f, 0.f, 0.f};
  for (int a = lo + threadIdx.x; a < hi; a += blockDim.x) {
#pragma unroll
    for (int c = 0; c < 3; ++c) s[c] += x0[3 * a + c];
  }
  block_sum<3>(s, s_red, s_mean);
  if (threadIdx.x < 3) s_mean[threadIdx.x] = __fdiv_rn(s_mean[threadIdx.x], (float)(hi > lo ? hi - lo : 1));
  __syncthreads();
}

// a generated atom's noised continuous type feature: alpha * onehot / 4 + sigma * eps, else onehot / 4
__device__ __forceinline__ float noised_type(bool gen, bool hot, float alpha, float sigma, float eps) {
  const float c0 = hot ? 0.25f : 0.f;
  return gen ? __fadd_rn(__fmul_rn(alpha, c0), __fmul_rn(sigma, eps)) : c0;
}

__global__ void __launch_bounds__(kGraphThreads) sbdd_eval_noise_kernel(SbddEvalArgs p) {
  __shared__ float s_red[kGraphWarps][3];
  __shared__ float s_mean0[3], s_m[3];
  const int g = blockIdx.x;                                  // replicated graph
  const int n_rep = 2 * p.n_t, B1 = p.b.n_graphs / n_rep, n1 = p.b.n_lig / n_rep;
  const int n_rec1 = (int)((p.n_nodes - p.b.n_lig) / n_rep);
  const int r = g / B1, j = r >> 1;
  const bool at_zero = (r & 1) != 0;
  const int2 rng = graph_ligand_range(p.b.lig_node, p.b.n_lig, p.b.graph_ptr, g);
  const int lo = rng.x, hi = rng.y, n_g = hi - lo;
  const int lo1 = lo - r * n1, hi1 = hi - r * n1;            // the same atoms in the batch
  const cbg_sbdd_eval_coef& cf = p.coef.c[j];
  const float ax = at_zero ? cf.pos_alpha_0 : cf.pos_alpha_t, sx = at_zero ? cf.pos_sigma_0 : cf.pos_sigma_t;
  const float ac = at_zero ? cf.type_alpha_0 : cf.type_alpha_t, sc = at_zero ? cf.type_sigma_0 : cf.type_sigma_t;
  const float* ex = (at_zero ? p.x_0_noise : p.x_t_noise) + (size_t)j * n1 * 3;
  const int K = p.b.num_classes;
  const float* ec = (at_zero ? p.c_0_noise : p.c_t_noise) + (size_t)j * n1 * K;
  clean_mean(p.b.x0, lo1, hi1, s_red, s_mean0);
  const float mean0[3] = {s_mean0[0], s_mean0[1], s_mean0[2]};
  // x_noisy = alpha * x0c + sigma * eps for every ligand atom; its graph mean m
  float s[3] = {0.f, 0.f, 0.f};
  for (int a = lo1 + threadIdx.x; a < hi1; a += blockDim.x) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float x0c = __fsub_rn(p.b.x0[3 * a + c], mean0[c]);
      s[c] += __fadd_rn(__fmul_rn(ax, x0c), __fmul_rn(sx, ex[3 * a + c]));
    }
  }
  block_sum<3>(s, s_red, s_m);
  if (threadIdx.x < 3) s_m[threadIdx.x] = __fdiv_rn(s_m[threadIdx.x], (float)(n_g > 0 ? n_g : 1));
  __syncthreads();
  const float m[3] = {s_m[0], s_m[1], s_m[2]};
  for (int a = lo1 + threadIdx.x; a < hi1; a += blockDim.x) {
    const int i = a + r * n1;
    const bool gen = p.b.gen[i] != 0;
    float4 v = p.b.x4[p.b.lig_node[i]];
    float xv[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float x0c = __fsub_rn(p.b.x0[3 * a + c], mean0[c]);
      xv[c] = gen ? __fsub_rn(__fadd_rn(__fmul_rn(ax, x0c), __fmul_rn(sx, ex[3 * a + c])), m[c]) : x0c;
    }
    v.x = xv[0]; v.y = xv[1]; v.z = xv[2];
    p.b.x4[p.b.lig_node[i]] = v;
  }
  // pocket rows: compose_context puts a graph's protein atoms first; x_rec - mean0 - m
  const int pb = p.b.graph_ptr[g], pe = p.b.graph_ptr[g + 1] - n_g;
  for (int pn = pb + threadIdx.x; pn < pe; pn += blockDim.x) {
    const int q = pn - lo - r * n_rec1;                      // protein atom of the batch
    float4 v = p.b.x4[pn];
    v.x = __fsub_rn(__fsub_rn(p.x_rec[3 * q], mean0[0]), m[0]);
    v.y = __fsub_rn(__fsub_rn(p.x_rec[3 * q + 1], mean0[1]), m[1]);
    v.z = __fsub_rn(__fsub_rn(p.x_rec[3 * q + 2], mean0[2]), m[2]);
    p.b.x4[pn] = v;
  }
  // ligand rows of h: bias + sum_c W[c] * c_tau[c] (one warp per atom, four columns per lane, like step_init)
  const int lane = threadIdx.x & 31;
  for (int i = lo + (threadIdx.x >> 5); i < hi; i += kGraphWarps) {
    const int a = i - r * n1;
    const bool gen = p.b.gen[i] != 0;
    const int v0 = (int)p.b.v0[a];
    float4 acc = ldg4(p.b.h_lig_bias + (size_t)i * CBG_H + 4 * lane);
    for (int c = 0; c < K; ++c)
      fma4(acc, ldg4(p.b.emb_wt + c * CBG_H + 4 * lane), noised_type(gen, c == v0, ac, sc, ec[(size_t)a * K + c]));
    st4(p.b.h + (size_t)p.b.lig_node[i] * CBG_H + 4 * lane, acc);
  }
}

__device__ __forceinline__ float cdf_standard_gaussian(float x) {
  return __fmul_rn(0.5f, __fadd_rn(1.f, erff(__fdiv_rn(x, 1.41421356f))));     // x / math.sqrt(2) in fp32
}

__global__ void __launch_bounds__(kGraphThreads) sbdd_eval_loss_kernel(SbddEvalArgs p) {
  __shared__ float s_red3[kGraphWarps][3];
  __shared__ float s_red6[kGraphWarps][6];
  __shared__ float s_mean0[3], s_tot[6];
  const int n_rep = 2 * p.n_t, B1 = p.b.n_graphs / n_rep, n1 = p.b.n_lig / n_rep;
  const int j = blockIdx.x / B1, g = blockIdx.x - j * B1;    // timestep, graph of the batch
  const int2 rng = graph_ligand_range(p.b.lig_node, p.b.n_lig, p.b.graph_ptr, g);     // replica 0's atoms are the batch's
  const int lo = rng.x, hi = rng.y, n_g = hi - lo;
  const cbg_sbdd_eval_coef& cf = p.coef.c[j];
  const int K = p.b.num_classes;
  clean_mean(p.b.x0, lo, hi, s_red3, s_mean0);
  const float mean0[3] = {s_mean0[0], s_mean0[1], s_mean0[2]};
  const float* ext = p.x_t_noise + (size_t)j * n1 * 3;
  const float* ex0 = p.x_0_noise + (size_t)j * n1 * 3;
  const float* ect = p.c_t_noise + (size_t)j * n1 * K;
  const float* ec0 = p.c_0_noise + (size_t)j * n1 * K;
  const float sigma0_cat = __fmul_rn(cf.type_sigma_0, 4.f);
  float* vp = p.vec_pos + (size_t)j * 3 * n1 * 3;             // eps_pred, score_0, score_pred
  float* va = p.vec_atom + (size_t)j * 3 * n1 * K;
  // error_t of both heads, error of the t = 0 positions, |alpha_T x0c|^2, log p(h | z_0), |alpha_T c0|^2
  float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int a = lo + threadIdx.x; a < hi; a += blockDim.x) {
    const int it = (2 * j) * n1 + a, i0 = (2 * j + 1) * n1 + a;
    const float4 xt4 = p.b.x4[p.b.lig_node[it]], x04 = p.b.x4[p.b.lig_node[i0]];
    const float xp_t[3] = {xt4.x, xt4.y, xt4.z}, xp_0[3] = {x04.x, x04.y, x04.z};
    float et = 0.f, e0 = 0.f, mu = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float eps = ext[3 * a + c];
      vp[3 * a + c] = xp_t[c];
      vp[(size_t)n1 * 3 + 3 * a + c] = __fmul_rn(eps, cf.pos_sigma_t);
      vp[(size_t)2 * n1 * 3 + 3 * a + c] = __fmul_rn(xp_t[c], cf.pos_sigma_t);
      const float dt = __fsub_rn(eps, xp_t[c]), d0 = __fsub_rn(ex0[3 * a + c], xp_0[c]);
      const float xa = __fmul_rn(cf.pos_alpha_T, __fsub_rn(p.b.x0[3 * a + c], mean0[c]));
      et = c == 0 ? __fmul_rn(dt, dt) : __fadd_rn(et, __fmul_rn(dt, dt));
      e0 = c == 0 ? __fmul_rn(d0, d0) : __fadd_rn(e0, __fmul_rn(d0, d0));
      mu = c == 0 ? __fmul_rn(xa, xa) : __fadd_rn(mu, __fmul_rn(xa, xa));
    }
    acc[0] += et; acc[1] += e0; acc[2] += mu;
    // types: error_t against the logits of the t copy; the discretised likelihood of the t = 0 copy's noised types
    const bool gen = p.b.gen[i0] != 0;
    const int v0 = (int)p.b.v0[a];
    const float* lg = p.logits + (size_t)it * K;
    float lp[CBG_MAXCLS];
    float ea = 0.f, mx = -INFINITY;
    for (int c = 0; c < K; ++c) {
      const float eps = ect[(size_t)a * K + c], cp = lg[c];
      va[(size_t)a * K + c] = cp;
      va[(size_t)n1 * K + (size_t)a * K + c] = __fmul_rn(eps, cf.type_sigma_t);
      va[(size_t)2 * n1 * K + (size_t)a * K + c] = __fmul_rn(cp, cf.type_sigma_t);
      const float d = __fsub_rn(eps, cp);
      ea = c == 0 ? __fmul_rn(d, d) : __fadd_rn(ea, __fmul_rn(d, d));
      const float cen = __fsub_rn(__fmul_rn(noised_type(gen, c == v0, cf.type_alpha_0, cf.type_sigma_0, ec0[(size_t)a * K + c]), 4.f), 1.f);
      const float pr = __fsub_rn(cdf_standard_gaussian(__fdiv_rn(__fadd_rn(cen, 0.5f), sigma0_cat)),
                                 cdf_standard_gaussian(__fdiv_rn(__fsub_rn(cen, 0.5f), sigma0_cat)));
      lp[c] = logf(__fadd_rn(pr, 1e-10f));
      mx = fmaxf(mx, lp[c]);
    }
    float se = 0.f;
    for (int c = 0; c < K; ++c) se += expf(lp[c] - mx);
    acc[3] += ea;
    acc[4] += __fsub_rn(lp[v0], __fadd_rn(logf(se), mx));     // logp of the atom's class (onehot weight 1)
    const float ca = __fmul_rn(cf.type_alpha_T, 0.25f);
    acc[5] += __fmul_rn(ca, ca);
  }
  block_sum<6>(acc, s_red6, s_tot);
  if (threadIdx.x == 0) {
    const float dp = (float)((n_g - 1) * 3), dc = (float)((n_g - 1) * K);   // subspace_dimensionality
    float* o = p.terms + ((size_t)j * B1 + g) * 6;
    o[0] = __fmul_rn(cf.pos_t_weight, s_tot[0]);
    o[1] = __fsub_rn(__fmul_rn(0.5f, s_tot[1]), __fmul_rn(dp, cf.pos_log_const));
    o[2] = __fsub_rn(__fadd_rn(__fmul_rn(dp, cf.pos_log_inv_sigma_T), __fmul_rn(0.5f, __fadd_rn(__fmul_rn(dp, cf.pos_sigma2_T), s_tot[2]))),
                     __fmul_rn(0.5f, dp));
    o[3] = __fmul_rn(cf.type_t_weight, s_tot[3]);
    o[4] = __fsub_rn(-s_tot[4], __fmul_rn(dc, cf.type_log_const));
    o[5] = __fsub_rn(__fadd_rn(cf.type_log_inv_sigma_T, __fmul_rn(0.5f, __fadd_rn(cf.type_sigma2_T, s_tot[5]))), 0.5f);
  }
}

// one thread per timestep: get_score_loss's loss.mean() over the B = (last ligand graph + 1) rows of scatter_add
__global__ void sbdd_eval_reduce_kernel(SbddEvalArgs p) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= p.n_t) return;
  const int B1 = p.b.n_graphs / (2 * p.n_t);
  int B = 0;
  for (int g = B1 - 1; g >= 0 && B == 0; --g)
    if (lower_bound(p.b.lig_node, p.b.n_lig, p.b.graph_ptr[g]) < lower_bound(p.b.lig_node, p.b.n_lig, p.b.graph_ptr[g + 1])) B = g + 1;
  const float* tm = p.terms + (size_t)j * B1 * 6;
  float sp = 0.f, sa = 0.f;
  for (int g = 0; g < B; ++g) {
    sp += __fadd_rn(__fadd_rn(tm[6 * g], tm[6 * g + 1]), tm[6 * g + 2]);
    sa += __fadd_rn(__fadd_rn(tm[6 * g + 3], tm[6 * g + 4]), tm[6 * g + 5]);
  }
  p.t_loss[2 * j] = __fdiv_rn(sp, (float)(B > 0 ? B : 1));
  p.t_loss[2 * j + 1] = __fdiv_rn(sa, (float)(B > 0 ? B : 1));
}

}  // namespace

int cbg_launch_sbdd_eval_noise(const SbddEvalArgs& a, cudaStream_t st) {
  if (a.b.n_graphs <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_STEP_INIT, st);
  sbdd_eval_noise_kernel<<<a.b.n_graphs, kGraphThreads, 0, st>>>(a);
  CBG_LAUNCHED(CBG_K_STEP_INIT, st);
  return 0;
}

int cbg_launch_sbdd_eval_loss(const SbddEvalArgs& a, cudaStream_t st) {
  if (a.b.n_graphs <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_REVERSE, st);
  sbdd_eval_loss_kernel<<<a.b.n_graphs / 2, kGraphThreads, 0, st>>>(a);      // n_t * B: one CTA per (timestep, graph)
  CBG_LAUNCHED(CBG_K_REVERSE, st);
  CBG_PROF_BEGIN(CBG_K_REVERSE, st);
  sbdd_eval_reduce_kernel<<<(a.n_t + 31) / 32, 32, 0, st>>>(a);
  CBG_LAUNCHED(CBG_K_REVERSE, st);
  return 0;
}
