// TargetDiff validation loss (TargetDiff.forward with self.training == False, targetdiff.py:41-124) on a plan whose
// graphs are R replicas of one batch, replica r noised at its own timestep t_r:
//   eval_noise_kernel   forward noising of positions (CTNVPScheduler.forward_add_noise, diffusion_scheduler.py:117-134)
//                       and types (TypeVPScheduler.forward_add_noise / qct_c0_sample, :339-346, :380-396) plus the
//                       ligand rows of the node state (what step_init_kernel does for a sampling step)
//   eval_loss_kernel    per (replica, graph): position MSE (CTNVPScheduler.get_loss type='denoise', :185-201) and the
//                       type KL / decoder NLL (TypeVPScheduler.get_loss / compute_loss / q_v_posterior, :348-418),
//                       summed in a fixed order; writes x_pred and c_pred = softmax(logits)
//   eval_reduce_kernel  per replica: scatter_mean(...).mean() over graphs 0 .. (last graph with a generated atom)
// No atomics: repeated runs are bit-identical.
#include <math.h>
#include "cbg_kernels.cuh"

namespace {

__global__ void __launch_bounds__(128) eval_noise_kernel(EvalArgs p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;      // replicated ligand atom
  if (i >= p.b.n_lig) return;
  const int n1 = p.b.n_lig / p.n_rep;
  const int r = i / n1, a = i - r * n1;
  const cbg_eval_coef cf = p.coef.c[r];
  const int K = p.b.num_classes;
  const bool gen = p.b.gen[i] != 0;
  // positions: x_t = sqrt(a) * x0 + sqrt(1 - a) * eps   (two separately rounded products and one add)
  const float sa = __fsqrt_rn(cf.alphas_cumprod), s1 = __fsqrt_rn(__fsub_rn(1.f, cf.alphas_cumprod));
  float xt[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float x0 = p.b.x0[3 * a + c];
    xt[c] = gen ? __fadd_rn(__fmul_rn(sa, x0), __fmul_rn(s1, p.pos_noise[3 * (size_t)i + c])) : x0;
    p.xt[3 * (size_t)i + c] = xt[c];
  }
  // types: v_t = argmax(log q(v_t | v_0) + Gumbel(u)),  log q = log_add_exp(log_c0 + lac[t], l1mac[t] - log K)
  const int v0 = (int)p.b.v0[a];
  const float logK = (float)log((double)K);
  const float b = __fsub_rn(cf.log_one_minus_alphas_cumprod, logK);
  int arg = 0;
  float best = -INFINITY;
  for (int c = 0; c < K; ++c) {
    const float lq = log_add_exp(__fadd_rn(c == v0 ? 0.f : log_1e30(), cf.log_alphas_cumprod), b);
    const float u = p.type_u[(size_t)i * K + c];
    const float score = -logf(-logf(u + 1e-30f) + 1e-30f) + lq;
    if (score > best) { best = score; arg = c; }
  }
  const int vt = gen ? arg : v0;
  p.vt[i] = vt;
  store_noised_ligand(p.b, i, xt, vt);
}

// q_v_posterior(log_v0, log_vt, t) (diffusion_scheduler.py:407-418) for one atom; log_vt is the clamped log one-hot of vt
__device__ __forceinline__ void q_v_posterior(const float* lv0, int vt, const cbg_eval_coef& cf, float logK, int K, float* out) {
  const float ba = __fsub_rn(cf.log_one_minus_alphas_cumprod_prev, logK), bb = __fsub_rn(cf.log_one_minus_alpha, logK);
  float m = -INFINITY;
  for (int c = 0; c < K; ++c) {
    const float A = log_add_exp(__fadd_rn(lv0[c], cf.log_alphas_cumprod_prev), ba);
    const float B = log_add_exp(__fadd_rn(c == vt ? 0.f : log_1e30(), cf.log_alpha), bb);
    out[c] = __fadd_rn(A, B);
    m = fmaxf(m, out[c]);
  }
  float s = 0.f;
  for (int c = 0; c < K; ++c) s += expf(out[c] - m);
  const float lse = m + logf(s);
  for (int c = 0; c < K; ++c) out[c] = __fsub_rn(out[c], lse);
}

__global__ void __launch_bounds__(kGraphThreads) eval_loss_kernel(EvalArgs p) {
  __shared__ float s_red[kGraphWarps][3], s_tot[3];
  const int g = blockIdx.x;                                  // replicated graph
  const int r = g / (p.b.n_graphs / p.n_rep);
  const int2 rng = graph_ligand_range(p.b.lig_node, p.b.n_lig, p.b.graph_ptr, g);
  const int lo = rng.x, hi = rng.y;
  const int n1 = p.b.n_lig / p.n_rep;
  const cbg_eval_coef cf = p.coef.c[r];
  const int K = p.b.num_classes;
  const float logK = (float)log((double)K);
  float sum_pos = 0.f, sum_atom = 0.f, cnt = 0.f;
  for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const int a = i - r * n1;
    const float4 xp = p.b.x4[p.b.lig_node[i]];
    p.x_pred[3 * (size_t)i] = xp.x; p.x_pred[3 * (size_t)i + 1] = xp.y; p.x_pred[3 * (size_t)i + 2] = xp.z;
    // log_softmax of the classifier logits; c_pred = exp(log_softmax)
    float lcp[CBG_MAXCLS], lc0[CBG_MAXCLS], lpt[CBG_MAXCLS], lpp[CBG_MAXCLS];
    float mx = -INFINITY;
    for (int c = 0; c < K; ++c) { lcp[c] = p.logits[(size_t)i * K + c]; mx = fmaxf(mx, lcp[c]); }
    float se = 0.f;
    for (int c = 0; c < K; ++c) se += expf(lcp[c] - mx);
    const float lse = logf(se);
    for (int c = 0; c < K; ++c) {
      lcp[c] = __fsub_rn(__fsub_rn(lcp[c], mx), lse);
      p.c_pred[(size_t)i * K + c] = expf(lcp[c]);
    }
    if (p.b.gen[i] == 0) continue;
    // positions: ||x_pred - x0||^2
    const float d0 = __fsub_rn(xp.x, p.b.x0[3 * a]), d1 = __fsub_rn(xp.y, p.b.x0[3 * a + 1]), d2 = __fsub_rn(xp.z, p.b.x0[3 * a + 2]);
    sum_pos += __fadd_rn(__fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)), __fmul_rn(d2, d2));
    // types: KL(q(v_{t-1} | v_t, v_0) || q(v_{t-1} | v_t, c_pred)), or at t == 0 the decoder NLL -sum exp(log_c0) log p
    const int v0 = (int)p.b.v0[a], vt = (int)p.vt[i];
    for (int c = 0; c < K; ++c) lc0[c] = c == v0 ? 0.f : log_1e30();
    q_v_posterior(lc0, vt, cf, logK, K, lpt);
    q_v_posterior(lcp, vt, cf, logK, K, lpp);
    float kl = 0.f, nll = 0.f;
    for (int c = 0; c < K; ++c) {
      kl += __fmul_rn(expf(lpt[c]), __fsub_rn(lpt[c], lpp[c]));
      nll += __fmul_rn(expf(lc0[c]), lpp[c]);
    }
    nll = -nll;
    const float mask = cf.t_is_zero ? 1.f : 0.f;
    sum_atom += __fadd_rn(__fmul_rn(mask, nll), __fmul_rn(__fsub_rn(1.f, mask), kl));
    cnt += 1.f;
  }
  float v[3] = {sum_pos, sum_atom, cnt};
  block_sum<3>(v, s_red, s_tot);
  if (threadIdx.x == 0) {
    const float n = fmaxf(s_tot[2], 1.f);                     // scatter_mean: sum / max(count, 1)
    p.graph_loss[2 * (size_t)g] = __fdiv_rn(s_tot[0], n);
    p.graph_loss[2 * (size_t)g + 1] = __fdiv_rn(s_tot[1], n);
    p.graph_cnt[g] = (int)s_tot[2];
  }
}

// one thread per replica: the output of scatter_mean has max(generated graph id) + 1 rows (graphs without generated
// atoms below that id count as 0); .mean() of no rows is NaN
__global__ void eval_reduce_kernel(EvalArgs p) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.n_rep) return;
  const int B = p.b.n_graphs / p.n_rep;
  int last = -1;
  for (int g = 0; g < B; ++g) if (p.graph_cnt[r * B + g] > 0) last = g;
  float s0 = 0.f, s1 = 0.f;
  for (int g = 0; g <= last; ++g) { s0 += p.graph_loss[2 * (size_t)(r * B + g)]; s1 += p.graph_loss[2 * (size_t)(r * B + g) + 1]; }
  const float n = (float)(last + 1);
  p.rep_loss[2 * r] = last < 0 ? NAN : __fdiv_rn(s0, n);
  p.rep_loss[2 * r + 1] = last < 0 ? NAN : __fdiv_rn(s1, n);
}

}  // namespace

int cbg_launch_eval_noise(const EvalArgs& a, cudaStream_t st) {
  if (a.b.n_lig <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_STEP_INIT, st);
  eval_noise_kernel<<<(a.b.n_lig + 127) / 128, 128, 0, st>>>(a);
  CBG_LAUNCHED(CBG_K_STEP_INIT, st);
  return 0;
}

int cbg_launch_eval_loss(const EvalArgs& a, cudaStream_t st) {
  if (a.b.n_graphs <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_REVERSE, st);
  eval_loss_kernel<<<a.b.n_graphs, kGraphThreads, 0, st>>>(a);
  CBG_LAUNCHED(CBG_K_REVERSE, st);
  CBG_PROF_BEGIN(CBG_K_REVERSE, st);
  eval_reduce_kernel<<<(a.n_rep + 63) / 64, 64, 0, st>>>(a);
  CBG_LAUNCHED(CBG_K_REVERSE, st);
  return 0;
}
