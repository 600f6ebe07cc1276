// DiffBP validation loss (DiffBP.forward with self.training == False, diffbp.py:133-230) on a plan whose graphs are R
// replicas of one batch, replica r noised at its own timestep t_r:
//   bp_eval_noise_kernel   forward noising of positions with the RAW normal draw (CTNVPScheduler.forward_add_noise with
//                          zero_center=True, diffusion_scheduler.py:117-134) and the absorbing-state type mask
//                          (MaskTypeSchedule.forward_add_noise, :452-472), plus the ligand rows of the node state
//   bp_eval_loss_kernel    per (replica, graph): zero-centred noise target and its graph mean (the CoM target), the
//                          CoM head's eps_pred / com_pred, the position and CoM score losses (get_score_loss, :203-219),
//                          the masked-type cross-entropy of softmax(logits) (get_loss, :500-511), the posterior mean
//                          xs_mean (xs_mean, :167-182) and the interior loss of the graph's ligand atoms
//                          (interior_loss, diffbp.py:19-30: protein -> ligand kNN with k = 48)
//   bp_eval_reduce_kernel  per replica: scatter_mean(...).mean() sizing of the three graph losses, flat mean of the
//                          interior loss
// No atomics: repeated runs are bit-identical.
#include <math.h>
#include "cbg_kernels.cuh"

namespace {

__global__ void __launch_bounds__(128) bp_eval_noise_kernel(BpEvalArgs p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;      // replicated ligand atom
  if (i >= p.b.n_lig) return;
  const int n1 = p.b.n_lig / p.n_rep;
  const int r = i / n1, a = i - r * n1;
  const cbg_bp_eval_coef cf = p.coef.c[r];
  const bool gen = p.b.gen[i] != 0;
  // positions: x_t = sqrt(a) * x0 + sqrt(1 - a) * eps with the raw eps (the zero-centred one is only the target)
  const float sa = __fsqrt_rn(cf.alphas_cumprod), s1 = __fsqrt_rn(__fsub_rn(1.f, cf.alphas_cumprod));
  float xt[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float x0 = p.b.x0[3 * a + c];
    xt[c] = gen ? __fadd_rn(__fmul_rn(sa, x0), __fmul_rn(s1, p.pos_noise[3 * (size_t)i + c])) : x0;
    p.xt[3 * (size_t)i + c] = xt[c];
  }
  // types: generated atoms drawn below t / T go to the absorbing state 0
  const bool mask = gen && p.type_u[i] < cf.mask_prob;
  const int vt = mask ? 0 : (int)p.b.v0[a];
  p.vt[i] = vt;
  p.mask[i] = mask ? 1 : 0;
  store_noised_ligand(p.b, i, xt, vt);
}

// the kNN distance of oracle.graph_ops.pairwise_sqdist_f32: centre (protein) minus point, individually rounded
__device__ __forceinline__ float sqdist(const float4 c, const float4 x) {
  const float dx = __fsub_rn(c.x, x.x), dy = __fsub_rn(c.y, x.y), dz = __fsub_rn(c.z, x.z);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__global__ void __launch_bounds__(kGraphThreads) bp_eval_loss_kernel(BpEvalArgs p) {
  __shared__ float s_red9[kGraphWarps][9];
  __shared__ float s_red5[kGraphWarps][5];
  __shared__ float s_red1[kGraphWarps][1];
  __shared__ float s_mean[9], s_tot[5], s_inter[1];
  const int g = blockIdx.x;                                  // replicated graph
  const int r = g / (p.b.n_graphs / p.n_rep);
  const int2 rng = graph_ligand_range(p.b.lig_node, p.b.n_lig, p.b.graph_ptr, g);
  const int lo = rng.x, hi = rng.y, n_g = hi - lo;
  const int n1 = p.b.n_lig / p.n_rep;
  const cbg_bp_eval_coef cf = p.coef.c[r];
  const int K = p.b.num_classes;
  // ---- graph means over ALL ligand atoms: raw noise, denoiser shift x_pred - x_t, CoM-head shift x_com - x_t
  {
    float s[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
      const float4 xc = p.b.x4[p.b.lig_node[i]];
      const float com[3] = {xc.x, xc.y, xc.z};
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float xt = p.xt[3 * (size_t)i + c];
        s[c] += p.pos_noise[3 * (size_t)i + c];
        s[3 + c] += __fsub_rn(p.x_pred[3 * (size_t)i + c], xt);
        s[6 + c] += __fsub_rn(com[c], xt);
      }
    }
    block_sum<9>(s, s_red9, s_mean);
    if (threadIdx.x < 9) s_mean[threadIdx.x] = __fdiv_rn(s_mean[threadIdx.x], (float)(n_g > 0 ? n_g : 1));
    __syncthreads();
  }
  // ---- per atom: targets / predictions, score losses, masked-type cross-entropy, xs_mean
  const float sigma = __fsqrt_rn(__fsub_rn(1.f, cf.alphas_cumprod));
  const float denom = __fsqrt_rn(__fsub_rn(1.f, cf.beta));
  float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};                 // pos, com, atom, generated count, masked count
  for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const int a = i - r * n1;
    const bool gen = p.b.gen[i] != 0;
    float* vec = p.vec + ((size_t)r * 8 * n1 + a) * 3;
    const size_t q = (size_t)n1 * 3;                         // stride between the eight vector outputs
    float dp = 0.f, dc = 0.f, xs[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float xt = p.xt[3 * (size_t)i + c];
      const float e0 = __fsub_rn(p.pos_noise[3 * (size_t)i + c], s_mean[c]);
      const float ep = __fsub_rn(__fsub_rn(p.x_pred[3 * (size_t)i + c], xt), s_mean[3 + c]);
      const float c0 = s_mean[c], cp = s_mean[6 + c];
      vec[c] = e0; vec[q + c] = ep; vec[2 * q + c] = __fmul_rn(e0, sigma); vec[3 * q + c] = __fmul_rn(ep, sigma);
      vec[4 * q + c] = c0; vec[5 * q + c] = cp; vec[6 * q + c] = __fmul_rn(c0, sigma); vec[7 * q + c] = __fmul_rn(cp, sigma);
      const float d0 = __fsub_rn(ep, e0), d1 = __fsub_rn(cp, c0);
      dp = c == 0 ? __fmul_rn(d0, d0) : __fadd_rn(dp, __fmul_rn(d0, d0));
      dc = c == 0 ? __fmul_rn(d1, d1) : __fadd_rn(dc, __fmul_rn(d1, d1));
      const float score = -__fdiv_rn(__fadd_rn(ep, cp), sigma);
      xs[c] = gen ? __fdiv_rn(__fadd_rn(xt, __fmul_rn(cf.beta, score)), denom) : xt;
    }
    p.xs[i] = make_float4(xs[0], xs[1], xs[2], 0.f);
    if (gen) { acc[0] += dp; acc[1] += dc; acc[3] += 1.f; }
    // c_pred = softmax(logits); the loss is cross_entropy(c_pred, v0), i.e. a second log-softmax on the probabilities
    const float* lg = p.logits + (size_t)i * K;
    float mx = -INFINITY;
    for (int c = 0; c < K; ++c) mx = fmaxf(mx, lg[c]);
    float se = 0.f;
    for (int c = 0; c < K; ++c) se += expf(lg[c] - mx);
    float m2 = -INFINITY, pv0 = 0.f;
    const int v0 = (int)p.b.v0[a];
    for (int c = 0; c < K; ++c) {
      const float pr = __fdiv_rn(expf(lg[c] - mx), se);
      p.c_pred[(size_t)i * K + c] = pr;
      m2 = fmaxf(m2, pr);
      if (c == v0) pv0 = pr;
    }
    if (p.mask[i]) {
      float s2 = 0.f;
      for (int c = 0; c < K; ++c) s2 += expf(p.c_pred[(size_t)i * K + c] - m2);
      acc[2] += -__fsub_rn(__fsub_rn(pv0, m2), logf(s2));
      acc[4] += 1.f;
    }
  }
  block_sum<5>(acc, s_red5, s_tot);          // its barriers also publish p.xs to the whole CTA
  // ---- interior loss: protein atoms of the graph are its first nodes (compose_context puts them before the ligand)
  const int pb = p.b.graph_ptr[g], pe = p.b.graph_ptr[g + 1] - n_g;
  const bool select = n_g > CBG_BP_INTER_K;
  if (select) {
    // per protein atom, one warp: the 48th smallest (d^2, ligand index) pair; the bits of a non-negative float order
    // like the float, so a bitwise radix select finds the 48th smallest d^2, then the tie at that d^2 is cut by index
    const int lane = threadIdx.x & 31;
    for (int pn = pb + (threadIdx.x >> 5); pn < pe; pn += kGraphWarps) {
      const float4 xp = p.b.x4[pn];
      unsigned prefix = 0u;
      for (int bit = 31; bit >= 0; --bit) {
        const unsigned cand = prefix | (1u << bit);
        int cnt = 0;
        for (int j = lo + lane; j < hi; j += 32) cnt += __float_as_uint(sqdist(xp, p.xs[j])) < cand ? 1 : 0;
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        if (cnt <= CBG_BP_INTER_K - 1) prefix = cand;
      }
      int below = 0;
      for (int j = lo + lane; j < hi; j += 32) below += __float_as_uint(sqdist(xp, p.xs[j])) < prefix ? 1 : 0;
      int need = CBG_BP_INTER_K - __reduce_add_sync(0xffffffffu, below);      // >= 1 atoms at d^2 == prefix
      int jt = hi - 1;
      for (int j0 = lo; j0 < hi; j0 += 32) {
        const int j = j0 + lane;
        const unsigned eq = __ballot_sync(0xffffffffu, j < hi && __float_as_uint(sqdist(xp, p.xs[j])) == prefix);
        const int n_eq = __popc(eq);
        if (n_eq >= need) {
          unsigned m = eq;
          for (int s = 1; s < need; ++s) m &= m - 1;           // drop the need-1 lowest set bits
          jt = j0 + __ffs(m) - 1;
          break;
        }
        need -= n_eq;
      }
      if (lane == 0) p.thr[pn] = make_int2((int)prefix, jt);
    }
    __syncthreads();
  }
  float inter = 0.f;
  for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const float4 xl = p.xs[i];
    float s = 0.f;                                           // protein terms in protein-index order
    for (int pn = pb; pn < pe; ++pn) {
      const float d2 = sqdist(p.b.x4[pn], xl);
      if (select) {
        const int2 t = p.thr[pn];
        const unsigned b = __float_as_uint(d2);
        if (b > (unsigned)t.x || (b == (unsigned)t.x && i > t.y)) continue;
      }
      s += expf(__fmul_rn(d2, -0.5f));
    }
    const float lpl = __fmul_rn(-2.f, logf(__fadd_rn(s, 1e-3f)));
    inter += fmaxf(__fsub_rn(5.f, lpl), 0.f);
  }
  float iv[1] = {inter};
  block_sum<1>(iv, s_red1, s_inter);
  if (threadIdx.x == 0) {
    const float ng = fmaxf(s_tot[3], 1.f), nm = fmaxf(s_tot[4], 1.f);       // scatter_mean: sum / max(count, 1)
    float* o = p.graph_part + 8 * (size_t)g;
    o[0] = __fdiv_rn(s_tot[0], ng); o[1] = __fdiv_rn(s_tot[1], ng); o[2] = __fdiv_rn(s_tot[2], nm);
    o[3] = s_inter[0]; o[4] = s_tot[3]; o[5] = s_tot[4];
  }
}

// one thread per replica.  pos / com: scatter_mean over the generated atoms has (last generated graph id + 1) rows,
// graphs without one count as 0 below that id; no generated atom at all gives NaN.  atom: the same over the masked
// atoms, but no masked atom gives 0 (the reference's len(loss) == 0 branch).  inter: flat mean over all ligand atoms.
__global__ void bp_eval_reduce_kernel(BpEvalArgs p) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.n_rep) return;
  const int B = p.b.n_graphs / p.n_rep;
  const float* gp = p.graph_part + 8 * (size_t)r * B;
  int last_g = -1, last_m = -1;
  for (int g = 0; g < B; ++g) {
    if (gp[8 * g + 4] > 0.f) last_g = g;
    if (gp[8 * g + 5] > 0.f) last_m = g;
  }
  float sp = 0.f, sc = 0.f, sa = 0.f, si = 0.f;
  for (int g = 0; g <= last_g; ++g) { sp += gp[8 * g]; sc += gp[8 * g + 1]; }
  for (int g = 0; g <= last_m; ++g) sa += gp[8 * g + 2];
  for (int g = 0; g < B; ++g) si += gp[8 * g + 3];
  p.rep_loss[4 * r + 0] = last_g < 0 ? NAN : __fdiv_rn(sp, (float)(last_g + 1));
  p.rep_loss[4 * r + 1] = last_m < 0 ? 0.f : __fdiv_rn(sa, (float)(last_m + 1));
  p.rep_loss[4 * r + 2] = last_g < 0 ? NAN : __fdiv_rn(sc, (float)(last_g + 1));
  p.rep_loss[4 * r + 3] = __fdiv_rn(si, (float)(p.b.n_lig / p.n_rep));
}

}  // namespace

int cbg_launch_bp_eval_noise(const BpEvalArgs& a, cudaStream_t st) {
  if (a.b.n_lig <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_STEP_INIT, st);
  bp_eval_noise_kernel<<<(a.b.n_lig + 127) / 128, 128, 0, st>>>(a);
  CBG_LAUNCHED(CBG_K_STEP_INIT, st);
  return 0;
}

int cbg_launch_bp_eval_loss(const BpEvalArgs& a, cudaStream_t st) {
  if (a.b.n_graphs <= 0) return 0;
  CBG_PROF_BEGIN(CBG_K_REVERSE, st);
  bp_eval_loss_kernel<<<a.b.n_graphs, kGraphThreads, 0, st>>>(a);
  CBG_LAUNCHED(CBG_K_REVERSE, st);
  CBG_PROF_BEGIN(CBG_K_REVERSE, st);
  bp_eval_reduce_kernel<<<(a.n_rep + 63) / 64, 64, 0, st>>>(a);
  CBG_LAUNCHED(CBG_K_REVERSE, st);
  return 0;
}
