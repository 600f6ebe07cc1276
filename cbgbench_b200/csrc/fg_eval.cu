// D3FG validation loss (`difffg` / `difffg_v2` forward in eval mode, repo/models/diffusion/difffg.py:65-171 / :283-389),
// DESIGN.md section 17, on a plan whose graphs are R replicas of one batch, replica r noised at its own timestep t_r:
//   fg_eval_noise_kernel   one warp per (replica, FG): forward noising of the position, the orientation and the FG type,
//                          written to the outputs and to the ligand rows of the composed x / o / h
//   cbg_ipa_launch         the IPATransformer over all R * B graphs (csrc/ipa.cu)
//   fg_eval_loss_kernel    one CTA per (replica, graph), one warp per FG (lane k = class k): the position, rotation and
//                          type terms of the generated FGs, summed in a fixed order, plus the result vectors
//   fg_eval_reduce_kernel  one thread per replica: scatter_mean(...).mean() over graphs 0 .. (last graph with a generated FG)
// No atomics: repeated calls are bit-identical.
#include <math.h>
#include "../../include/cbg_b200.h"
#include "cbg_kernels.cuh"

namespace {

struct FgEvalArgs {
  cbg_fg_plan p;
  CoefArray<cbg_fg_eval_coef, CBG_EVAL_MAX_REPLICAS> coef;
  int n_rep, loss_form;
  const float* x0;           // [n1,3]
  const long long* v0;       // [n1]
  const float* o0;           // [n1,3]
  const float* pos_noise;    // [n_lig,3]
  const float* rot_draws;    // [n_lig,6]
  const float* type_u;       // [n_lig,K]
  const float* eps_pos;      // [N,3] encoder rows (loss kernel)
  const float* r_next;       // [N,9]
  const float* logits;       // [N,K]
  float* xt;                 // [n_lig,3]
  float* ot;                 // [n_lig,3] or NULL
  long long* vt;             // [n_lig]
  float* pred;               // [n_lig,3]
  float* score;              // [n_rep,2,n1,3] or NULL
  float* c_pred;             // [n_lig,K]
  float* R_pred;             // [n_lig,9]
  float* R0;                 // [n1,9]
  float* graph_loss;         // [n_graphs,4]
  float* rep_loss;           // [n_rep,3]
};

__global__ void __launch_bounds__(256) fg_eval_noise_kernel(FgEvalArgs A) {
  const cbg_fg_plan& p = A.p;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;   // replicated FG
  if (i >= p.n_lig) return;
  const int n1 = p.n_lig / A.n_rep;
  const int r = i / n1, a = i - r * n1;
  const cbg_fg_eval_coef& cf = A.coef.c[r];
  const int K = p.num_classes, H = p.hidden;
  const int node = p.lig_node[i];
  const bool gen = p.gen_lig[i] != 0;

  // positions: x_t = sqrt(abar) * x0 + sqrt(1 - abar) * eps   (two separately rounded products and one add)
  if (lane < 3) {
    const float x0 = A.x0[3 * a + lane];
    const float x = gen ? __fadd_rn(__fmul_rn(cf.pos_sqrt_alphas_cumprod, x0),
                                    __fmul_rn(cf.pos_sqrt_one_minus_alphas_cumprod, A.pos_noise[3 * (size_t)i + lane]))
                        : x0;
    A.xt[3 * (size_t)i + lane] = x;
    p.x[3 * (size_t)node + lane] = x;
  }

  // orientation: o_t = log(exp(e) exp(sqrt(abar_rot) o0)), e drawn from angular_distrib_fwd at t (no zeroing at t <= 1)
  if (lane == 0) {
    float e[3], E[9], R0s[9], Rn[9], w[3];
    fg_draw_rotation(A.rot_draws + 6 * (size_t)i, cf.t, cf.rot_std, cf.rot_gaussian != 0, p.angle_x, p.angle_cdf,
                     p.n_bins, e);
    const float* o0 = A.o0 + 3 * a;
    so3vec_to_rotation(e[0], e[1], e[2], E);
    so3vec_to_rotation(__fmul_rn(cf.rot_sqrt_alphas_cumprod, o0[0]), __fmul_rn(cf.rot_sqrt_alphas_cumprod, o0[1]),
                       __fmul_rn(cf.rot_sqrt_alphas_cumprod, o0[2]), R0s);
    mat3_mul(E, R0s, Rn);
    rotation_to_so3vec(Rn, w);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float o = gen ? w[c] : o0[c];
      if (A.ot) A.ot[3 * (size_t)i + c] = o;
      p.o[3 * (size_t)node + c] = o;
    }
  }

  // FG type: v_t = argmax(Gumbel(u) + log q(v_t | v_0)), log q = log_add_exp(log_c0 + lac[t], l1mac[t] - log K)
  const bool on = lane < K;
  const int v0 = (int)A.v0[a];
  const float logK = (float)log((double)K);
  const float lq = log_add_exp(__fadd_rn(lane == v0 ? 0.f : log_1e30(), cf.log_alphas_cumprod),
                                  __fsub_rn(cf.log_one_minus_alphas_cumprod, logK));
  const float u = on ? A.type_u[(size_t)i * K + lane] : 0.5f;
  const float sc = on ? -logf(-logf(u + 1e-30f) + 1e-30f) + lq : -INFINITY;
  const int arg = fg_warp_argmax(sc, on ? lane : 1 << 30);
  const int v = gen ? arg : v0;
  if (lane == 0) A.vt[i] = v;
  // h = ligand_fg_emb(onehot49(v_t)) + ligand_indicator(1)   (context_emb.py:95-128)
  const float* wv = p.fg_emb_t + (size_t)v * H;
  for (int f = lane; f < H; f += 32) p.h[(size_t)node * H + f] = (wv[f] + p.fg_emb_b[f]) + p.lig_indicator[f];
}

// q_v_posterior (diffusion_scheduler.py:407-418) of class `lane`: log q(v_{t-1} | v_t, v_0) normalised over the lanes;
// lv0 is log v_0 (log one-hot or log-probabilities), vt the noised class.  Lanes >= K return -inf.
__device__ __forceinline__ float fg_q_v_posterior(float lv0, int vt, const cbg_fg_eval_coef& cf, float logK, bool on,
                                                  int lane) {
  const float A = log_add_exp(__fadd_rn(lv0, cf.log_alphas_cumprod_prev),
                                 __fsub_rn(cf.log_one_minus_alphas_cumprod_prev, logK));
  const float B = log_add_exp(__fadd_rn(lane == vt ? 0.f : log_1e30(), cf.log_alpha),
                                 __fsub_rn(cf.log_one_minus_alpha, logK));
  const float un = on ? __fadd_rn(A, B) : -INFINITY;
  const float m = fg_warp_max(un);
  const float lse = m + logf(warp_sum(on ? expf(un - m) : 0.f));
  return on ? __fsub_rn(un, lse) : -INFINITY;
}

// 1 - cos(x, y) of F.cosine_embedding_loss with target 1: sum(xy) / sqrt((sum(x^2) + 1e-12) (sum(y^2) + 1e-12))
__device__ __forceinline__ float fg_one_minus_cos(const float (&x)[3], const float (&y)[3]) {
  const float xy = __fadd_rn(__fadd_rn(__fmul_rn(x[0], y[0]), __fmul_rn(x[1], y[1])), __fmul_rn(x[2], y[2]));
  const float xx = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(x[0], x[0]), __fmul_rn(x[1], x[1])), __fmul_rn(x[2], x[2])), 1e-12f);
  const float yy = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(y[0], y[0]), __fmul_rn(y[1], y[1])), __fmul_rn(y[2], y[2])), 1e-12f);
  return __fsub_rn(1.f, __fdiv_rn(xy, __fsqrt_rn(__fmul_rn(xx, yy))));
}

__global__ void __launch_bounds__(kGraphThreads) fg_eval_loss_kernel(FgEvalArgs A) {
  __shared__ float s_red[kGraphWarps][4], s_tot[4];
  const cbg_fg_plan& p = A.p;
  const int g = blockIdx.x;                                       // replicated graph
  const int B = p.n_graphs / A.n_rep;
  const int r = g / B;
  const int2 rng = graph_ligand_range(p.lig_node, p.n_lig, p.graph_ptr, g);
  const int n1 = p.n_lig / A.n_rep;
  const cbg_fg_eval_coef& cf = A.coef.c[r];
  const int K = p.num_classes;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool on = lane < K;
  const float logK = (float)log((double)K);
  const bool score_form = A.loss_form == CBG_FG_LOSS_SCORE;
  const float sigma = cf.pos_sqrt_one_minus_alphas_cumprod;
  float sum_pos = 0.f, sum_rot = 0.f, sum_fg = 0.f, cnt = 0.f;   // lane 0 of each warp, over the warp's FGs in order
  for (int i = rng.x + warp; i < rng.y; i += kGraphWarps) {
    const int a = i - r * n1;
    const int node = p.lig_node[i];
    const bool gen = p.gen_lig[i] != 0;
    // positions: pred = the encoder's eps_pos; the target is eps (score form) or x0 (denoise form)
    float d2 = 0.f;
    if (lane < 3) {
      const float pr = A.eps_pos[3 * (size_t)node + lane];
      A.pred[3 * (size_t)i + lane] = pr;
      float tgt;
      if (score_form) {
        tgt = A.pos_noise[3 * (size_t)i + lane];
        const size_t s = ((size_t)r * 2 * n1 + a) * 3 + lane;
        A.score[s] = __fmul_rn(tgt, sigma);
        A.score[s + (size_t)n1 * 3] = __fmul_rn(pr, sigma);
      } else {
        tgt = A.x0[3 * a + lane];
      }
      const float d = __fsub_rn(pr, tgt);
      d2 = __fmul_rn(d, d);
    }
    const float d2_1 = __shfl_sync(CBG_FULL, d2, 1), d2_2 = __shfl_sync(CBG_FULL, d2, 2);
    // rotations: R_pred = the encoder's R_next, R0 = exp(o0); sum over the three columns of 1 - cos
    if (lane < 9) A.R_pred[9 * (size_t)i + lane] = A.r_next[9 * (size_t)node + lane];
    float rot = 0.f;
    if (lane == 0) {
      float R0[9], Rp[9];
      so3vec_to_rotation(A.o0[3 * a], A.o0[3 * a + 1], A.o0[3 * a + 2], R0);
      if (r == 0) {
#pragma unroll
        for (int e = 0; e < 9; ++e) A.R0[9 * (size_t)a + e] = R0[e];
      }
#pragma unroll
      for (int e = 0; e < 9; ++e) Rp[e] = A.r_next[9 * (size_t)node + e];
      float l[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const float x[3] = {Rp[j], Rp[3 + j], Rp[6 + j]}, y[3] = {R0[j], R0[3 + j], R0[6 + j]};
        l[j] = fg_one_minus_cos(x, y);
      }
      rot = __fadd_rn(__fadd_rn(l[0], l[1]), l[2]);
    }
    // types: log_softmax of the logits (c_pred = its exp), then KL(q(v_{t-1} | v_t, v_0) || q(v_{t-1} | v_t, c_pred)), or
    // at t == 0 the decoder NLL -sum exp(log_c0) log p
    const float lg = on ? A.logits[(size_t)node * K + lane] : -INFINITY;
    const float mx = fg_warp_max(lg);
    const float se = warp_sum(on ? expf(lg - mx) : 0.f);
    const float lcp = __fsub_rn(__fsub_rn(lg, mx), logf(se));
    if (on) A.c_pred[(size_t)i * K + lane] = expf(lcp);
    const int v0 = (int)A.v0[a], vt = (int)A.vt[i];
    const float lc0 = lane == v0 ? 0.f : log_1e30();
    const float lpt = fg_q_v_posterior(lc0, vt, cf, logK, on, lane);
    const float lpp = fg_q_v_posterior(lcp, vt, cf, logK, on, lane);
    const float kl = warp_sum(on ? __fmul_rn(expf(lpt), __fsub_rn(lpt, lpp)) : 0.f);
    const float nll = -warp_sum(on ? __fmul_rn(expf(lc0), lpp) : 0.f);
    if (lane == 0 && gen) {
      sum_pos += __fadd_rn(__fadd_rn(d2, d2_1), d2_2);
      sum_rot += rot;
      const float mask = cf.t_is_zero ? 1.f : 0.f;
      sum_fg += __fadd_rn(__fmul_rn(mask, nll), __fmul_rn(__fsub_rn(1.f, mask), kl));
      cnt += 1.f;
    }
  }
  float v[4] = {sum_pos, sum_rot, sum_fg, cnt};
  block_sum<4>(v, s_red, s_tot);
  if (threadIdx.x == 0) {
    const float n = fmaxf(s_tot[3], 1.f);                         // scatter_mean: sum / max(count, 1)
#pragma unroll
    for (int c = 0; c < 3; ++c) A.graph_loss[4 * (size_t)g + c] = __fdiv_rn(s_tot[c], n);
    A.graph_loss[4 * (size_t)g + 3] = s_tot[3];
  }
}

// one thread per replica: the output of scatter_mean has max(generated graph id) + 1 rows (graphs without generated FGs
// below that id count as 0); .mean() of no rows is NaN
__global__ void fg_eval_reduce_kernel(FgEvalArgs A) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= A.n_rep) return;
  const int B = A.p.n_graphs / A.n_rep;
  const float* gl = A.graph_loss + 4 * (size_t)r * B;
  int last = -1;
  for (int g = 0; g < B; ++g) if (gl[4 * g + 3] > 0.f) last = g;
  float s[3] = {0.f, 0.f, 0.f};
  for (int g = 0; g <= last; ++g)
    for (int c = 0; c < 3; ++c) s[c] += gl[4 * g + c];
  const float n = (float)(last + 1);
  for (int c = 0; c < 3; ++c) A.rep_loss[3 * r + c] = last < 0 ? NAN : __fdiv_rn(s[c], n);
}

}  // namespace

extern "C" int32_t cbg_fg_eval_loss_f32(const cbg_fg_plan* plan, const cbg_fg_eval_coef* coefs, int32_t n_rep,
                                        int32_t loss_form, const float* x0, const int64_t* v0, const float* o0,
                                        const float* pos_noise, const float* rot_draws, const float* type_u, float* xt,
                                        float* ot, int64_t* vt, float* pred, float* score, float* c_pred, float* R_pred,
                                        float* R0, float* graph_loss, float* rep_loss, void* stream) {
  if (!plan || !coefs) { cbg_set_error("cbg_fg_eval_loss_f32: plan or coefs is NULL"); return 1; }
  const cbg_fg_plan& p = *plan;
  if (n_rep < 1 || n_rep > CBG_EVAL_MAX_REPLICAS) {
    cbg_set_error("cbg_fg_eval_loss_f32: n_rep=%d outside [1,%d]", n_rep, CBG_EVAL_MAX_REPLICAS);
    return 1;
  }
  if (loss_form != CBG_FG_LOSS_SCORE && loss_form != CBG_FG_LOSS_DENOISE) {
    cbg_set_error("cbg_fg_eval_loss_f32: loss_form=%d (0 score, 1 denoise)", loss_form);
    return 1;
  }
  if (int rc = check_ipa_shape("cbg_fg_eval_loss_f32", p.hidden, p.num_classes, p.n_nodes, p.num_blocks, p.num_sublayers,
                               p.k, p.workspace, p.workspace_bytes,
                               cbg_fg_workspace_bytes(p.n_nodes, p.hidden, p.num_classes)))
    return rc;
  if (p.n_lig < n_rep || p.n_lig > p.n_nodes || p.n_lig % n_rep || p.n_graphs < n_rep || p.n_graphs % n_rep) {
    cbg_set_error("cbg_fg_eval_loss_f32: plan (n_nodes=%lld, n_lig=%d, n_graphs=%d) is not %d replicas of one batch",
                  (long long)p.n_nodes, p.n_lig, p.n_graphs, n_rep);
    return 1;
  }
  if (p.n_bins < 2) { cbg_set_error("cbg_fg_eval_loss_f32: n_bins=%d", p.n_bins); return 1; }
  for (int r = 0; r < n_rep; ++r) {
    if (coefs[r].t < 0) { cbg_set_error("cbg_fg_eval_loss_f32: coefs[%d].t=%d", r, coefs[r].t); return 1; }
  }
  if (!p.blob || !p.graph_ptr || !p.lig_flag || !p.gen_flag || !p.lig_node || !p.gen_lig || !p.x || !p.o || !p.h ||
      !p.fg_emb_t || !p.fg_emb_b || !p.lig_indicator || !p.angle_x || !p.angle_cdf) {
    cbg_set_error("cbg_fg_eval_loss_f32: NULL pointer in the plan");
    return 1;
  }
  if (!x0 || !v0 || !o0 || !pos_noise || !rot_draws || !type_u || !xt || !vt || !pred || !c_pred || !R_pred || !R0 ||
      !graph_loss || !rep_loss || (loss_form == CBG_FG_LOSS_SCORE && !score)) {
    cbg_set_error("cbg_fg_eval_loss_f32: NULL batch, draw or output pointer");
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int N = (int)p.n_nodes, H = p.hidden, K = p.num_classes;
  const FgRows rows = fg_rows(p.workspace, p.n_nodes, H, K);
  FgEvalArgs A;
  A.p = p;
  for (int r = 0; r < n_rep; ++r) A.coef.c[r] = coefs[r];
  A.n_rep = n_rep; A.loss_form = loss_form;
  A.x0 = x0; A.v0 = (const long long*)v0; A.o0 = o0;
  A.pos_noise = pos_noise; A.rot_draws = rot_draws; A.type_u = type_u;
  A.eps_pos = rows.eps_pos; A.r_next = rows.r_next; A.logits = rows.logits;
  A.xt = xt; A.ot = ot; A.vt = (long long*)vt; A.pred = pred; A.score = loss_form == CBG_FG_LOSS_SCORE ? score : nullptr;
  A.c_pred = c_pred; A.R_pred = R_pred; A.R0 = R0; A.graph_loss = graph_loss; A.rep_loss = rep_loss;
  CBG_PROF_BEGIN(CBG_K_STEP_INIT, st);
  fg_eval_noise_kernel<<<(p.n_lig + 7) / 8, 256, 0, st>>>(A);
  CBG_LAUNCHED(CBG_K_STEP_INIT, st);
  if (int rc = cbg_ipa_launch(p.blob, H, p.num_sublayers, p.num_blocks, K, p.x, p.o, p.h, p.graph_ptr, p.n_graphs,
                              p.max_graph_nodes, p.lig_flag, p.gen_flag, N, p.k, rows.eps_pos, rows.h_out, rows.o_pred,
                              rows.r_next, rows.logits, (char*)p.workspace, st))
    return rc;
  CBG_PROF_BEGIN(CBG_K_REVERSE, st);
  fg_eval_loss_kernel<<<p.n_graphs, kGraphThreads, 0, st>>>(A);
  CBG_LAUNCHED(CBG_K_REVERSE, st);
  CBG_PROF_BEGIN(CBG_K_REVERSE, st);
  fg_eval_reduce_kernel<<<(n_rep + 63) / 64, 64, 0, st>>>(A);
  CBG_LAUNCHED(CBG_K_REVERSE, st);
  return 0;
}
