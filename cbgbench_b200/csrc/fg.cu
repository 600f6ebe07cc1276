// D3FG sampling step (`difffg` / `difffg_v2`, repo/models/diffusion/difffg.py:174-246), DESIGN.md section 16.
//
// One call per reverse step t:
//   fg_embed_kernel    ligand rows of the composed arrays from the state: x = xc, o = o_t and
//                      h = ligand_fg_emb(onehot49(argmax c_t)) + ligand_indicator(1)   (context_emb.py:95-128)
//   cbg_ipa_launch     the IPATransformer on the composed graph (csrc/ipa.cu)
//   fg_reverse_kernel  one warp per functional group: CTNVPScheduler.backward_remove_noise (score form,
//                      diffusion_scheduler.py:144-165), RotVPScheduler.backward_remove_noise (:558-574, so3.py:111-146)
//                      and TypeVPScheduler.backward_remove_noise (:367-378); lane k holds class k.
// The protein rows are step-invariant and written once per batch by the host.  No atomics: a step is bit-reproducible.
#include <math.h>
#include "../../include/cbg_b200.h"
#include "cbg_kernels.cuh"

namespace {

__global__ void __launch_bounds__(256) fg_embed_kernel(cbg_fg_plan p, const float* __restrict__ x_t,
                                                       const float* __restrict__ c_t, const float* __restrict__ o_t) {
  const int a = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (a >= p.n_lig) return;
  const int K = p.num_classes, H = p.hidden;
  const int i = p.lig_node[a];
  const float cv = lane < K ? c_t[(size_t)a * K + lane] : -INFINITY;
  const int v = fg_warp_argmax(cv, lane < K ? lane : 1 << 30);
  const float* w = p.fg_emb_t + (size_t)v * H;
  for (int f = lane; f < H; f += 32) p.h[(size_t)i * H + f] = (w[f] + p.fg_emb_b[f]) + p.lig_indicator[f];
  if (lane < 3) {
    p.x[3 * i + lane] = x_t[3 * a + lane];
    p.o[3 * i + lane] = o_t[3 * a + lane];
  }
}

struct FgOut {
  const float* eps_pos;   // [N,3]
  const float* o_pred;    // [N,3]
  const float* logits;    // [N,K]
};

__global__ void __launch_bounds__(256) fg_reverse_kernel(cbg_fg_plan p, cbg_fg_coef cf, FgOut in,
                                                         const float* __restrict__ x_t, const float* __restrict__ c_t,
                                                         const float* __restrict__ o_t, const float* __restrict__ pos_noise,
                                                         const float* __restrict__ rot_draws,
                                                         const float* __restrict__ type_u, float* __restrict__ x_next,
                                                         float* __restrict__ c_next, float* __restrict__ o_next,
                                                         float* __restrict__ theta_out) {
  const int a = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (a >= p.n_lig) return;
  const int K = p.num_classes;
  const int i = p.lig_node[a];
  const bool gen = p.gen_lig[a] != 0;

  // positions: x' = (x + b * (-eps / sqrt(1 - abar))) / sqrt(1 - b) + [t != 0] sqrt(b) n
  if (lane < 3) {
    const float xt = x_t[3 * a + lane];
    const float score = __fdiv_rn(-in.eps_pos[3 * i + lane], cf.pos_sigma);
    float xs = __fdiv_rn(__fadd_rn(xt, __fmul_rn(cf.pos_beta, score)), cf.pos_sqrt_one_minus_beta);
    xs = __fadd_rn(xs, __fmul_rn(cf.pos_noise_scale, pos_noise[3 * a + lane]));
    x_next[3 * a + lane] = gen ? xs : xt;
  }

  // orientation: R' = exp(e) exp(o_pred), e = normalize(axis) * theta (zero at t <= 1)
  if (lane == 0) {
    const float* rd = rot_draws + (size_t)a * 6;
    float e[3] = {0.f, 0.f, 0.f};
    float theta = 0.f;
    if (cf.rot_noise)
      theta = fg_draw_rotation(rd, cf.t, cf.rot_std, cf.rot_gaussian != 0, p.angle_x, p.angle_cdf, p.n_bins, e);
    float E[9], Rp[9], Rn[9], w[3];
    so3vec_to_rotation(e[0], e[1], e[2], E);
    so3vec_to_rotation(in.o_pred[3 * i], in.o_pred[3 * i + 1], in.o_pred[3 * i + 2], Rp);
    mat3_mul(E, Rp, Rn);
    rotation_to_so3vec(Rn, w);
#pragma unroll
    for (int c = 0; c < 3; ++c) o_next[3 * a + c] = gen ? w[c] : o_t[3 * a + c];
    if (theta_out) theta_out[a] = theta;
  }

  // FG type: q(v_{t-1} | v_t, softmax(logits)), Gumbel-max draw; lane k = class k
  const bool on = lane < K;
  const float lg = on ? in.logits[(size_t)i * K + lane] : -INFINITY;
  const float mx = fg_warp_max(lg);
  const float se = warp_sum(on ? expf(lg - mx) : 0.f);
  const float log_c_pred = (lg - mx) - logf(se);
  const float ctv = on ? c_t[(size_t)a * K + lane] : -INFINITY;
  const float logK = logf((float)K);
  const float A = log_add_exp(log_c_pred + cf.log_alphas_cumprod_prev, cf.log_one_minus_alphas_cumprod_prev - logK);
  const float B = log_add_exp(logf(ctv + 1e-8f) + cf.log_alpha, cf.log_one_minus_alpha - logK);
  const float un = on ? A + B : -INFINITY;
  const float m2 = fg_warp_max(un);
  const float lse2 = m2 + logf(warp_sum(on ? expf(un - m2) : 0.f));
  const float u = on ? type_u[(size_t)a * K + lane] : 0.5f;
  const float score = on ? -logf(-logf(u + 1e-30f) + 1e-30f) + (un - lse2) : -INFINITY;
  const int sampled = fg_warp_argmax(score, on ? lane : 1 << 30);
  const int kept = fg_warp_argmax(ctv, on ? lane : 1 << 30);
  const int v = gen ? sampled : kept;
  if (on) c_next[(size_t)a * K + lane] = lane == v ? 1.f : 0.f;
}

}  // namespace

FgRows fg_rows(void* ws, long long n_nodes, int hidden, int K) {
  const size_t n = (size_t)n_nodes;
  char* b = (char*)ws;
  size_t off = align256((size_t)cbg_ipa_workspace_bytes(n_nodes, hidden));
  auto take = [&](size_t nbytes) { float* p = b ? (float*)(b + off) : nullptr; off += align256(nbytes); return p; };
  FgRows r;
  r.eps_pos = take(n * 3 * 4);
  r.o_pred = take(n * 3 * 4);
  r.h_out = take(n * hidden * 4);
  r.r_next = take(n * 9 * 4);
  r.logits = take(n * K * 4);
  r.bytes = off;
  return r;
}

extern "C" {

int64_t cbg_fg_workspace_bytes(int64_t n_nodes, int32_t hidden, int32_t num_classes) {
  return (int64_t)fg_rows(nullptr, n_nodes, hidden, num_classes).bytes;
}

int32_t cbg_fg_step_f32(const cbg_fg_plan* plan, cbg_fg_coef coef, const float* x_t, const float* c_t, const float* o_t,
                        const float* pos_noise, const float* rot_draws, const float* type_u, float* x_next, float* c_next,
                        float* o_next, void* stream) {
  if (!plan) { cbg_set_error("cbg_fg_step_f32: plan is NULL"); return 1; }
  const cbg_fg_plan& p = *plan;
  if (int rc = check_ipa_shape("cbg_fg_step_f32", p.hidden, p.num_classes, p.n_nodes, p.num_blocks, p.num_sublayers, p.k,
                               p.workspace, p.workspace_bytes,
                               cbg_fg_workspace_bytes(p.n_nodes, p.hidden, p.num_classes)))
    return rc;
  if (p.n_lig < 0 || p.n_lig > p.n_nodes) {
    cbg_set_error("cbg_fg_step_f32: n_nodes=%lld n_lig=%d", (long long)p.n_nodes, p.n_lig);
    return 1;
  }
  if (p.n_bins < 2 || coef.t < 0) { cbg_set_error("cbg_fg_step_f32: n_bins=%d t=%d", p.n_bins, coef.t); return 1; }
  if (p.n_lig > 0 && (!x_t || !c_t || !o_t || !pos_noise || !rot_draws || !type_u || !x_next || !c_next || !o_next)) {
    cbg_set_error("cbg_fg_step_f32: NULL state or draw pointer");
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int N = (int)p.n_nodes, H = p.hidden, K = p.num_classes;
  const FgRows rows = fg_rows(p.workspace, p.n_nodes, H, K);
  const int grid = (p.n_lig + 7) / 8;
  if (grid > 0) {
    CBG_PROF_BEGIN(CBG_K_STEP_INIT, st);
    fg_embed_kernel<<<grid, 256, 0, st>>>(p, x_t, c_t, o_t);
    CBG_LAUNCHED(CBG_K_STEP_INIT, st);
  }
  if (int rc = cbg_ipa_launch(p.blob, H, p.num_sublayers, p.num_blocks, K, p.x, p.o, p.h, p.graph_ptr, p.n_graphs,
                              p.max_graph_nodes, p.lig_flag, p.gen_flag, N, p.k, rows.eps_pos, rows.h_out, rows.o_pred,
                              rows.r_next, rows.logits, (char*)p.workspace, st))
    return rc;
  if (grid > 0) {
    CBG_PROF_BEGIN(CBG_K_REVERSE, st);
    fg_reverse_kernel<<<grid, 256, 0, st>>>(p, coef, FgOut{rows.eps_pos, rows.o_pred, rows.logits}, x_t, c_t, o_t,
                                            pos_noise, rot_draws, type_u, x_next, c_next, o_next, nullptr);
    CBG_LAUNCHED(CBG_K_REVERSE, st);
  }
  return 0;
}

int32_t cbg_fg_reverse_f32(const cbg_fg_plan* plan, cbg_fg_coef coef, const float* eps_pos, const float* o_pred,
                           const float* logits, const float* x_t, const float* c_t, const float* o_t, const float* pos_noise,
                           const float* rot_draws, const float* type_u, float* x_next, float* c_next, float* o_next,
                           float* theta, void* stream) {
  if (!plan) { cbg_set_error("cbg_fg_reverse_f32: plan is NULL"); return 1; }
  const cbg_fg_plan& p = *plan;
  if (p.num_classes < 1 || p.num_classes > CBG_IPA_MAXCLS) {
    cbg_set_error("cbg_fg_reverse_f32: num_classes=%d outside [1,%d]", p.num_classes, CBG_IPA_MAXCLS);
    return 1;
  }
  if (p.n_lig < 0 || p.n_bins < 2 || coef.t < 0) {
    cbg_set_error("cbg_fg_reverse_f32: n_lig=%d n_bins=%d t=%d", p.n_lig, p.n_bins, coef.t);
    return 1;
  }
  if (p.n_lig == 0) return 0;
  if (!p.lig_node || !p.gen_lig || !p.angle_x || !p.angle_cdf) {
    cbg_set_error("cbg_fg_reverse_f32: NULL lig_node / gen_lig / angle_x / angle_cdf in the plan");
    return 1;
  }
  if (!eps_pos || !o_pred || !logits || !x_t || !c_t || !o_t || !pos_noise || !rot_draws || !type_u || !x_next ||
      !c_next || !o_next) {
    cbg_set_error("cbg_fg_reverse_f32: NULL row, state or draw pointer");
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  CBG_PROF_BEGIN(CBG_K_REVERSE, st);
  fg_reverse_kernel<<<(p.n_lig + 7) / 8, 256, 0, st>>>(p, coef, FgOut{eps_pos, o_pred, logits}, x_t, c_t, o_t, pos_noise,
                                                      rot_draws, type_u, x_next, c_next, o_next, theta);
  CBG_LAUNCHED(CBG_K_REVERSE, st);
  return 0;
}

}  // extern "C"
