// Internal launcher declarations (one per kernel family).  Not part of the C-ABI.
#pragma once
#include "../../include/cbg_b200.h"
#include "cbg_common.cuh"

#define CBG_MODE_KNN 0
#define CBG_MODE_RADIUS 1

// graph.cu
// static_only != 0: neighbour search restricted to nodes without the generate bit (centres with
// the bit get an empty row) - the static-only kNN lists behind the R-cache
// snbr (optional): static-only lists of the same graphs -> incremental search for non-moving centres
int cbg_launch_knn(const float4* x4, const int* graph_ptr, int n_graphs, int max_graph_nodes, int mode,
                   int k, float r_max, int static_only, const int* snbr, int* nbr, cudaStream_t st);
// ew_static (optional): gates of the static-only neighbour lists, reused for static edges
// glist (optional, with ew_static): scratch of 64 + 32*n_nodes ints; the moving edges are compacted into it
// and their gates computed by a second, dense launch
// full_static (optional, with ew_static): per node, 1 when all 32 slots hold static edges (fast path of edge_setup)
int cbg_launch_edge_gate(const float* blob_global, const float4* x4, const int* nbr, long long n_nodes,
                         const float* ew_static, int* glist, float* ew, cudaStream_t st,
                         unsigned char* full_static = nullptr);

// Receptive-field pruning (sampling path): depth[i] = last layer whose X2H output of node i can still
// influence a generated / classified atom (-2: never).  order[] lists nodes by decreasing depth,
// cnt_ge[l + 1] = number of nodes with depth >= l for l = -1 .. num_layers-1.
int cbg_launch_depth(const int* nbr, const int* graph_ptr, int n_graphs, int max_graph_nodes, long long n_nodes,
                     const int* seed_idx, int n_seed, const int* cls_idx, int n_cls, int num_layers,
                     int* depth, int* order, int* cnt_ge, cudaStream_t st);

// node_gemm.cu
struct NodeGemmArgs {
  const float* a;        // [*,128] input rows (h)
  const int* row_idx;    // optional gather list (node ids); nullptr = identity
  int n_rows;            // rows to process
  const float* wt;       // Wt[k][ldw] (k-major), already offset to the first plane's column
  const float* bias;     // [n_planes*128], already offset
  int ldw;               // row stride of wt in floats
  int n_planes;          // planes computed by this launch (the last one is q_hidden if has_q)
  float* out[CBG_NPLANES];  // destination plane per computed plane ([N,128], indexed by node id)
  int has_q;             // 1: last plane goes LN->ReLU->W1T GEMM -> out_q instead of global
  const float* q_ln;     // gamma[128], beta[128]
  const float* q_w1t;    // [128][128] k-major
  const float* q_b1;     // [128]
  float* out_q;          // [N,128]
  // tensor-core path only: pre-split weight planes of the sub-layer (layout: cbg_layout.h *_NODE_TC)
  const int* n_rows_dev;   // optional: rows to process is min(n_rows, *n_rows_dev) (device-side list length)
  const float* tc_planes;  // plane 0 of the sub-layer
  int tc_first_plane;      // index of this launch's first plane (q second Linear is always plane 5)
  const float* tch_planes; // f16 (hi | lo) images of the same six planes (node_gemm_f16.cu)
  // f16 kernel only: merged launch - planes >= CBG_NODE_SRC_PLANES (destination planes Pi, q) are computed for the first
  // min(n_rows, *n_dst_dev) rows of the list only, the source planes Pj for all n_rows (nullptr = no second limit)
  const int* n_dst_dev;
  long long* trace;        // debug: globaltimer stamps of CTA 0 (cbg_debug_node_gemm_trace)
};
int cbg_launch_node_gemm(const NodeGemmArgs& a, cudaStream_t st);      // fp32 SIMT
// wgmma 3xTF32; cluster = 1/2/4 CTAs sharing weight chunks by multicast, 0 = default (env CBG_GEMM_CLUSTER)
int cbg_launch_node_gemm_tc(const NodeGemmArgs& a, cudaStream_t st, int cluster = 0);
// wgmma f16 with the (hi, lo) split: default
int cbg_launch_node_gemm_f16(const NodeGemmArgs& a, cudaStream_t st);
void cbg_node_gemm_f16_set_trace(long long* buf_dev);

// edge.cu
struct EdgeArgs {
  const float4* x4;      // [N] xyz + flags
  const int* nbr;        // [N,32]
  const float* ew;       // [N,32]
  const float* pj_k;     // planes [N,128]
  const float* pj_v;
  const float* pi_k;
  const float* pi_v;
  const float* q;        // [N,128] (already scaled by 1/sqrt(8))
  const float* layer;    // base of this layer's weight block
  float* w;              // [N,32,16] scratch: alpha * e_w
  float* h;              // [N,128] in/out (x2h_v residual update)
  const int* node_idx;   // h2x: list of generated nodes
  int n_nodes;           // x2h: N ; h2x: number of generated nodes
  float* dx;             // h2x: [n_nodes,4] coordinate deltas (compact, same order as node_idx)
  const int* n_nodes_dev; // optional device-side length of node_idx (x2h with a pruned node list)
  const float* rc_k;     // x2h: R-cache of this layer's hk / hv MLP ([N][32][128]) or nullptr
  const float* rc_v;
  int* ticket;           // x2h: optional work counter (zeroed by the caller) for dynamic node scheduling; k uses ticket[0], v ticket[1]
  const unsigned char* fstat;  // x2h with an R-cache: 1 = all 32 in-edges of the node are static (nbr row == its static list)
  long long* trace;      // x2h_tc debugging: per-tile SM-clock stamps of CTA 0 ([tile][16 event slots]) or nullptr
  int trace_tiles;
  int w_compact;         // x2h_tc: 1 = w is indexed by the position in node_idx ([n_nodes,32,16], H2X), 0 = by node id
};
int cbg_launch_rcache(const float* layers, int num_layers, const float4* x4, const int* snbr, int n_nodes,
                      float* rcache, cudaStream_t st);
int cbg_launch_x2h(const EdgeArgs& a, cudaStream_t st);
// x2h_tc.cu: both X2H kernels on wgmma (activations as register A fragments, f16 hi/lo split); edge order of w = neighbour-table order
int cbg_launch_x2h_tc(const EdgeArgs& a, cudaStream_t st);
// hardware self-test of the wgmma operand conventions (tests): d[128][128] = a[128][32] * b[128][32]^T, f16 inputs
// debugging: x2h_tc kernels of later launches stamp CTA 0's pipeline events into buf ([max_tiles][16] int64; nullptr = off)
void cbg_x2h_tc_set_trace(long long* buf, int max_tiles);
// H2X on the same wgmma kernel (generated nodes only): a.w = compact [n_nodes,32,16] scratch, a.dx = [n_nodes,4] out
int cbg_launch_h2x_tc(const EdgeArgs& a, cudaStream_t st);
int cbg_launch_umma_selftest(const void* a, const void* b, float* d, int a_from_smem, cudaStream_t st);
int cbg_launch_h2x(const EdgeArgs& a, cudaStream_t st);
int cbg_edge_init(void);  // sets max-dynamic-smem attributes once
int cbg_edge_set_impl(int impl, int warps);  // X2H implementation switch (cbg_set_edge_impl)

// misc.cu
int cbg_launch_pack_x4(const float* x, const unsigned char* lig_flag, const unsigned char* gen_flag,
                       long long n, float4* x4, cudaStream_t st);
int cbg_launch_unpack_x(const float4* x4, long long n, float* x, cudaStream_t st);
int cbg_launch_gather_x(const float4* x4, const int* idx, int n, float* out /*[n,3]*/, cudaStream_t st);
int cbg_launch_apply_dx(float4* x4, const int* node_idx, const float* dx, int n, cudaStream_t st);
int cbg_launch_classifier(const float* blob_global, const float* h, const int* row_idx, int n_rows,
                          int num_classes, float* logits, cudaStream_t st);
int cbg_launch_step_init(const float* x_lig, const float* c_lig, const int* lig_node, int n_lig,
                         int num_classes, const float* emb_wt, const float* h_lig_bias,
                         const float* h_static, long long n_nodes, float4* x4, float* h, cudaStream_t st);
struct ReverseArgs {
  const float* x0;         // denoiser output coordinates (x0 prediction), row stride x0_stride floats
  int x0_stride;           // 4 when reading the packed node array, 3 for a plain [n,3] tensor
  const int* x0_idx;       // optional row index per ligand atom (lig_node); nullptr = identity
  const float* logits;     // [n_lig, K]
  const float* x_t;        // [n_lig,3]
  const float* c_t;        // [n_lig,K]
  const unsigned char* gen;  // [n_lig]
  const float* pos_noise;  // [n_lig,3]
  const float* type_u;     // [n_lig,K]
  float c0, ct;            // posterior_mean_c0_coef[t], posterior_mean_ct_coef[t]
  float lac_prev, l1mac_prev, la, l1ma;  // type tables at t-1 (clamped) and t
  int n_lig, num_classes;
  float* x_next;           // [n_lig,3]
  float* c_next;           // [n_lig,K]
  long long* v_next;       // [n_lig]
};
// logvar = posterior_logvar[t]; nonzero = 0 at t == 0 else 1
int cbg_launch_reverse(const ReverseArgs& a, float logvar, float nonzero, cudaStream_t st);

// Per-step inputs / outputs of the TargetDiff step in DEVICE memory: what changes from step to step when the step is
// replayed from a CUDA graph (cbg_sample_step_graph_f32): the graph's kernels read these through one pointer.
struct StepIO {
  const float* x_t;
  const float* c_t;
  const float* pos_noise;
  const float* type_u;
  float* x_next;
  float* c_next;
  long long* v_next;
  float c0, ct, lac_prev, l1mac_prev, la, l1ma, logvar, nonzero;
};
int cbg_launch_step_init_io(const StepIO* io, const int* lig_node, int n_lig, int num_classes, const float* emb_wt,
                            const float* h_lig_bias, const float* h_static, long long n_nodes, float4* x4, float* h,
                            cudaStream_t st);
// the step-invariant members of `a` are used, the per-step ones (x_t, c_t, noise, outputs, coefficients) come from *io
int cbg_launch_reverse_io(const ReverseArgs& a, const StepIO* io, cudaStream_t st);

// Validation losses (eval.cu, bp_eval.cu, sbdd_eval.cu, fg_eval.cu).  The plan's ligand atoms and graphs are R replicas
// of one batch, replica-major: atom i belongs to replica i / n1 and is atom i % n1 of the batch (n1 = n_lig / R).
constexpr int CBG_EVAL_MAX_REPLICAS = 64;
// the per-replica coefficients (the public cbg_*_eval_coef structs), passed by value in the kernel arguments: no H2D
// copy per call
template <class C, int N> struct CoefArray { C c[N]; };
// the batch block of the three argument structs (api.cu: open_eval fills it)
struct EvalBatch {
  int n_lig, n_graphs, num_classes;   // n_lig / n_graphs: replicated totals
  const int* lig_node;       // [n_lig] ascending composed node index
  const int* graph_ptr;      // [n_graphs+1]
  const unsigned char* gen;  // [n_lig] replicated ligand_gen_flag
  const float* x0;           // [n1,3] the batch's ligand_pos
  const long long* v0;       // [n1]
  const float* emb_wt;       // [K,128]
  const float* h_lig_bias;   // [n_lig,128]
  float4* x4;                // node coordinates + flags
  float* h;                  // [N,128] node features
};
// replicated ligand atom i noised to (xt, vt) in the denoiser's node state: its coordinates (flags kept) and
// h = (b_atom + indicator) + W_atom one_hot(vt)
__device__ __forceinline__ void store_noised_ligand(const EvalBatch& b, int i, const float (&xt)[3], int vt) {
  const int node = b.lig_node[i];
  float4 v = b.x4[node];
  v.x = xt[0]; v.y = xt[1]; v.z = xt[2];
  b.x4[node] = v;
  const float* bias = b.h_lig_bias + (size_t)i * CBG_H;
  const float* w = b.emb_wt + (size_t)vt * CBG_H;
  float* h = b.h + (size_t)node * CBG_H;
  for (int k = 0; k < CBG_H; k += 4) st4(h + k, add4(ldg4(bias + k), ldg4(w + k)));
}

// eval.cu: TargetDiff validation loss over R = n_rep replicas of a batch (cbg_eval_loss_f32)
struct EvalArgs {
  CoefArray<cbg_eval_coef, CBG_EVAL_MAX_REPLICAS> coef;
  int n_rep;
  EvalBatch b;
  const float* pos_noise;    // [n_lig,3]
  const float* type_u;       // [n_lig,K]
  const float* logits;       // [n_lig,K] classifier output (loss kernel)
  float* xt;                 // [n_lig,3]
  long long* vt;             // [n_lig]
  float* x_pred;             // [n_lig,3]
  float* c_pred;             // [n_lig,K]
  float* graph_loss;         // [n_graphs,2] per-graph (pos, atom) means over generated atoms (0 without any)
  int* graph_cnt;            // [n_graphs] generated atoms per graph (scratch)
  float* rep_loss;           // [n_rep,2]
};
int cbg_launch_eval_noise(const EvalArgs& a, cudaStream_t st);
// eval_loss_kernel (one CTA per graph) followed by eval_reduce_kernel (one thread per replica)
int cbg_launch_eval_loss(const EvalArgs& a, cudaStream_t st);

// DiffSBDD reverse step (SURVEY.md section 8 row f2): one CTA per graph.
//   mode 0  zs = z_t / a - b * eps_pred + s * noise              (sample_p_zs_given_zt, diffusion_scheduler.py:1005-1039)
//   mode 1  zs = a * (z_t - b * eps_pred) + s * noise            (sample_p_xh_given_z0, diffsbdd.py:323-360; a = 1/alpha_0)
// for the coordinates (eps_pred = the denoiser's output coordinates of the ligand atoms, read from x4) followed by
// the COM projection remove_mean_batch (diffusion_scheduler.py:706-710): the mean of zs over the graph's ligand
// atoms is subtracted from zs AND from the pocket atoms of the graph (x4 rows without the ligand bit).
// Types: mode 0 the same update without projection (eps_pred = logits), mode 1 c_next = 4 * c_t.
struct SbddArgs {
  float4* x4;               // [N] node coordinates + flags (pocket rows are shifted in place)
  const int* graph_ptr;     // [B+1]
  const int* lig_node;      // [n_lig] ascending composed index of every ligand atom
  int n_lig, num_classes, n_graphs;
  const float* logits;      // [n_lig,K]
  const float* x_t;         // [n_lig,3]
  const float* c_t;         // [n_lig,K]
  const float* x_noise;     // [n_lig,3]
  const float* c_noise;     // [n_lig,K]
  float a, b, s;
  int mode;
  float* x_next;            // [n_lig,3]
  float* c_next;            // [n_lig,K]
};
int cbg_launch_sbdd_reverse(const SbddArgs& a, cudaStream_t st);

// DiffBP (row f2).  x4[idx[a]].xyz = x[a] (flags kept): puts the step's INPUT ligand coordinates back before the
// CoM head runs on them (diffbp.py:80-97 works on x_composed, not on the denoiser's output)
int cbg_launch_scatter_x(const float* x /*[n,3]*/, const int* idx, int n, float4* x4, cudaStream_t st);
// edge gate of the listed rows only (the CoM head needs it for the generated atoms' edges)
int cbg_launch_edge_gate_rows(const float* blob_global, const float4* x4, const int* nbr, const int* row_idx,
                              int n_rows, float* ew, cudaStream_t st);
// Fused DiffBP reverse step, one CTA per graph:
//   eps  = (x_pred - x_t) - mean_g(x_pred - x_t) + mean_g(x_com - x_t)          CoMPredictor.forward diffbp.py:80-101
//   x_s  = (x_t + beta * (-eps / sqrt(1 - abar))) / sqrt(1 - beta) + nonzero * sqrt(beta) * noise, gen-masked
//                                                  CTNVPScheduler.backward_remove_noise('score') diffusion_scheduler.py:144-165
//   v_s  = (u < prob) & gen & (v_t == 0) ? argmax softmax(logits) : v_t   MaskTypeSchedule.backward_remove_noise :474-498
struct BpArgs {
  const float4* x4;         // ligand rows hold x_com (output of the CoM head's H2X stack)
  const int* graph_ptr;
  const int* lig_node;
  int n_lig, num_classes, n_graphs;
  const float* x_pred;      // [n_lig,3] denoiser output coordinates
  const float* logits;      // [n_lig,K]
  const float* x_t;         // [n_lig,3]
  const float* c_t;         // [n_lig,K]
  const unsigned char* gen; // [n_lig]
  const float* pos_noise;   // [n_lig,3]
  const float* type_u;      // [n_lig]
  float abar, beta, nonzero, prob;
  float* x_next;            // [n_lig,3]
  float* c_next;            // [n_lig,K]
  long long* v_next;        // [n_lig]
  float* eps_out;           // optional [n_lig,3]
};
int cbg_launch_bp_reverse(const BpArgs& a, cudaStream_t st);

// bp_eval.cu: DiffBP validation loss over R = n_rep replicas of a batch (cbg_bp_eval_loss_f32).  After the CoM head
// the ligand rows of x4 hold x_com.
constexpr int CBG_BP_INTER_K = 48;       // interior loss: protein -> ligand kNN (diffbp.py:19)
struct BpEvalArgs {
  CoefArray<cbg_bp_eval_coef, CBG_EVAL_MAX_REPLICAS> coef;
  int n_rep;
  EvalBatch b;
  const float* pos_noise;    // [n_lig,3] raw normal draws
  const float* type_u;       // [n_lig] uniform draws of the type mask
  const float* logits;       // [n_lig,K] classifier output
  const float* x_pred;       // [n_lig,3] denoiser output coordinates
  float* xt;                 // [n_lig,3]
  long long* vt;             // [n_lig]
  unsigned char* mask;       // [n_lig] type mask
  float* vec;                // [n_rep, 8, n_lig/n_rep, 3]: eps_0, eps_pred, score_0, score_pred, then the _com four
  float* c_pred;             // [n_lig,K]
  float4* xs;                // [n_lig] scratch: posterior mean of x_{t-1} (interior loss)
  int2* thr;                 // [N] scratch: per protein node, (d^2 bits, ligand index) of its 48th nearest ligand atom
  float* graph_part;         // [n_graphs,8] scratch: per-graph means / counts / interior-loss sum
  float* rep_loss;           // [n_rep,4]: pos, atom, com, inter
};
int cbg_launch_bp_eval_noise(const BpEvalArgs& a, cudaStream_t st);
// bp_eval_loss_kernel (one CTA per graph) followed by bp_eval_reduce_kernel (one thread per replica)
int cbg_launch_bp_eval_loss(const BpEvalArgs& a, cudaStream_t st);

// sbdd_eval.cu: DiffSBDD validation loss over n_t timesteps of a batch (cbg_sbdd_eval_loss_f32).  The plan holds R = 2 n_t
// replicas: replica 2j is timestep j noised at t_j, replica 2j+1 timestep j noised at 0.  After the denoiser the ligand
// rows of x4 hold x_pred.
struct SbddEvalArgs {
  CoefArray<cbg_sbdd_eval_coef, CBG_EVAL_MAX_REPLICAS / 2> coef;
  int n_t;
  long long n_nodes;
  EvalBatch b;
  const float* x_rec;        // [n_rec1,3] the batch's protein_pos
  const float* x_t_noise;    // [n_t,n1,3] / [n_t,n1,K] / [n_t,n1,3] / [n_t,n1,K]: the four draws of each timestep
  const float* c_t_noise;
  const float* x_0_noise;
  const float* c_0_noise;
  const float* logits;       // [n_lig,K] classifier output
  float* vec_pos;            // [n_t,3,n1,3]: eps_pred, score_0, score_pred of the positions
  float* vec_atom;           // [n_t,3,n1,K]: the same of the types
  float* terms;              // [n_t,B,6]: pos_t, pos_0, pos_kl, atom_t, atom_0, atom_kl per graph of the batch
  float* t_loss;             // [n_t,2]: pos, atom
};
int cbg_launch_sbdd_eval_noise(const SbddEvalArgs& a, cudaStream_t st);
// sbdd_eval_loss_kernel (one CTA per (timestep, graph)) followed by sbdd_eval_reduce_kernel (one thread per timestep)
int cbg_launch_sbdd_eval_loss(const SbddEvalArgs& a, cudaStream_t st);

// batch.cu (row f3: device-side batch construction)
int cbg_launch_pocket_stats(const float* prot_pos, const int* prot_ptr, int n_pockets, const float* ctx_pos,
                            const int* ctx_ptr, int centre_mode, float* space_size, float* centre, cudaStream_t st);
int cbg_launch_ligand_sizes(const double* bounds, int n_bounds, const int* bin_ptr, const int* values, const double* cdf,
                            const float* space_size, int n_pockets, int repeat, const double* u, const int* ctx_ptr,
                            const int* extra, int* n_lig, int* lig_ptr, cudaStream_t st);
int cbg_launch_build_batch(const float* prot_pos, const int* prot_element, const unsigned char* prot_backbone,
                           const int* prot_aa, const int* prot_ptr, int n_pockets, int repeat, const float* centre,
                           const float* ctx_pos, const int* ctx_type, const int* ctx_ptr, const int* lig_ptr,
                           const float* pos_noise, const float* type_u, int num_classes, int type_dist, int pos_dist,
                           float* o_prot_pos, float* o_prot_feat, long long* o_prot_aa, long long* o_prot_batch,
                           float* o_prot_tr, float* o_lig_pos, long long* o_lig_type, long long* o_lig_batch,
                           unsigned char* o_lig_ctx, unsigned char* o_lig_gen, cudaStream_t st);

// ipa.cu (row f4): the IPATransformer forward behind cbg_ipa_forward_f32, arguments already validated; ws holds
// cbg_ipa_workspace_bytes(N, hidden) bytes, 256-byte aligned
int cbg_ipa_launch(const float* blob, int hidden, int num_sublayers, int num_blocks, int num_classes, const float* x,
                   const float* o, const float* h_in, const int* graph_ptr, int n_graphs, int max_graph_nodes,
                   const unsigned char* lig_flag, const unsigned char* gen_flag, int N, int k, float* eps_pos, float* h_out,
                   float* o_next, float* R_next, float* logits, char* ws, cudaStream_t st);
// The IPATransformer shape checks shared by cbg_ipa_forward_f32, cbg_fg_step_f32 and cbg_fg_eval_loss_f32: hidden 128 /
// 256, num_classes in [1, CBG_IPA_MAXCLS], n_nodes in [1, 2^31 / (5 * 256)), num_blocks >= 1, num_sublayers >= 0,
// k in [1, CBG_KMAX] and a non-NULL, 256-byte aligned workspace of at least need_bytes.  Returns 0, or 1 with the error
// set (message prefixed by fn).
int check_ipa_shape(const char* fn, int hidden, int num_classes, long long n_nodes, int num_blocks, int num_sublayers,
                    int k, const void* workspace, long long workspace_bytes, long long need_bytes);

// fg.cu: the D3FG encoder workspace = cbg_ipa_workspace_bytes(n_nodes, hidden) bytes of IPATransformer scratch, then
// the encoder's five output row arrays.  ws == NULL returns the sizes only (null pointers).
struct FgRows {
  float* eps_pos;   // [N,3]
  float* o_pred;    // [N,3]
  float* h_out;     // [N,hidden]
  float* r_next;    // [N,9]
  float* logits;    // [N,K]
  size_t bytes;     // the whole workspace
};
FgRows fg_rows(void* ws, long long n_nodes, int hidden, int K);

// ---- SO(3) maps of repo/models/utils/so3.py in fp32, used by ipa.cu (heads) and fg.cu (D3FG orientation step) ----------
__device__ __forceinline__ void mat3_mul(const float* A, const float* B, float* C) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) C[3 * r + c] = A[3 * r] * B[c] + A[3 * r + 1] * B[3 + c] + A[3 * r + 2] * B[6 + c];
}
// R = exp_skewsym(so3vec_to_skewsym(w))   so3.py:33-57
__device__ __forceinline__ void so3vec_to_rotation(float wx, float wy, float wz, float* R) {
  const float S[9] = {0.f, wz, -wy, -wz, 0.f, wx, wy, -wx, 0.f};
  const float xn = sqrtf(wx * wx + wy * wy + wz * wz);
  const float bb = (sinf(xn) + 1e-8f) / (xn + 1e-8f);
  const float cb = (1.f - cosf(xn) + 1e-8f) / (xn * xn + 2e-8f);
  float S2[9];
  mat3_mul(S, S, S2);
#pragma unroll
  for (int e = 0; e < 9; ++e) R[e] = ((e % 4 == 0) ? 1.f : 0.f) + bb * S[e] + cb * S2[e];
}
// w = skewsym_to_so3vec(log_rotation(R))   so3.py:10-31, 60-63, reformulated so that it is finite for every angle and
// exp(w) = R to fp32 accuracy on all of [0, pi] (DESIGN.md section 16).  The reference's acos((tr - 1) / 2) / (2 sin)
// is NaN when rounding puts the trace above 3, and its sqrt(1 - cos^2) loses the angle quadratically near pi.
// Here c = clamp((tr - 1) / 2, -1, 1), v = the skew vector of R = sin(theta) n, theta = atan2(|v|, c).  For c >= 0
// w = (theta / |v|) v (ratio 1 as |v| -> 0); for c < 0 the axis comes from the symmetric part
// (R + R^T) / 2 - c I = (1 - c) n n^T (the row of the largest diagonal entry), signed by v, and w = theta n.
__device__ __forceinline__ void rotation_to_so3vec(const float* R, float* w) {
  const float c = fminf(fmaxf((R[0] + R[4] + R[8] - 1.f) * 0.5f, -1.f), 1.f);
  const float v[3] = {0.5f * (R[5] - R[7]), 0.5f * (R[6] - R[2]), 0.5f * (R[1] - R[3])};
  const float s = norm3df(v[0], v[1], v[2]);
  const float theta = atan2f(s, c);
  if (c >= 0.f) {
    const float k = s > 0.f ? theta / s : 1.f;
#pragma unroll
    for (int e = 0; e < 3; ++e) w[e] = k * v[e];
    return;
  }
  const int j = (R[0] >= R[4] && R[0] >= R[8]) ? 0 : (R[4] >= R[8] ? 1 : 2);
  float n[3];
#pragma unroll
  for (int e = 0; e < 3; ++e) n[e] = (e == j) ? R[4 * j] - c : 0.5f * (R[3 * j + e] + R[3 * e + j]);
  const float rn = norm3df(n[0], n[1], n[2]);          // >= (1 - c) / sqrt(3) > 0.57
  const float sg = (n[0] * v[0] + n[1] * v[1] + n[2] * v[2]) < 0.f ? -theta : theta;
#pragma unroll
  for (int e = 0; e < 3; ++e) w[e] = sg * (n[e] / rn);
}

// ---- categorical helpers of the type schedules (misc.cu, eval.cu, fg.cu, fg_eval.cu) --------------------------------------
__device__ __forceinline__ float log_add_exp(float a, float b) {         // categorical.py:35-37
  const float m = fmaxf(a, b);
  return m + logf(expf(a - m) + expf(b - m));
}
// log(clamp(0, 1e-30)) in fp32 (index_to_log_onehot, categorical.py:5-11): the off-class entry of a log one-hot
__device__ __forceinline__ float log_1e30() { return __int_as_float(-1031133259); }   // -69.07755f

// ---- D3FG per-FG helpers shared by fg.cu (reverse step) and fg_eval.cu (validation loss): one warp per functional
// group, lane k holding class k ------------------------------------------------------------------------------------------
__device__ __forceinline__ float fg_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(CBG_FULL, v, o));
  return v;
}

// torch.argmax over the lanes: the largest value, the lowest index among equal values
__device__ __forceinline__ int fg_warp_argmax(float v, int idx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(CBG_FULL, v, o);
    const int oi = __shfl_xor_sync(CBG_FULL, idx, o);
    if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
  return idx;
}

// The rotation noise e = normalize(axis) * theta of random_normal_so3 (so3.py:140-146) for one FG, with theta drawn
// by ApproxAngularDistribution.sample (:111-138) from the distribution whose tables are angle_x [T,n_bins] /
// angle_cdf [T,n_bins-1]: |2 std + std n| mod pi when `gaussian`, else the histogram bin
// b = min{i : C_t[i] > u C_t[n_bins - 2]} (the definition of the multinomial draw) and X[b] + u' (X[b+1] - X[b]).
// rd = axis N(0,1)^3 | bin uniform u | in-bin uniform u' | Gaussian-branch N(0,1) n.  Returns theta.
__device__ __forceinline__ float fg_draw_rotation(const float* rd, int t, float std, bool gaussian,
                                                  const float* angle_x, const double* angle_cdf, int n_bins,
                                                  float (&e)[3]) {
  float theta;
  if (gaussian) {
    theta = fmodf(fabsf(__fadd_rn(std * 2.f, __fmul_rn(rd[5], std))), 3.14159265358979323846f);
  } else {
    const int nc = n_bins - 1;
    const double* C = angle_cdf + (size_t)t * nc;
    const double target = (double)rd[3] * C[nc - 1];
    int lo = 0, hi = nc - 1;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (C[mid] > target) hi = mid; else lo = mid + 1;
    }
    const float* X = angle_x + (size_t)t * n_bins;
    theta = __fadd_rn(X[lo], __fmul_rn(rd[4], __fsub_rn(X[lo + 1], X[lo])));
  }
  // F.normalize: a / max(|a|, 1e-12); norm3df does not overflow for |a| up to FLT_MAX (axis draws of 1e30)
  const float nrm = fmaxf(norm3df(rd[0], rd[1], rd[2]), 1e-12f);
#pragma unroll
  for (int c = 0; c < 3; ++c) e[c] = __fmul_rn(__fdiv_rn(rd[c], nrm), theta);
  return theta;
}
