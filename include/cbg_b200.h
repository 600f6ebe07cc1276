/* cbg_b200 - C-ABI of the H100-native (sm_90a) CBGBench diffusion-sampling hot path.
 *
 * The reference (EDAPINENUT/CBGBench @ 983fca2) is 100 % Python/PyTorch and
 * has NO FFI / plugin / operator boundary of its own (SURVEY.md section 8b): its seam is the Python
 * factory get_e3_gnn() (repo/modules/e3nn/__init__.py:5-18) returning an nn.Module whose
 * forward(x, h, batch_idx, lig_flag, gen_flag) -> (x, h, c) is repo/modules/e3nn/unitransformer.py:102-123,
 * iterated by TargetDiff.sample (repo/models/diffusion/targetdiff.py:127-184).  The entry points
 * below are what a ctypes binding for that seam needs; each one cites the reference code it
 * replaces.  INTEGRATION.md shows the reference-side stub.
 *
 * Conventions
 *   - plain C, no C++ types or exceptions across the boundary;
 *   - every pointer is a DEVICE pointer owned by the caller unless the name ends in _host;
 *   - fp32 data, int32 indices, uint8 flags; row-major contiguous;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream); calls only
 *     enqueue work (no host synchronisation) unless the name ends in _host;
 *   - return 0 on success; non-zero = error, message from cbg_last_error() (thread-local);
 *   - graphs are contiguous node ranges: graph g owns nodes graph_ptr[g] .. graph_ptr[g+1]-1
 *     (the reference's sorted PyG `batch` vector, repo/modules/common.py:189-214);
 *   - neighbour tables have fixed width CBG_NBR_WIDTH = 32 (k <= 32), nearest first,
 *     padded with -1 (graphs with fewer than k+1 atoms, radius mode).
 */
#ifndef CBG_B200_H_
#define CBG_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CBG_NBR_WIDTH 32
#define CBG_HIDDEN 128
#define CBG_N_HEADS 16
#define CBG_MAX_CLASSES 16

#define CBG_CUTOFF_KNN 0     /* reference default, unitransformer.py:27-28,78-80 */
#define CBG_CUTOFF_RADIUS 1  /* defined in SURVEY.md section 8c (reference branch is dead code, unitransformer.py:76-77) */

int32_t cbg_version(void);
const char* cbg_last_error(void);
/* number of CUDA kernels this library has launched in the calling process (bench.py gpu_launches) */
int64_t cbg_launch_count(void);

/* Optional per-kernel profile: while enabled every kernel launch of the library is bracketed by
 * CUDA events on the launching stream; cbg_profile_collect synchronises and returns the summed
 * device time (ms) and launch count per kernel family (bench.py roofline block). */
int32_t cbg_profile_num_families(void);
const char* cbg_profile_family_name(int32_t i);
int32_t cbg_profile_enable(int32_t on);
int32_t cbg_profile_collect(double* ms_per_family, int64_t* launches_per_family);

/* TESTING hook (process-wide, not thread-safe; production code never calls it): implementation of the fused X2H / H2X
 * edge kernels.  impl 6 (default): the wgmma tile kernel (csrc/x2h_tc.cu: activations as register A fragments, f16 hi/lo split);
 * impl 0: the fp32 SIMT kernels (csrc/edge.cu), kept as an independent implementation for the parity tests - the only
 * consumer of the optional R-cache.  warps = CTA size of the SIMT kernels (8, 12, 16; 0 keeps the current value).
 * Also env CBG_EDGE_IMPL / CBG_EDGE_WARPS.  Needs a current CUDA device. */
int32_t cbg_set_edge_impl(int32_t impl, int32_t warps);
/* Hardware self-test of the wgmma operand conventions the X2H kernels rely on (tests only):
 * d[128][128] (fp32) = a[128][32] * b[128][32]^T with f16 row-major device inputs; a_from_smem = 0 feeds A from
 * registers (the accumulator-compatible fragment layout), 1 from shared memory (canonical K-major layout). */
int32_t cbg_selftest_umma_f16(const void* a, const void* b, float* d, int32_t a_from_smem, void* stream);
/* Debugging: the next launch of the attention-weight tile kernel (max_tiles > 0) or aggregation kernel (max_tiles < 0,
 * |max_tiles| rows) stamps the per-tile events of CTA 0 (SM clock; slots 0 - 4: G staged, MMA1, activations, MMA2, epilogue) into buf_dev[|max_tiles| + 1][16] (int64, device memory;
 * the last row takes kernel entry / end of prologue / exit); NULL turns it off.  Process-wide, one-shot. */
int32_t cbg_debug_x2h_trace(int64_t* buf_dev, int32_t max_tiles);
/* debug: %globaltimer stamps (ns) of CTA 0 of every following f16 node-GEMM launch into buf_dev[32] (NULL = off):
 * [0] start, [1] A tile staged, [2+g] accumulator g complete, [10+g] epilogue of g done, [20] end */
int32_t cbg_debug_node_gemm_trace(int64_t* buf_dev);
/* Other TESTING switches of the SIMT kernels (process-wide): "static_fast" = 1 (default; env CBG_STATIC_FAST) lets them
 * skip the coordinate gathers / RBF set-up of nodes whose 32 in-edges are all served from the R-cache (bit-identical);
 * "dyn_sched" = 1 (default; env CBG_DYN_SCHED): their warps draw the next node from a work counter instead of a static
 * round-robin (bit-identical). */
int32_t cbg_set_option(const char* key, int32_t value);

/* ---- packed weight blob layout (single source of truth: csrc/cbg_layout.h) -------------------
 * blob = [global section][layer 0][layer 1]...; section 0 = global, 1 = per-layer.
 * Replaces the nn.Module parameter tree of UniTransformer (state-dict keys in SURVEY.md section 8b). */
int64_t cbg_blob_global_floats(void);
int64_t cbg_blob_layer_floats(void);
int32_t cbg_blob_num_fields(int32_t section);
const char* cbg_blob_field_name(int32_t section, int32_t idx);
int64_t cbg_blob_field_offset(int32_t section, int32_t idx);
int64_t cbg_blob_field_size(int32_t section, int32_t idx);

/* bytes of the optional R-cache of a sampling plan: 2 * num_layers * n_nodes * 32 * 128 floats */
int64_t cbg_rcache_bytes(int64_t n_nodes, int32_t num_layers);

/* scratch bytes needed by the calls below for n_nodes nodes of which n_gen carry gen_flag */
int64_t cbg_workspace_bytes(int64_t n_nodes, int64_t n_gen);

/* Neighbour lists on device.
 * Replaces torch_geometric.nn.knn_graph(x, k, batch, flow='source_to_target')
 * (call site unitransformer.py:79-80; third-party torch_cluster kernel).  nbr[i, s] = global index
 * of the s-th nearest j != i of i's graph (ties -> lower index), -1 padded.  The reference's
 * edge_index is [nbr[i,s] ; i] for all valid slots, grouped by i. */
int32_t cbg_build_neighbors_f32(const float* x /*[N,3]*/, const int32_t* graph_ptr /*[B+1]*/,
                                int32_t n_graphs, int64_t n_nodes, int32_t max_graph_nodes,
                                int32_t mode, int32_t k, float r_max,
                                int32_t* nbr /*[N,32] out*/,
                                void* workspace, size_t workspace_bytes, void* stream);

/* Global edge gate e_w = sigmoid(dist_emb(|x_i - x_j|)) (unitransformer.py:109-112,
 * embs/dist_emb.py:6-14).  ew[i, s] for slot s of node i (0 for padded slots). */
int32_t cbg_edge_gate_f32(const float* blob, const float* x /*[N,3]*/, const int32_t* nbr /*[N,32]*/,
                          int64_t n_nodes, float* ew /*[N,32] out*/,
                          void* workspace, size_t workspace_bytes, void* stream);

/* One full denoiser forward = UniTransformer.forward (unitransformer.py:102-123): graph build,
 * edge gate, num_layers x (X2HAttention, H2XAttention, masked coordinate update), classifier.
 * Inputs are not modified.  gen_idx lists the nodes with gen_flag set (any order);
 * cls_idx = NULL computes logits for all nodes (logits_out [N,K]) else only for the listed
 * rows (logits_out [n_cls,K]).  stop_after_layers < 0 runs all layers (testing hook: run
 * only the first stop_after_layers layers, then the classifier). */
int32_t cbg_denoiser_forward_f32(const float* blob, int32_t num_layers, int32_t num_classes,
                                 const float* x /*[N,3]*/, const float* h /*[N,128]*/,
                                 const int32_t* graph_ptr, int32_t n_graphs, int32_t max_graph_nodes,
                                 const uint8_t* lig_flag /*[N]*/, const uint8_t* gen_flag /*[N]*/,
                                 const int32_t* gen_idx, int32_t n_gen,
                                 const int32_t* cls_idx, int32_t n_cls,
                                 int64_t n_nodes, int32_t mode, int32_t k, float r_max,
                                 int32_t stop_after_layers,
                                 float* x_out /*[N,3]*/, float* h_out /*[N,128]*/, float* logits_out,
                                 void* workspace, size_t workspace_bytes, void* stream);

/* Same call with HOST buffers (pageable or pinned): copies inputs to the device, runs the
 * forward, copies x_out/h_out/logits_out back and synchronises.  Device scratch is cached
 * inside the library.  blob_host holds the packed weights; it is re-uploaded when
 * blob_version changes. */
int32_t cbg_denoiser_forward_host_f32(const float* blob_host, int64_t blob_floats, int64_t blob_version,
                                      int32_t num_layers, int32_t num_classes,
                                      const float* x_host, const float* h_host,
                                      const int32_t* graph_ptr_host, int32_t n_graphs,
                                      const uint8_t* lig_flag_host, const uint8_t* gen_flag_host,
                                      int64_t n_nodes, int32_t mode, int32_t k, float r_max,
                                      float* x_out_host, float* h_out_host, float* logits_out_host);

/* Node projections of one attention sub-layer alone (testing / integration hook): the five planes
 * [Pj_k, Pj_v, Pi_k, Pi_v, q] of sub-layer `sublayer` (0 = X2H, 1 = H2X) for the listed rows
 * (row_idx NULL = rows 0..n_rows-1), planes = [5][n_nodes][128].  impl 0 = fp32 SIMT kernel,
 * 1 = wgmma 3xTF32 kernel, 2 = wgmma f16 (hi, lo) kernel (default of the library), 11 / 12 / 14 = the 3xTF32 kernel
 * with weight chunks multicast over clusters of 1 / 2 / 4 CTAs (1 takes the cluster size from env CBG_GEMM_CLUSTER,
 * default 1: without that variable 1 and 11 run the same code).  blob_layer points at the layer's block inside the packed blob.
 * Replaces the h-dependent part of MLP.net[0] and hq_func/xq_func (x2h_attention.py:58-83). */
int32_t cbg_node_proj_f32(const float* blob_layer, int32_t sublayer, int32_t impl, const float* h,
                          const int32_t* row_idx, int32_t n_rows, int64_t n_nodes, float* planes, void* stream);

/* ---- fused sampling step: embed -> denoiser -> reverse diffusion step -------------------------
 * One iteration of the loop body of TargetDiff.sample (targetdiff.py:150-182):
 *   PLContextEmbedder.forward (context_emb.py:179-231), compose_context (common.py:189-214,
 *   hoisted: the permutation is step-invariant), denoiser, then
 *   CTNVPScheduler.backward_remove_noise(type='denoise') (diffusion_scheduler.py:144-165) and
 *   TypeVPScheduler.backward_remove_noise (diffusion_scheduler.py:367-378).
 * Random numbers stay with the caller (torch.randn_like / rand_like order of the reference). */
typedef struct cbg_sample_plan {
  const float* blob;            /* packed denoiser weights */
  int32_t num_layers;
  int32_t num_classes;
  const float* emb_wt;          /* [K,128] context_embedder.ligand_atom_emb.weight^T */
  const float* h_lig_bias;      /* [n_lig,128] ligand_atom_emb.bias + ligand_indicator(lig_flag) */
  const float* h_static;        /* [N,128] step-invariant node features (protein rows) */
  const int32_t* graph_ptr;     /* [B+1] over composed nodes ([protein | ligand] per graph) */
  int32_t n_graphs;
  int32_t max_graph_nodes;
  int64_t n_nodes;
  const int32_t* lig_node;      /* [n_lig] composed node index of every ligand atom */
  int32_t n_lig;
  const uint8_t* gen_lig;       /* [n_lig] ligand_gen_flag */
  const int32_t* gen_node;      /* [n_gen] composed node indices with gen_flag */
  int32_t n_gen;
  int32_t mode;                 /* CBG_CUTOFF_* */
  int32_t k;
  float r_max;
  void* workspace;
  size_t workspace_bytes;
  float* rcache;                /* optional (NULL = off): cbg_rcache_bytes() of scratch for the step-invariant
                                   first-Linear terms of edges between non-generated atoms (SURVEY.md App. B);
                                   filled by cbg_sample_begin_f32, streamed by the fused X2H kernels */
  size_t rcache_bytes;
  int32_t prune;                /* 1: receptive-field pruning - layer l only updates the nodes that can still
                                   influence a generated / ligand atom through the remaining layers (exact for
                                   everything cbg_sample_step_f32 returns; intermediate h of other nodes is skipped) */
  int32_t static_lists;         /* 1: atoms without gen_flag never move, so cbg_sample_begin_f32 builds their static-only
                                   neighbour lists and edge gates once per batch; every step's neighbour search is then
                                   incremental and static edges reuse their gate (exact).  Implied by rcache != NULL.
                                   Must be 0 for samplers that move the pocket (DiffSBDD). */
} cbg_sample_plan;

typedef struct cbg_step_coef {  /* scheduler table entries of the current step (host scalars) */
  float pos_c0;                 /* pos_scheduler.posterior_mean_c0_coef[t] */
  float pos_ct;                 /* pos_scheduler.posterior_mean_ct_coef[t] */
  float pos_logvar;             /* pos_scheduler.posterior_logvar[t] */
  float pos_nonzero;            /* 0 if t == 0 else 1 */
  float log_alphas_cumprod_prev;          /* type_scheduler.log_alphas_cumprod_v[max(t-1,0)] */
  float log_one_minus_alphas_cumprod_prev;/* type_scheduler.log_one_minus_alphas_cumprod_v[max(t-1,0)] */
  float log_alpha;              /* type_scheduler.log_alphas_v[t] */
  float log_one_minus_alpha;    /* type_scheduler.log_one_minus_alphas_v[t] */
} cbg_step_coef;

/* writes the static part of the node state (all coordinates + flags) into the plan workspace */
int32_t cbg_sample_begin_f32(const cbg_sample_plan* plan, const float* x_nodes /*[N,3]*/,
                             const uint8_t* lig_flag /*[N]*/, const uint8_t* gen_flag /*[N]*/, void* stream);

/* Measurement hook (bench.py roofline): node counts of the receptive-field pruning of the LAST step run on this plan,
 * counts_host[l + 1] = nodes whose X2H output of layer l is still needed (= rows the X2H kernels of layer l process),
 * counts_host[0] = nodes needed at all; num_layers + 1 entries.  Copies to host memory and synchronises the stream. */
int32_t cbg_sample_prune_counts_host(const cbg_sample_plan* plan, int32_t* counts_host /*[num_layers+1]*/, void* stream);

int32_t cbg_sample_step_f32(const cbg_sample_plan* plan, const cbg_step_coef* coef,
                            const float* x_t /*[n_lig,3]*/, const float* c_t /*[n_lig,K]*/,
                            const float* pos_noise /*[n_lig,3]*/, const float* type_uniform /*[n_lig,K]*/,
                            float* x_next /*[n_lig,3]*/, float* c_next /*[n_lig,K]*/, int64_t* v_next /*[n_lig]*/,
                            float* x0_pred /*[n_lig,3] or NULL*/, float* logits /*[n_lig,K] or NULL*/,
                            void* stream);

/* cbg_sample_step_f32 replayed from a CUDA graph: the first call for a plan runs eagerly, the second captures the step
 * (its ~85 kernel launches, fork/join events and memsets) on `stream`, later calls cost one small H2D copy of the per-step
 * pointers / schedule coefficients plus one cudaGraphLaunch.  Results are bit-identical to cbg_sample_step_f32 (same
 * kernels, same order).  The plan must be unchanged between calls (same contents); x0_pred / logits outputs are not
 * available on this path.  cbg_sample_step_graph_nodes: kernel launches inside the captured graph (0: not captured yet). */
int32_t cbg_sample_step_graph_f32(const cbg_sample_plan* plan, const cbg_step_coef* coef,
                                  const float* x_t, const float* c_t, const float* pos_noise, const float* type_uniform,
                                  float* x_next, float* c_next, int64_t* v_next, void* stream);
int64_t cbg_sample_step_graph_nodes(const cbg_sample_plan* plan, void* stream);

/* ---- validation loss: TargetDiff.forward in eval mode (targetdiff.py:41-124) -----------------------------------------
 *
 * The plan is one cbg_sample_begin_f32 filled over n_rep replicas of one batch of B graphs and n_lig / n_rep ligand atoms:
 * graph r*B + g and ligand atom r*(n_lig/n_rep) + a of the plan are graph g and atom a of the batch, noised at replica r's
 * timestep.  One call enqueues: forward noising of positions (CTNVPScheduler.forward_add_noise, diffusion_scheduler.py:
 * 117-134) and types (q(v_t | v_0) Gumbel sample, :339-346 / :380-396) -> the denoiser with receptive-field pruning ->
 * classifier on the ligand rows -> per-graph position MSE and type KL (decoder NLL at t == 0) (:185-201, :348-418) ->
 * per-replica scatter_mean(...).mean().  The denoiser does not see t, so the replicas share one pass.  Every reduction
 * runs in a fixed order (no atomics): repeated calls are bit-identical. */
typedef struct cbg_eval_coef {  /* scheduler table entries of one replica's timestep t (host scalars) */
  float alphas_cumprod;                    /* pos_scheduler.alphas_cumprod[t] */
  float log_alphas_cumprod;                /* type_scheduler.log_alphas_cumprod_v[t] */
  float log_one_minus_alphas_cumprod;      /* type_scheduler.log_one_minus_alphas_cumprod_v[t] */
  float log_alphas_cumprod_prev;           /* type_scheduler.log_alphas_cumprod_v[max(t-1,0)] */
  float log_one_minus_alphas_cumprod_prev; /* type_scheduler.log_one_minus_alphas_cumprod_v[max(t-1,0)] */
  float log_alpha;                         /* type_scheduler.log_alphas_v[t] */
  float log_one_minus_alpha;               /* type_scheduler.log_one_minus_alphas_v[t] */
  int32_t t_is_zero;                       /* 1: the type loss is the decoder NLL instead of the KL */
} cbg_eval_coef;

/* coefs: host array [n_rep], n_rep <= 64.  x0 / v0: the batch's ligand_pos [n_lig/n_rep,3] / ligand_atom_type.
 * Noise [n_rep, n_lig/n_rep, 3] (normal) and [n_rep, n_lig/n_rep, K] (uniform) comes from the caller.
 * Outputs: xt, x_pred [n_rep, n_lig/n_rep, 3]; vt [n_rep, n_lig/n_rep]; c_pred = softmax(logits) [n_rep, n_lig/n_rep, K];
 * graph_loss [n_rep*B, 2] per-graph (pos, atom) means over generated atoms (0 for a graph without any);
 * rep_loss [n_rep, 2] per-replica (pos, atom) losses (NaN when no atom is generated). */
int32_t cbg_eval_loss_f32(const cbg_sample_plan* plan, const cbg_eval_coef* coefs, int32_t n_rep,
                          const float* x0, const int64_t* v0, const float* pos_noise, const float* type_uniform,
                          float* xt, int64_t* vt, float* x_pred, float* c_pred, float* graph_loss, float* rep_loss,
                          void* stream);

/* the reverse step alone (testing / integration hook); refuses NULL pointers and n < 0 before touching the device */
int32_t cbg_reverse_step_f32(const cbg_step_coef* coef, const float* x0_pred /*[n,3]*/, const float* logits /*[n,K]*/,
                             const float* x_t, const float* c_t, const uint8_t* gen /*[n]*/,
                             const float* pos_noise, const float* type_uniform,
                             int32_t n, int32_t num_classes,
                             float* x_next, float* c_next, int64_t* v_next, void* stream);

/* ---- SURVEY.md section 8 row f2: the other diffusion samplers that drive the same denoiser -------------------
 *
 * DiffSBDD (diffsbdd.py:240-321): every step is embed -> denoiser -> sample_p_zs_given_zt
 * (diffusion_scheduler.py:1005-1039) for coordinates and (continuous) type features, with the COM projection
 * remove_mean_batch (:706-710) that also translates the pocket.  All graphs share (s, t), so the schedule enters as
 * three host scalars.  mode 1 is the final stage sample_p_xh_given_z0 (diffsbdd.py:323-360).
 * The plan is the one of cbg_sample_begin_f32 WITHOUT an R-cache (the pocket is not static here). */
typedef struct cbg_sbdd_coef {
  float a;       /* mode 0: alpha_t|s                      mode 1: 1 / alpha_0            */
  float b;       /* mode 0: sigma2_t|s / alpha_t|s / sigma_t   mode 1: sigma_0            */
  float s;       /* mode 0: sigma_t|s * sigma_s / sigma_t  mode 1: exp(0.5 * gamma_0)     */
  int32_t mode;  /* 0: z_s = z_t / a - b * eps + s * noise;  1: z = a * (z_t - b * eps) + s * noise, c_next = 4 c_t */
} cbg_sbdd_coef;

int32_t cbg_sbdd_step_f32(const cbg_sample_plan* plan, const cbg_sbdd_coef* coef,
                          const float* x_t /*[n_lig,3]*/, const float* c_t /*[n_lig,K]*/,
                          const float* x_noise /*[n_lig,3]*/, const float* c_noise /*[n_lig,K]*/,
                          float* x_next /*[n_lig,3]*/, float* c_next /*[n_lig,K]*/,
                          float* x_pred /*[n_lig,3] or NULL*/, float* logits /*[n_lig,K] or NULL*/, void* stream);

/* The DiffSBDD reverse step alone (testing hook): the kernel of cbg_sbdd_step_f32 on caller-given rows.  x4 [N,4] holds
 * the node coordinates and the flag float (bit 0 = ligand): its ligand rows are the denoiser's output coordinates
 * eps_pred, its pocket rows (bit 0 clear) are shifted in place by their graph's ligand mean.  Graph g owns the nodes
 * [graph_ptr[g], graph_ptr[g + 1]); lig_node [n_lig] must be ascending and every entry must lie inside the node range
 * of the graph it belongs to.  The pocket of a graph without ligand atoms is not moved (its mean is taken as 0).
 * Refuses NULL pointers, num_classes outside [1, 16], n_graphs < 0, n_lig < 0 and a mode other than 0 / 1 before
 * touching the device. */
int32_t cbg_sbdd_reverse_f32(float* x4 /*[N,4]*/, const int32_t* graph_ptr /*[n_graphs+1]*/, int32_t n_graphs,
                             const int32_t* lig_node /*[n_lig]*/, int32_t n_lig, int32_t num_classes,
                             const cbg_sbdd_coef* coef, const float* logits /*[n_lig,K]*/,
                             const float* x_t /*[n_lig,3]*/, const float* c_t /*[n_lig,K]*/,
                             const float* x_noise /*[n_lig,3]*/, const float* c_noise /*[n_lig,K]*/,
                             float* x_next /*[n_lig,3]*/, float* c_next /*[n_lig,K]*/, void* stream);

/* DiffBP (diffbp.py:240-299): embed -> denoiser -> CoM head (CoMPredictor, diffbp.py:30-101: the step's kNN graph,
 * its own edge gate, com_layers x H2X on the denoiser's final h starting from the step's input coordinates) ->
 * CTNVPScheduler.backward_remove_noise(type='score') (diffusion_scheduler.py:144-165) on eps + eps_com and
 * MaskTypeSchedule.backward_remove_noise (:474-498).  com_blob packs the CoM head in the denoiser's blob layout
 * (gate fields of the global block, H2X fields of com_layers layer blocks).  type_uniform is [n_lig]. */
typedef struct cbg_bp_coef {
  float alpha_cumprod;   /* pos_scheduler.alphas_cumprod[t] */
  float beta;            /* pos_scheduler.betas[t] */
  float nonzero;         /* 0 if t == 0 else 1 */
  float change_prob;     /* clamp((T - t) / T, 0, 1) */
} cbg_bp_coef;

int32_t cbg_bp_step_f32(const cbg_sample_plan* plan, const float* com_blob, int32_t com_layers,
                        const cbg_bp_coef* coef, const float* x_t /*[n_lig,3]*/, const float* c_t /*[n_lig,K]*/,
                        const float* pos_noise /*[n_lig,3]*/, const float* type_uniform /*[n_lig]*/,
                        float* x_next /*[n_lig,3]*/, float* c_next /*[n_lig,K]*/, int64_t* v_next /*[n_lig]*/,
                        float* eps_out /*[n_lig,3] or NULL: eps + eps_com*/, float* logits /*[n_lig,K] or NULL*/,
                        void* stream);

/* The DiffBP reverse step alone (testing hook): the kernel of cbg_bp_step_f32 on caller-given rows.  x4 [N,4] as in
 * cbg_sbdd_reverse_f32, its ligand rows holding x_com (the CoM head's output coordinates); it is only read.  graph_ptr /
 * lig_node as in cbg_sbdd_reverse_f32 (ascending, inside the graphs' node ranges).  x_pred: the denoiser's output
 * coordinates [n_lig,3]; type_uniform [n_lig]; eps_out may be NULL.  Refuses NULL pointers (other than eps_out),
 * num_classes outside [1, 16], n_graphs < 0 and n_lig < 0 before touching the device. */
int32_t cbg_bp_reverse_f32(const float* x4 /*[N,4]*/, const int32_t* graph_ptr /*[n_graphs+1]*/, int32_t n_graphs,
                           const int32_t* lig_node /*[n_lig]*/, int32_t n_lig, int32_t num_classes,
                           const cbg_bp_coef* coef, const float* x_pred /*[n_lig,3]*/, const float* logits /*[n_lig,K]*/,
                           const float* x_t /*[n_lig,3]*/, const float* c_t /*[n_lig,K]*/, const uint8_t* gen /*[n_lig]*/,
                           const float* pos_noise /*[n_lig,3]*/, const float* type_uniform /*[n_lig]*/,
                           float* x_next /*[n_lig,3]*/, float* c_next /*[n_lig,K]*/, int64_t* v_next /*[n_lig]*/,
                           float* eps_out /*[n_lig,3] or NULL*/, void* stream);

/* ---- validation loss: DiffBP.forward in eval mode (diffbp.py:133-230) ------------------------------------------------
 *
 * Same replica layout as cbg_eval_loss_f32 (graph r*B + g and ligand atom r*(n_lig/n_rep) + a of the plan are graph g
 * and atom a of the batch).  One call enqueues: forward noising of positions with the raw normal draw
 * (CTNVPScheduler.forward_add_noise, zero_center=True) and the absorbing-state type mask (MaskTypeSchedule.
 * forward_add_noise) -> the denoiser -> classifier -> the CoM head of cbg_bp_step_f32 on the noised coordinates ->
 * per-graph position / CoM score losses, masked-type cross-entropy of softmax(logits) and the interior loss
 * (diffbp.py:19-30: for each protein atom its min(48, n_lig_g) nearest ligand atoms of the graph at the posterior
 * mean of x_{t-1}, nearest first, ties to the lower ligand index) -> per-replica reduction.  No atomics: repeated calls
 * are bit-identical. */
typedef struct cbg_bp_eval_coef {  /* one replica's timestep t */
  float alphas_cumprod;            /* pos_scheduler.alphas_cumprod[t] */
  float beta;                      /* pos_scheduler.betas[t] */
  float mask_prob;                 /* float(t) / T in fp32: probability that a generated atom is masked */
} cbg_bp_eval_coef;

/* coefs: host array [n_rep], n_rep <= 64.  com_blob / com_layers as in cbg_bp_step_f32.  x0 / v0: the batch's
 * ligand_pos [n_lig/n_rep,3] / ligand_atom_type.  Draws from the caller: pos_noise [n_rep, n_lig/n_rep, 3] (normal),
 * type_uniform [n_rep, n_lig/n_rep] (uniform).  Outputs: xt [n_rep, n_lig/n_rep, 3]; vt / mask [n_rep, n_lig/n_rep]
 * (the noised type and the type mask); vec [n_rep, 8, n_lig/n_rep, 3] = eps_0, eps_pred, score_0, score_pred,
 * eps_0_com, eps_pred_com, score_0_com, score_pred_com (score = eps * sqrt(1 - alphas_cumprod)); c_pred = softmax(logits)
 * [n_rep, n_lig/n_rep, K]; rep_loss [n_rep, 4] = pos, atom, com, inter (pos / com NaN when no atom is generated, atom 0
 * when no atom is masked). */
int32_t cbg_bp_eval_loss_f32(const cbg_sample_plan* plan, const float* com_blob, int32_t com_layers,
                             const cbg_bp_eval_coef* coefs, int32_t n_rep, const float* x0, const int64_t* v0,
                             const float* pos_noise, const float* type_uniform, float* xt, int64_t* vt, uint8_t* mask,
                             float* vec, float* c_pred, float* rep_loss, void* stream);

/* ---- validation loss: DiffSBDD.forward in eval mode (diffsbdd.py:48-191) ----------------------------------------------
 *
 * Every timestep t of the batch is noised twice, at t and at 0, and both copies go through the denoiser.  The plan holds
 * 2 n_t replicas of the batch (graph r*B + g and ligand atom r*(n_lig/(2 n_t)) + a are graph g and atom a): replica 2j
 * is timestep j at t_j, replica 2j+1 timestep j at 0.  No static lists or R-cache: the pocket moves with each copy.
 * One call enqueues: remove_mean_batch of the clean ligand and pocket, forward_pos_center_noise (the noisy ligand's mean
 * over all its atoms is removed from the generated atoms and the pocket; the other ligand atoms stay at their centred
 * clean positions) and forward_type_add_noise of the types onehot / 4 (diffusion_scheduler.py:706-775) -> the denoiser
 * -> classifier -> per (timestep, graph) the six terms of get_score_loss in eval mode (:897-920), the denoiser's ligand
 * output coordinates acting as the position noise prediction and the logits as the type noise prediction -> the per-t
 * means.  No atomics: repeated calls are bit-identical.  Every scalar below is the reference's fp32 torch expression. */
typedef struct cbg_sbdd_eval_coef {  /* one timestep t (gamma_t = gamma[round(t/T * T)], s = (t-1)/T) */
  float pos_alpha_t, pos_sigma_t;    /* sqrt(sigmoid(-gamma_t)), sqrt(sigmoid(gamma_t)) of pos_scheduler */
  float type_alpha_t, type_sigma_t;  /* the same of type_scheduler */
  float pos_alpha_0, pos_sigma_0;    /* at t = 0 */
  float type_alpha_0, type_sigma_0;
  float pos_t_weight;                /* -T * 0.5 * (1 - exp(-(gamma_s - gamma_t))) */
  float type_t_weight;
  float pos_log_const;               /* -0.5 * gamma_0 - 0.5 * log(2 pi) */
  float type_log_const;
  float pos_alpha_T, type_alpha_T;   /* at t = 1 (the prior) */
  float pos_log_inv_sigma_T;         /* log(1 / sigma_T) */
  float type_log_inv_sigma_T;
  float pos_sigma2_T, type_sigma2_T; /* sigma_T ** 2 */
} cbg_sbdd_eval_coef;

/* coefs: host array [n_t], n_t <= 32.  x0 / v0 / x_rec: the batch's ligand_pos [n1,3] / ligand_atom_type [n1] /
 * protein_pos [n_rec1,3] (NULL when the batch has no protein atoms), n1 = n_lig / (2 n_t).  Draws from the caller (normal):
 * x_t_noise [n_t,n1,3], c_t_noise [n_t,n1,K] (the copy at t), x_0_noise, c_0_noise (the copy at 0).  Outputs:
 * vec_pos [n_t,3,n1,3] = eps_pred, score_0, score_pred of the positions (score = eps * sigma_t), vec_atom [n_t,3,n1,K]
 * the same of the types; terms [n_t,B,6] = pos_t, pos_0, pos_kl, atom_t, atom_0, atom_kl of every graph of the batch
 * (B = n_graphs / (2 n_t)); t_loss [n_t,2] = pos, atom: the mean over the graphs up to the last one with ligand atoms. */
int32_t cbg_sbdd_eval_loss_f32(const cbg_sample_plan* plan, const cbg_sbdd_eval_coef* coefs, int32_t n_t,
                               const float* x0, const int64_t* v0, const float* x_rec, const float* x_t_noise,
                               const float* c_t_noise, const float* x_0_noise, const float* c_0_noise, float* vec_pos,
                               float* vec_atom, float* terms, float* t_loss, void* stream);

/* ---- SURVEY.md section 8 row f3: sampling-time transforms + batch construction on the device ------------------
 *
 * The reference builds a sampling batch by evaluating dataset[i] num_samples times (sample.py:177), i.e. by running
 * the Python transform list of configs/<task>/test/<model>.yml once per sample, and collating with PyG.  The three calls
 * below produce the same flat batch from the raw pocket arrays on the device.  Pockets are ragged ranges
 * (prot_ptr[n_pockets+1]); every pocket is sampled `repeat` times; sample s belongs to pocket s / repeat.
 * Random numbers are the caller's (numpy / torch order of the reference: one uniform per sample for the size prior,
 * optionally one randint(1, 8), then rand [n, K] for the types and randn [n, 3] for the positions). */

/* Pocket centre and "space size".
 *   centre_mode 0: centre = mean of the pocket atoms (center_pos(center_flag=protein), translation.py:11-24, and
 *                  center_whole_pos without a ligand, :36-50); space size measured on the centred coordinates
 *   centre_mode 1: centre = mean of the pocket's context ligand atoms, 0 if it has none (center_pos(ligand,
 *                  mask_flag=ctx_flag)); space size measured on the raw coordinates (assign_gensize runs first)
 * space_size = median of the 10 largest pairwise atom distances (AssignMolSize.get_space_size, init_lig.py:247-250). */
int32_t cbg_pocket_stats_f32(const float* prot_pos /*[n_atoms,3]*/, const int32_t* prot_ptr /*[n_pockets+1]*/,
                             int32_t n_pockets, const float* ctx_pos /*[n_ctx,3] or NULL*/,
                             const int32_t* ctx_ptr /*[n_pockets+1] or NULL*/, int32_t centre_mode,
                             float* space_size /*[n_pockets] out*/, float* centre /*[n_pockets,3] out*/, void* stream);

/* Size prior (repo/datasets/transforms/_atom_num_dist.npy) as flat device arrays: bin b (b = 0..n_bounds) is chosen by
 * the first bound greater than the space size (init_lig.py:47-52) and holds values[bin_ptr[b]:bin_ptr[b+1]] with the
 * cumulative distribution cdf[...] = cumsum(p) / sum(p) that numpy's legacy choice(values, p=p) searches
 * (side='right') with its uniform draw (sample_atom_num, init_lig.py:27-31). */
typedef struct cbg_size_prior {
  const double* bounds;
  int32_t n_bounds;
  const int32_t* bin_ptr;   /* [n_bounds + 2] */
  const int32_t* values;
  const double* cdf;
} cbg_size_prior;

/* Ligand atom counts of the n_pockets * repeat samples and their exclusive prefix sum.  With ctx_ptr (context tasks,
 * AssignGenSize init_lig.py:253-296) a draw that does not exceed the pocket's context atom count is replaced by
 * context + extra[s] (the reference's torch.randint(1, 8)). */
int32_t cbg_sample_ligand_sizes(const cbg_size_prior* prior, const float* space_size /*[n_pockets]*/, int32_t n_pockets,
                                int32_t repeat, const double* u /*[S]*/, const int32_t* ctx_ptr /*or NULL*/,
                                const int32_t* extra /*[S] or NULL*/, int32_t* n_lig /*[S] out*/,
                                int32_t* lig_ptr /*[S+1] out*/, void* stream);

#define CBG_TYPE_UNIFORM 0    /* assign_atomtype / assign_genatomtype 'uniform': Gumbel arg-max over zero logits (init_lig.py:22-26) */
#define CBG_TYPE_ABSORBING 1  /* 'absorbing' (state 0); also used for 'zeros' (the caller allocates the [n,K] zero features) */
#define CBG_POS_GAUSSIAN 0            /* assign_molpos / assign_genpos 'gaussian' (init_lig.py:404-457) */
#define CBG_POS_ZERO_MEAN_GAUSSIAN 1  /* 'zero_mean_gaussian': the sample's mean is removed (de-novo only) */

typedef struct cbg_batch_spec {
  /* raw pockets (protein_featurizer.py:19-30 runs on the device) */
  const float* prot_pos;          /* [n_atoms,3] */
  const int32_t* prot_element;    /* [n_atoms] atomic numbers */
  const uint8_t* prot_backbone;   /* [n_atoms] is_backbone */
  const int32_t* prot_aa;         /* [n_atoms] atom_to_aa_type */
  const int32_t* prot_ptr;        /* [n_pockets+1] */
  int32_t n_pockets;
  int32_t repeat;
  const float* centre;            /* [n_pockets,3] from cbg_pocket_stats_f32 */
  /* context ligand atoms per pocket (NULL / NULL / NULL for de-novo): they come first in every sample, are centred like
   * the pocket, keep their types and get ctx_flag = 1, gen_flag = 0 */
  const float* ctx_pos;
  const int32_t* ctx_type;
  const int32_t* ctx_ptr;
  const int32_t* lig_ptr;         /* [S+1] from cbg_sample_ligand_sizes */
  const float* pos_noise;         /* [n_lig_total,3] standard normal (rows of context atoms are ignored) */
  const float* type_u;            /* [n_lig_total,K] uniform(0,1) or NULL unless type_dist == CBG_TYPE_UNIFORM */
  int32_t num_classes;
  int32_t type_dist;
  int32_t pos_dist;
  /* outputs = the flat batch of SURVEY.md section 8b (graph id = sample index) */
  float* protein_pos;             /* [S_atoms,3] centred */
  float* protein_atom_feature;    /* [S_atoms,7] */
  int64_t* protein_aa_type;       /* [S_atoms] */
  int64_t* protein_element_batch; /* [S_atoms] */
  float* protein_translation;     /* [S_atoms,3] the centre, per atom (translation.py:19) */
  float* ligand_pos;              /* [n_lig_total,3] */
  int64_t* ligand_atom_type;      /* [n_lig_total] */
  int64_t* ligand_element_batch;  /* [n_lig_total] */
  uint8_t* ligand_ctx_flag;       /* [n_lig_total] or NULL */
  uint8_t* ligand_gen_flag;       /* [n_lig_total] or NULL */
} cbg_batch_spec;

int32_t cbg_build_batch_f32(const cbg_batch_spec* spec, void* stream);

/* ---- SURVEY.md section 8 row f4: D3FG encoder `IPATransformer` (repo/modules/e3nn/itatransformer.py:14-145) --------------
 * X2H-only encoder (InvAttentionLayer :147-188, coordinates fixed) at hidden width 128 or 256 (configs/denovo/train/
 * d3fg_fg.yml:5: 256), then the rotation / translation / type heads and the SO(3) update (:127-145):
 *   eps_pos [N,3], h [N,H], o_next [N,3] (so3 vector), R_next [N,3,3], logits [N,K]
 * = IPATransformer.forward(x, o, h, batch_idx, lig_flag, gen_flag).  Weights: one blob = the global block of the denoiser
 * layout (edge-gate fields) | head block | num_sublayers layer blocks; the field table below is the single source of
 * truth the Python packer queries (cbgbench_b200/ipatransformer.py). */
int64_t cbg_ipa_head_floats(int32_t hidden);
int64_t cbg_ipa_layer_floats(int32_t hidden);
int32_t cbg_ipa_head_fields(void);
int32_t cbg_ipa_layer_fields(void);
const char* cbg_ipa_head_field_name(int32_t field);
const char* cbg_ipa_layer_field_name(int32_t field);
int64_t cbg_ipa_head_field_offset(int32_t hidden, int32_t field);
int64_t cbg_ipa_head_field_size(int32_t hidden, int32_t field);
int64_t cbg_ipa_layer_field_offset(int32_t hidden, int32_t field);
int64_t cbg_ipa_layer_field_size(int32_t hidden, int32_t field);
int64_t cbg_ipa_workspace_bytes(int64_t n_nodes, int32_t hidden);
int32_t cbg_ipa_forward_f32(const float* blob, int32_t hidden, int32_t num_sublayers /* num_layers * num_x2h */,
                            int32_t num_blocks, int32_t num_classes, const float* x /*[N,3]*/, const float* o /*[N,3]*/,
                            const float* h /*[N,hidden]*/, const int32_t* graph_ptr /*[B+1]*/, int32_t n_graphs,
                            int32_t max_graph_nodes, const uint8_t* lig_flag, const uint8_t* gen_flag, int64_t n_nodes,
                            int32_t k, float* eps_pos, float* h_out, float* o_next, float* r_next, float* logits,
                            void* workspace, int64_t workspace_bytes, void* stream);

/* ---- D3FG sampling (`difffg` / `difffg_v2`, repo/models/diffusion/difffg.py:174-246): one reverse step per call -------
 * Composed node arrays [protein | ligand per graph] live in the plan; the protein rows (x = C-alpha, o = backbone frame,
 * h = FG + residue embedding) are written once per batch by the host.  A step writes the ligand rows from the state
 * (fg_embed_kernel), runs the IPATransformer (cbg_ipa_launch) and applies the position / SO(3) / FG-type reverse updates
 * (fg_reverse_kernel, one warp per functional group) into the next state. */
typedef struct {
  const float* blob;              /* IPATransformer blob (cbg_ipa_*) */
  int32_t hidden, num_sublayers, num_blocks, num_classes, k;
  const int32_t* graph_ptr;       /* [n_graphs+1] composed rows per graph */
  int32_t n_graphs, max_graph_nodes;
  int64_t n_nodes;
  const uint8_t* lig_flag;        /* [N] composed order */
  const uint8_t* gen_flag;        /* [N] composed order */
  const int32_t* lig_node;        /* [n_lig] composed row of ligand row a */
  const uint8_t* gen_lig;         /* [n_lig] */
  int32_t n_lig;
  float* x;                       /* [N,3] composed positions */
  float* o;                       /* [N,3] composed so3 vectors */
  float* h;                       /* [N,hidden] composed node features */
  const float* fg_emb_t;          /* [num_classes,hidden] columns of ligand_fg_emb.weight */
  const float* fg_emb_b;          /* [hidden] ligand_fg_emb.bias */
  const float* lig_indicator;     /* [hidden] ligand_indicator(1) */
  const float* angle_x;           /* [T,n_bins] angular_distrib_inv.X */
  const double* angle_cdf;        /* [T,n_bins-1] inclusive float64 prefix sums of angular_distrib_inv.Y[:, :-1] */
  int32_t n_bins;
  void* workspace;
  int64_t workspace_bytes;
} cbg_fg_plan;

typedef struct {
  int32_t t;
  float pos_beta, pos_sigma, pos_sqrt_one_minus_beta, pos_noise_scale;  /* b, sqrt(1 - abar), sqrt(1 - b), [t != 0] sqrt(b) */
  float rot_std;                  /* angular_distrib_inv.stddevs[t] */
  int32_t rot_gaussian;           /* angular_distrib_inv.approx_flag[t] */
  int32_t rot_noise;              /* t > 1 */
  float log_alphas_cumprod_prev, log_one_minus_alphas_cumprod_prev, log_alpha, log_one_minus_alpha;
} cbg_fg_coef;

int64_t cbg_fg_workspace_bytes(int64_t n_nodes, int32_t hidden, int32_t num_classes);
/* x_t / c_t / o_t [n_lig,3|K|3] -> x_next / c_next / o_next; draws: pos_noise [n_lig,3] N(0,1), rot_draws [n_lig,6] =
 * axis N(0,1)^3 | bin uniform | in-bin uniform | Gaussian-branch N(0,1), type_u [n_lig,K] U[0,1) */
int32_t cbg_fg_step_f32(const cbg_fg_plan* plan, cbg_fg_coef coef, const float* x_t, const float* c_t, const float* o_t,
                        const float* pos_noise, const float* rot_draws, const float* type_u, float* x_next, float* c_next,
                        float* o_next, void* stream);

/* The reverse update alone (testing hook): fg_reverse_kernel on caller-given encoder rows.  eps_pos / o_pred / logits are
 * composed rows [*,3|3|K], read at lig_node[a]; the state and the draws are as for cbg_fg_step_f32.  Of the plan only
 * n_lig, num_classes, lig_node, gen_lig, angle_x, angle_cdf and n_bins are read.  theta [n_lig] (or NULL) receives the
 * drawn rotation angle (0 when coef.rot_noise is 0). */
int32_t cbg_fg_reverse_f32(const cbg_fg_plan* plan, cbg_fg_coef coef, const float* eps_pos, const float* o_pred,
                           const float* logits, const float* x_t, const float* c_t, const float* o_t,
                           const float* pos_noise, const float* rot_draws, const float* type_u, float* x_next,
                           float* c_next, float* o_next, float* theta, void* stream);

/* ---- validation loss: D3FG.forward in eval mode (`difffg` / `difffg_v2`, difffg.py:65-171 / :283-389) ------------------
 *
 * The plan holds n_rep replicas of one batch of B graphs and n1 = n_lig / n_rep functional groups, replica-major: graph
 * r*B + g and ligand row r*n1 + a are graph g and FG a of the batch, noised at replica r's timestep.  Its protein rows of
 * x / o / h are written by the host (once per batch, tiled n_rep times); angle_x / angle_cdf point at the FORWARD angular
 * tables (rot_scheduler.angular_distrib_fwd).  The encoder does not see t, so the replicas share one pass.  One call
 * enqueues:
 *   fg_eval_noise_kernel   one warp per (replica, FG): CTNVPScheduler.forward_add_noise (diffusion_scheduler.py:117-134),
 *                          RotVPScheduler.forward_add_noise (:531-556; o_t = log(exp(e) exp(sqrt(abar_rot) o_0)), e drawn
 *                          from angular_distrib_fwd, no zeroing at small t) and TypeVPScheduler.forward_add_noise (:339-346,
 *                          Gumbel-max over q(v_t | v_0)), each only where gen_lig is set, then the ligand rows of x / o / h
 *   cbg_ipa_launch         the IPATransformer over all n_rep * B graphs
 *   fg_eval_loss_kernel    one CTA per (replica, graph), over its generated FGs in a fixed order: the position loss
 *                          (score form: ||eps_pred - eps||^2, get_score_loss; denoise form: ||x_pred - x_0||^2, get_loss),
 *                          rotation_matrix_cosine_loss (difffg.py:16-31) and the type KL / decoder NLL at t == 0
 *                          (TypeVPScheduler.get_loss, :348-418)
 *   fg_eval_reduce_kernel  per replica: scatter_mean(...).mean() over graphs 0 .. (last graph with a generated FG)
 * No atomics: repeated calls are bit-identical. */
#define CBG_FG_LOSS_SCORE 0     /* difffg: get_score_loss(score_in=False) on the encoder's eps_pos */
#define CBG_FG_LOSS_DENOISE 1   /* difffg_v2: get_loss(type='denoise') on the encoder's eps_pos as x_pred */

typedef struct {                 /* one replica's timestep t: the reference's fp32 torch expressions, evaluated on the host */
  int32_t t;
  float pos_sqrt_alphas_cumprod;            /* pos_scheduler.alphas_cumprod[t].sqrt() */
  float pos_sqrt_one_minus_alphas_cumprod;  /* (1 - pos_scheduler.alphas_cumprod[t]).sqrt() */
  float rot_sqrt_alphas_cumprod;            /* rot_scheduler.alphas_cumprod[t].sqrt() */
  float rot_std;                            /* angular_distrib_fwd.stddevs[t] = sqrt(1 - rot abar[t]) */
  int32_t rot_gaussian;                     /* angular_distrib_fwd.approx_flag[t] */
  float log_alphas_cumprod, log_one_minus_alphas_cumprod;            /* type_scheduler tables at t */
  float log_alphas_cumprod_prev, log_one_minus_alphas_cumprod_prev;  /* ... at max(t - 1, 0) */
  float log_alpha, log_one_minus_alpha;                              /* log_alphas_v / log_one_minus_alphas_v at t */
  int32_t t_is_zero;                        /* 1: the type loss is the decoder NLL instead of the KL */
} cbg_fg_eval_coef;

/* coefs: host array [n_rep], 1 <= n_rep <= 64; every t must index the plan's angle tables.  loss_form: CBG_FG_LOSS_*.
 * The batch: x0 [n1,3] (C-alpha of ligand_pos_heavyatom), v0 [n1] (ligand_type_fg), o0 [n1,3] (ligand_o_fg).  Draws from
 * the caller: pos_noise [n_rep,n1,3] N(0,1), rot_draws [n_rep,n1,6] as for cbg_fg_step_f32, type_u [n_rep,n1,K] U[0,1).
 * Outputs: xt [n_rep,n1,3]; ot [n_rep,n1,3] or NULL; vt [n_rep,n1]; pred [n_rep,n1,3] (eps_pred or x_pred);
 * score [n_rep,2,n1,3] = score_0, score_pred (score = eps * sqrt(1 - abar)), required for CBG_FG_LOSS_SCORE, ignored
 * otherwise; c_pred = softmax(logits) [n_rep,n1,K]; R_pred [n_rep,n1,3,3] (the encoder's R_next); R0 = exp(o0) [n1,3,3];
 * graph_loss [n_rep*B,4] = per-graph pos, rot, fg means over generated FGs (0 without any) and their count;
 * rep_loss [n_rep,3] = pos, rot, fg (NaN when no FG is generated).  The plan's workspace is sized by
 * cbg_fg_workspace_bytes.  Refuses NULL pointers, n_rep, K, a plan that is not n_rep replicas, t < 0 and a missing,
 * unaligned or small workspace before touching the device. */
int32_t cbg_fg_eval_loss_f32(const cbg_fg_plan* plan, const cbg_fg_eval_coef* coefs, int32_t n_rep, int32_t loss_form,
                             const float* x0, const int64_t* v0, const float* o0, const float* pos_noise,
                             const float* rot_draws, const float* type_u, float* xt, float* ot, int64_t* vt, float* pred,
                             float* score, float* c_pred, float* R_pred, float* R0, float* graph_loss, float* rep_loss,
                             void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CBG_B200_H_ */
