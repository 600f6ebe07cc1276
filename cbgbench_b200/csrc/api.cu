// C-ABI of libcbg_b200.so (declared in include/cbg_b200.h) and the per-forward orchestration.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include <vector>

#include <nvtx3/nvToolsExt.h>     // header-only NVTX v3: ranges show up in Nsight Systems, cost nothing without a tool attached

#include "../../include/cbg_b200.h"
#include "cbg_kernels.cuh"

long long g_cbg_launches = 0;
int g_cbg_prof_on = 0;

namespace {
// RAII NVTX range (SURVEY.md section 5: tracing)
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};
struct ProfMark { int family; int is_end; cudaEvent_t ev; };
std::vector<ProfMark> g_prof_marks;
const char* const kFamilyNames[CBG_K_COUNT] = {"knn", "edge_gate", "node_gemm", "x2h_k", "x2h_v", "h2x",
                                               "classifier", "step_init", "reverse", "misc"};
}  // namespace

void cbg_prof_mark(int family, int is_end, cudaStream_t st) {
  cudaEvent_t ev;
  if (cudaEventCreate(&ev) != cudaSuccess) return;
  cudaEventRecord(ev, st);
  g_prof_marks.push_back({family, is_end, ev});
}

static thread_local char g_err[1024] = "";

void cbg_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

namespace {

struct FieldInfo { const char* name; long long size; };
const FieldInfo kGlobalFields[] = {
#define X(name, n) {#name, (long long)(n)},
    CBG_GLOBAL_FIELDS(X)
#undef X
};
const FieldInfo kLayerFields[] = {
#define X(name, n) {#name, (long long)(n)},
    CBG_LAYER_FIELDS(X)
#undef X
};

// workspace carve-up
struct Workspace {
  float4* x4;
  float* h;
  float* plane[CBG_NPLANES];   // X2H: pj_k, pj_v, pi_k, pi_v, q
  float* hplane[CBG_NPLANES];  // H2X: same five planes (separate so the H2X chain can overlap the next X2H GEMM)
  float* w;
  int* nbr;
  int* snbr;                   // static-only neighbour lists (R-cache build)
  float* sew;                  // edge gates of the static-only lists (valid when the plan has an R-cache)
  int* depth;                  // receptive-field pruning: per-node depth, nodes ordered by depth, counts
  int* order;
  int* cnt;
  float* ew;
  float* dx;
  float* hw;                   // H2X on the wgmma tile kernel: alpha * e_w of the generated nodes' edges, compact [n_gen,32,16]
  int* tickets;                // 64 work counters of the X2H launches of one step (dynamic node scheduling)
  unsigned char* fstat;        // per node: all 32 in-edges static this step (written by the edge gate when an R-cache is used)
  StepIO* io;                  // per-step pointers / coefficients of a graph-replayed step (cbg_sample_step_graph_f32)
  size_t bytes;
};

Workspace carve(void* base, long long n_nodes, long long n_gen) {
  Workspace ws;
  size_t off = 0;
  char* b = (char*)base;
  auto take = [&](size_t nbytes) { char* p = b ? b + off : nullptr; off += align256(nbytes); return p; };
  ws.x4 = (float4*)take((size_t)n_nodes * sizeof(float4));
  ws.h = (float*)take((size_t)n_nodes * CBG_H * 4);
  for (int p = 0; p < CBG_NPLANES; ++p) ws.plane[p] = (float*)take((size_t)n_nodes * CBG_H * 4);
  for (int p = 0; p < CBG_NPLANES; ++p) ws.hplane[p] = (float*)take((size_t)n_nodes * CBG_H * 4);
  ws.w = (float*)take((size_t)n_nodes * CBG_KMAX * CBG_HEADS * 4);
  ws.nbr = (int*)take((size_t)n_nodes * CBG_KMAX * 4);
  ws.snbr = (int*)take((size_t)n_nodes * CBG_KMAX * 4);
  ws.sew = (float*)take((size_t)n_nodes * CBG_KMAX * 4);
  ws.depth = (int*)take((size_t)n_nodes * 4);
  ws.order = (int*)take((size_t)n_nodes * 4);
  ws.cnt = (int*)take(96 * 4);
  ws.ew = (float*)take((size_t)n_nodes * CBG_KMAX * 4);
  ws.dx = (float*)take((size_t)(n_gen > 0 ? n_gen : 1) * 16);
  ws.hw = (float*)take((size_t)(n_gen > 0 ? n_gen : 1) * CBG_KMAX * CBG_HEADS * 4);
  ws.fstat = (unsigned char*)take((size_t)n_nodes);
  ws.tickets = (int*)take(64 * sizeof(int));
  ws.io = (StepIO*)take(sizeof(StepIO));
  ws.bytes = off;
  return ws;
}

int check_ws(const void* workspace, size_t have, long long n_nodes, long long n_gen, Workspace* out) {
  if (n_nodes < 0 || n_gen < 0) { cbg_set_error("negative size"); return 1; }
  Workspace ws = carve(const_cast<void*>(workspace), n_nodes, n_gen);
  if (!workspace || have < ws.bytes) {
    cbg_set_error("workspace too small: have %zu bytes, need %zu (cbg_workspace_bytes)", have, ws.bytes);
    return 1;
  }
  if (((uintptr_t)workspace & 255) != 0) { cbg_set_error("workspace must be 256-byte aligned"); return 1; }
  *out = ws;
  return 0;
}

// The CBG_* switches of the orchestration, read from the environment once per process (on first use).  "0" turns a
// default-on switch off.
struct Switches {
  int node_gemm;      // CBG_NODE_GEMM: simt 0 (fp32 SIMT), tf32 1 (3xTF32), anything else 2 (wgmma f16, (hi, lo) split)
  bool overlap;       // CBG_OVERLAP: side streams (AuxStream) instead of the caller's stream alone
  bool prune;         // CBG_PRUNE: receptive-field pruning of the sampling step (exact)
  bool gate_compact;  // CBG_GATE_COMPACT: compact the moving edges before their gates (ws.w is free until the first X2H)
  bool dyn_sched;     // CBG_DYN_SCHED: dynamic node scheduling of the X2H kernels (work counters), else round-robin
  bool static_fast;   // CBG_STATIC_FAST: edge_setup fast path for nodes whose 32 in-edges are all static (R-cache)
};
bool env_on(const char* name) {
  const char* e = getenv(name);
  return !(e && strcmp(e, "0") == 0);
}
Switches& switches() {
  static Switches s = [] {
    const char* g = getenv("CBG_NODE_GEMM");
    const int node_gemm = (g && strcmp(g, "simt") == 0) ? 0 : ((g && strcmp(g, "tf32") == 0) ? 1 : 2);
    return Switches{node_gemm, env_on("CBG_OVERLAP"), env_on("CBG_PRUNE"), env_on("CBG_GATE_COMPACT"),
                    env_on("CBG_DYN_SCHED"), env_on("CBG_STATIC_FAST")};
  }();
  return s;
}

int launch_node_gemm(const NodeGemmArgs& a, cudaStream_t st) {
  const int impl = switches().node_gemm;
  return impl == 2 ? cbg_launch_node_gemm_f16(a, st) : (impl == 1 ? cbg_launch_node_gemm_tc(a, st) : cbg_launch_node_gemm(a, st));
}

// The node projections of one sub-layer (cbg_layout.h): five planes pj_k, pj_v, pi_k, pi_v, q, the last one through
// the q head (LN -> ReLU -> second Linear).  A launch computes all of them, the source planes Pj (0..1) or the
// destination planes Pi / q (2..4).
enum SubLayer { kX2H = 0, kH2X = 1 };
enum class Planes { kAll, kSrc, kDst };
NodeGemmArgs node_gemm_args(const float* L, SubLayer sub, Planes shape, const float* a, const int* row_idx, int n_rows,
                            float* const planes[CBG_NPLANES]) {
  auto field = [&](int x2h, int h2x) { return L + cbg_layout::layer_offset(sub == kX2H ? x2h : h2x); };
  const int first = shape == Planes::kDst ? 2 : 0;
  NodeGemmArgs g{};
  g.a = a; g.row_idx = row_idx; g.n_rows = n_rows;
  g.wt = field(CBG_LF_X2H_NODE_WT, CBG_LF_H2X_NODE_WT) + first * CBG_H;
  g.bias = field(CBG_LF_X2H_NODE_B, CBG_LF_H2X_NODE_B) + first * CBG_H;
  g.ldw = 640;
  g.n_planes = shape == Planes::kAll ? 5 : (shape == Planes::kSrc ? 2 : 3);
  g.has_q = shape != Planes::kSrc;
  for (int p = 0; p < g.n_planes - g.has_q; ++p) g.out[p] = planes[first + p];
  if (g.has_q) {
    g.q_ln = field(CBG_LF_X2H_Q_LN, CBG_LF_H2X_Q_LN);
    g.q_w1t = field(CBG_LF_X2H_Q_W1T, CBG_LF_H2X_Q_W1T);
    g.q_b1 = field(CBG_LF_X2H_Q_B1, CBG_LF_H2X_Q_B1);
    g.out_q = planes[4];
  }
  g.tc_planes = field(CBG_LF_X2H_NODE_TC, CBG_LF_H2X_NODE_TC); g.tc_first_plane = first;
  g.tch_planes = field(CBG_LF_X2H_NODE_TCH, CBG_LF_H2X_NODE_TCH);
  return g;
}

// Side streams of the denoiser pass: the H2X chain of layer l overlaps the X2H node GEMM of layer l+1 (that GEMM needs
// only h).  Fork/join with events.
struct AuxStream {
  cudaStream_t s2 = nullptr, s3 = nullptr, s4 = nullptr;   // H2X chain, X2H source-plane GEMM, H2X destination GEMM
  cudaEvent_t ev_h = nullptr, ev_x = nullptr, ev_h0 = nullptr, ev_p = nullptr, ev_gi = nullptr;
  int state = -1;   // -1 unknown, 0 disabled, 1 ready
};
constexpr int kMaxDevices = 64;
AuxStream g_aux_dev[kMaxDevices];   // streams and events belong to a device: one set per device the caller uses

// The current device's side streams (created on first use), or nullptr when overlap is off or unavailable.
AuxStream* aux_streams() {
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return nullptr;
  AuxStream& a = g_aux_dev[dev];
  if (a.state < 0) {
    a.state = switches().overlap &&
              cudaStreamCreateWithFlags(&a.s2, cudaStreamNonBlocking) == cudaSuccess &&
              cudaStreamCreateWithFlags(&a.s3, cudaStreamNonBlocking) == cudaSuccess &&
              cudaStreamCreateWithFlags(&a.s4, cudaStreamNonBlocking) == cudaSuccess &&
              cudaEventCreateWithFlags(&a.ev_h, cudaEventDisableTiming) == cudaSuccess &&
              cudaEventCreateWithFlags(&a.ev_x, cudaEventDisableTiming) == cudaSuccess &&
              cudaEventCreateWithFlags(&a.ev_h0, cudaEventDisableTiming) == cudaSuccess &&
              cudaEventCreateWithFlags(&a.ev_p, cudaEventDisableTiming) == cudaSuccess &&
              cudaEventCreateWithFlags(&a.ev_gi, cudaEventDisableTiming) == cudaSuccess;
  }
  return a.state ? &a : nullptr;
}

// Receptive-field pruning of a plan's denoiser pass (only when the caller consumes nothing but the generated /
// classified rows): layer l updates h only for the nodes that can still reach such a row through the remaining layers.
bool plan_prunes(const cbg_sample_plan& p) {
  return p.prune != 0 && switches().prune && p.num_layers > 0 && (p.n_gen > 0 || p.n_lig > 0);
}

// One H2X sub-layer on the current h and the layer-input x: source planes Pj for all nodes, or for the first
// *src_rows_dev nodes of ws.order (pruned: the generated atoms and their neighbours), destination planes Pi / q for the
// generated nodes, then their coordinate update.  With side streams the destination GEMM runs on aux->s4 beside the
// source GEMM (both wait for the caller's fork) and the rest on st.
int run_h2x(const float* L, const Workspace& ws, long long n_nodes, const int* gen_idx, int n_gen,
            const int* src_rows_dev, const AuxStream* aux, cudaStream_t st) {
  NodeGemmArgs gj = node_gemm_args(L, kH2X, Planes::kSrc, ws.h, src_rows_dev ? ws.order : nullptr, (int)n_nodes, ws.hplane);
  gj.n_rows_dev = src_rows_dev;
  if (int rc = launch_node_gemm(gj, st)) return rc;
  const NodeGemmArgs gi = node_gemm_args(L, kH2X, Planes::kDst, ws.h, gen_idx, n_gen, ws.hplane);
  if (int rc = launch_node_gemm(gi, aux ? aux->s4 : st)) return rc;
  if (aux) {
    CBG_CUDA_OK(cudaEventRecord(aux->ev_gi, aux->s4));
    CBG_CUDA_OK(cudaStreamWaitEvent(st, aux->ev_gi, 0));
  }
  EdgeArgs x{};
  x.x4 = ws.x4; x.nbr = ws.nbr; x.ew = ws.ew;
  x.pj_k = ws.hplane[0]; x.pj_v = ws.hplane[1]; x.pi_k = ws.hplane[2]; x.pi_v = ws.hplane[3]; x.q = ws.hplane[4];
  x.layer = L; x.h = ws.h; x.node_idx = gen_idx; x.n_nodes = n_gen; x.dx = ws.dx;
  x.w = ws.hw;        // the X2H kernels of the next layer use ws.w while this chain runs
  if (int rc = cbg_launch_h2x(x, st)) return rc;
  return cbg_launch_apply_dx(ws.x4, gen_idx, ws.dx, n_gen, st);
}

// The denoiser pass of a plan on an initialised workspace (x4, h valid): graph build, edge gate, the layers.  The
// classified rows are the plan's ligand rows.
int run_denoiser(const cbg_sample_plan& p, const Workspace& ws, cudaStream_t st) {
  // One set of side streams / fork-join events per device (g_aux_dev): two host threads enqueueing denoiser passes on the
  // same GPU must not interleave their cudaEventRecord / cudaStreamWaitEvent pairs.  Enqueueing is serialised here; the
  // GPU work itself still overlaps across the callers' streams.
  static std::mutex core_mutex;
  std::lock_guard<std::mutex> core_lock(core_mutex);
  NvtxRange nvtx_core("cbg:denoiser");
  const long long n_nodes = p.n_nodes;
  const int num_layers = p.num_layers, n_gen = p.n_gen;
  const bool static_lists = p.static_lists != 0 || p.rcache != nullptr;   // the R-cache is indexed by the static lists
  if (n_nodes > 0x7fffffffLL / (CBG_KMAX * CBG_HEADS)) { cbg_set_error("n_nodes too large for 32-bit indexing"); return 1; }
  if (int rc = cbg_launch_knn(ws.x4, p.graph_ptr, p.n_graphs, p.max_graph_nodes, p.mode, p.k, p.r_max, 0,
                              static_lists ? ws.snbr : nullptr, ws.nbr, st)) return rc;
  const float* layers = p.blob + cbg_layout::kGlobalFloats;
  const bool prune = plan_prunes(p);
  AuxStream* const aux = n_gen > 0 ? aux_streams() : nullptr;
  const bool tickets = switches().dyn_sched && 2 * num_layers <= 64;
  if (tickets) CBG_CUDA_OK(cudaMemsetAsync(ws.tickets, 0, 64 * sizeof(int), st));
  // the edge gate and the pruning BFS both need only the neighbour table: run them side by side
  const bool fork_depth = prune && aux;
  if (fork_depth) {
    CBG_CUDA_OK(cudaEventRecord(aux->ev_h0, st));
    CBG_CUDA_OK(cudaStreamWaitEvent(aux->s3, aux->ev_h0, 0));
  }
  if (prune) {
    if (int rc = cbg_launch_depth(ws.nbr, p.graph_ptr, p.n_graphs, p.max_graph_nodes, n_nodes, p.gen_node, n_gen,
                                  p.lig_node, p.n_lig, num_layers, ws.depth, ws.order, ws.cnt,
                                  fork_depth ? aux->s3 : st)) return rc;
  }
  if (fork_depth) CBG_CUDA_OK(cudaEventRecord(aux->ev_p, aux->s3));
  if (int rc = cbg_launch_edge_gate(p.blob, ws.x4, ws.nbr, n_nodes, static_lists ? ws.sew : nullptr,
                                    switches().gate_compact ? (int*)ws.w : nullptr, ws.ew, st, ws.fstat)) return rc;
  if (fork_depth) CBG_CUDA_OK(cudaStreamWaitEvent(st, aux->ev_p, 0));
  cudaStream_t sx = aux ? aux->s2 : st;            // stream of the H2X chain
  bool x_pending = false;                          // an apply_dx on sx has not been joined yet
  for (int l = 0; l < num_layers; ++l) {
    const float* L = layers + (size_t)l * cbg_layout::kLayerFloats;
    NvtxRange nvtx_layer("cbg:layer");
    // ---- X2H: node planes, attention weights, aggregation (h updated in place)
    if (!prune) {
      const NodeGemmArgs g = node_gemm_args(L, kX2H, Planes::kAll, ws.h, nullptr, (int)n_nodes, ws.plane);
      if (int rc = launch_node_gemm(g, st)) return rc;          // reads h only: may overlap the previous H2X chain
    } else if (switches().node_gemm == 2) {
      // one launch: source planes Pj for every node a needed destination can gather (depth >= l-1), destination planes
      // Pi / q for the needed destinations only (depth >= l); both lists are prefixes of ws.order
      NodeGemmArgs g = node_gemm_args(L, kX2H, Planes::kAll, ws.h, ws.order, (int)n_nodes, ws.plane);
      g.n_rows_dev = ws.cnt + l; g.n_dst_dev = ws.cnt + l + 1;
      if (int rc = launch_node_gemm(g, st)) return rc;
    } else {
      NodeGemmArgs gp = node_gemm_args(L, kX2H, Planes::kSrc, ws.h, ws.order, (int)n_nodes, ws.plane);
      gp.n_rows_dev = ws.cnt + l;
      if (aux) {                            // the two X2H GEMMs only read h: run them side by side
        CBG_CUDA_OK(cudaEventRecord(aux->ev_h0, st));
        CBG_CUDA_OK(cudaStreamWaitEvent(aux->s3, aux->ev_h0, 0));
      }
      if (int rc = launch_node_gemm(gp, aux ? aux->s3 : st)) return rc;
      if (aux) CBG_CUDA_OK(cudaEventRecord(aux->ev_p, aux->s3));
      NodeGemmArgs gd = node_gemm_args(L, kX2H, Planes::kDst, ws.h, ws.order, (int)n_nodes, ws.plane);
      gd.n_rows_dev = ws.cnt + l + 1;
      if (int rc = launch_node_gemm(gd, st)) return rc;
      if (aux) CBG_CUDA_OK(cudaStreamWaitEvent(st, aux->ev_p, 0));
    }
    if (aux && x_pending) { CBG_CUDA_OK(cudaStreamWaitEvent(st, aux->ev_x, 0)); x_pending = false; }
    EdgeArgs e{};
    e.x4 = ws.x4; e.nbr = ws.nbr; e.ew = ws.ew;
    e.pj_k = ws.plane[0]; e.pj_v = ws.plane[1]; e.pi_k = ws.plane[2]; e.pi_v = ws.plane[3]; e.q = ws.plane[4];
    e.layer = L; e.w = ws.w; e.h = ws.h; e.node_idx = nullptr; e.n_nodes = (int)n_nodes; e.dx = nullptr;
    if (prune) { e.node_idx = ws.order; e.n_nodes_dev = ws.cnt + l + 1; }
    if (tickets) e.ticket = ws.tickets + 2 * l;
    if (p.rcache) {
      const size_t per = (size_t)n_nodes * (CBG_KMAX * CBG_H);
      e.rc_k = p.rcache + (size_t)(2 * l) * per;
      e.rc_v = p.rcache + (size_t)(2 * l + 1) * per;
      e.fstat = switches().static_fast ? ws.fstat : nullptr;
    }
    if (int rc = cbg_launch_x2h(e, st)) return rc;
    if (n_gen <= 0) continue;   // nothing moves: H2X output is multiplied by gen_flag == 0
    if (aux) {
      CBG_CUDA_OK(cudaEventRecord(aux->ev_h, st));
      CBG_CUDA_OK(cudaStreamWaitEvent(sx, aux->ev_h, 0));
      CBG_CUDA_OK(cudaStreamWaitEvent(aux->s4, aux->ev_h, 0));
    }
    // ---- H2X (uses the NEW h and the layer-input x); pruned: Pj for depth == top (generated atoms + neighbours)
    if (int rc = run_h2x(L, ws, n_nodes, p.gen_node, n_gen, prune ? ws.cnt + num_layers : nullptr, aux, sx)) return rc;
    if (aux) { CBG_CUDA_OK(cudaEventRecord(aux->ev_x, sx)); x_pending = true; }
  }
  if (aux && x_pending) CBG_CUDA_OK(cudaStreamWaitEvent(st, aux->ev_x, 0));   // join
  return 0;
}

// DiffBP's denoiser pass and heads: run_denoiser, the classifier on the ligand rows into `logits`, their output
// coordinates into x_pred, then the CoM head (CoMPredictor.forward, diffbp.py:80-101): the ligand rows of x4 get the
// step's INPUT coordinates x_t back, then the head's own edge gate and com_layers x H2X on the denoiser's final h move
// the generated rows.  Afterwards the ligand rows of x4 hold x_com.  Shared by the sampling step and the validation loss.
int run_bp_denoiser(const cbg_sample_plan& p, const float* com_blob, int com_layers, const Workspace& ws,
                    const float* x_t, float* logits, float* x_pred, cudaStream_t st) {
  if (int rc = run_denoiser(p, ws, st)) return rc;
  if (int rc = cbg_launch_classifier(p.blob, ws.h, p.lig_node, p.n_lig, p.num_classes, logits, st)) return rc;
  if (int rc = cbg_launch_gather_x(ws.x4, p.lig_node, p.n_lig, x_pred, st)) return rc;
  if (int rc = cbg_launch_scatter_x(x_t, p.lig_node, p.n_lig, ws.x4, st)) return rc;
  if (p.n_gen <= 0 || com_layers <= 0) return 0;
  if (int rc = cbg_launch_edge_gate_rows(com_blob, ws.x4, ws.nbr, p.gen_node, p.n_gen, ws.ew, st)) return rc;
  const int* src_rows_dev = plan_prunes(p) ? ws.cnt + p.num_layers : nullptr;   // run_denoiser built ws.order / ws.cnt
  const float* layers = com_blob + cbg_layout::kGlobalFloats;
  for (int l = 0; l < com_layers; ++l) {
    if (int rc = run_h2x(layers + (size_t)l * cbg_layout::kLayerFloats, ws, p.n_nodes, p.gen_node, p.n_gen, src_rows_dev,
                         nullptr, st)) return rc;
  }
  return 0;
}

// DiffBP scratch in the attention-weight buffer (free after the layers): logits [n_lig,K] | output coordinates [n_lig,3]
struct BpScratch { float* logits; float* x_pred; };
BpScratch bp_scratch(const Workspace& ws, int n_lig, int num_classes) {
  return {ws.w, ws.w + align256((size_t)n_lig * num_classes * 4) / 4};
}

// Prologue of the plan-driven entry points: the plan and the entry point's other required arguments (args_ok; null_msg
// is the error otherwise), a workspace that fits the plan, a class count the classifier supports.
int open_plan(const cbg_sample_plan* plan, bool args_ok, const char* null_msg, Workspace* ws) {
  if (!plan || !args_ok) { cbg_set_error("%s", null_msg); return 1; }
  if (int rc = check_ws(plan->workspace, plan->workspace_bytes, plan->n_nodes, plan->n_gen, ws)) return rc;
  const int K = plan->num_classes;
  if (K < 1 || K > CBG_MAXCLS) { cbg_set_error("num_classes=%d outside [1,%d]", K, CBG_MAXCLS); return 1; }
  return 0;
}

// The validation losses run noised copies of one batch as one plan, replica-major: n_t timesteps of `copies` replicas
// each (n_rep = n_t * copies, at most CBG_EVAL_MAX_REPLICAS).
int check_replicas(const cbg_sample_plan& p, int n_t, int copies = 1) {
  const int max_t = CBG_EVAL_MAX_REPLICAS / copies;
  if (n_t < 1 || n_t > max_t) { cbg_set_error("%s=%d outside [1,%d]", copies == 1 ? "n_rep" : "n_t", n_t, max_t); return 1; }
  const int n_rep = n_t * copies;
  if (p.n_lig < n_rep || p.n_lig % n_rep || p.n_graphs % n_rep) {
    cbg_set_error("plan (n_lig=%d, n_graphs=%d) is not %d replicas of one batch", p.n_lig, p.n_graphs, n_rep); return 1;
  }
  return 0;
}

// Prologue of the validation-loss entry points: open_plan, check_replicas, the batch block of the kernels' arguments and
// h reset to h_static (the noise kernel then writes the ligand rows).  Checks an entry point makes after it leave only
// that reset behind when they fail.
int open_eval(const cbg_sample_plan* plan, bool args_ok, const char* null_msg, int n_t, int copies, const float* x0,
              const int64_t* v0, Workspace* ws, EvalBatch* b, cudaStream_t st) {
  if (int rc = open_plan(plan, args_ok, null_msg, ws)) return rc;
  if (int rc = check_replicas(*plan, n_t, copies)) return rc;
  b->n_lig = plan->n_lig; b->n_graphs = plan->n_graphs; b->num_classes = plan->num_classes;
  b->lig_node = plan->lig_node; b->graph_ptr = plan->graph_ptr; b->gen = plan->gen_lig;
  b->x0 = x0; b->v0 = (const long long*)v0; b->emb_wt = plan->emb_wt; b->h_lig_bias = plan->h_lig_bias;
  b->x4 = ws->x4; b->h = ws->h;
  CBG_CUDA_OK(cudaMemcpyAsync(ws->h, plan->h_static, (size_t)plan->n_nodes * CBG_H * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// cached device scratch for the *_host entry points: one per DEVICE (the buffers belong to the device that was current
// when they were allocated); the weight blob is re-uploaded whenever the caller's (version, size, host pointer) changes -
// the version is a process-unique id handed out by the Python side, so two models never alias
struct HostCache {
  void* dev = nullptr;
  size_t bytes = 0;
  float* blob = nullptr;
  long long blob_floats = 0;
  long long blob_version = -1;
  const void* blob_host = nullptr;
};
HostCache g_cache_dev[kMaxDevices];

HostCache* host_cache() {
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return nullptr;
  return &g_cache_dev[dev];
}

int cache_reserve(HostCache& c, size_t bytes) {
  if (c.bytes >= bytes) return 0;
  if (c.dev) CBG_CUDA_OK(cudaFree(c.dev));
  c.dev = nullptr; c.bytes = 0;
  CBG_CUDA_OK(cudaMalloc(&c.dev, bytes));
  c.bytes = bytes;
  return 0;
}

}  // namespace

extern "C" {

int32_t cbg_version(void) { return 100; }
const char* cbg_last_error(void) { return g_err; }
int64_t cbg_launch_count(void) { return g_cbg_launches; }

int32_t cbg_set_edge_impl(int32_t impl, int32_t warps) { return cbg_edge_set_impl(impl, warps); }
int32_t cbg_debug_x2h_trace(int64_t* buf_dev, int32_t max_tiles) {
  cbg_x2h_tc_set_trace((long long*)buf_dev, max_tiles);
  return 0;
}
int32_t cbg_debug_node_gemm_trace(int64_t* buf_dev) {
  cbg_node_gemm_f16_set_trace((long long*)buf_dev);
  return 0;
}
int32_t cbg_selftest_umma_f16(const void* a, const void* b, float* d, int32_t a_from_smem, void* stream) {
  if (!a || !b || !d) { cbg_set_error("cbg_selftest_umma_f16: null argument"); return 1; }
  return cbg_launch_umma_selftest(a, b, d, a_from_smem, (cudaStream_t)stream);
}
int32_t cbg_set_option(const char* key, int32_t value) {
  if (key && strcmp(key, "static_fast") == 0) { switches().static_fast = value != 0; return 0; }
  if (key && strcmp(key, "dyn_sched") == 0) { switches().dyn_sched = value != 0; return 0; }
  if (key && strcmp(key, "x2h_trace_off") == 0) { cbg_x2h_tc_set_trace(nullptr, 0); return 0; }
  cbg_set_error("cbg_set_option: unknown key '%s'", key ? key : "(null)");
  return 1;
}

int32_t cbg_profile_num_families(void) { return CBG_K_COUNT; }
const char* cbg_profile_family_name(int32_t i) { return (i >= 0 && i < CBG_K_COUNT) ? kFamilyNames[i] : nullptr; }
int32_t cbg_profile_enable(int32_t on) {
  g_cbg_prof_on = on ? 1 : 0;
  return 0;
}
int32_t cbg_profile_collect(double* ms_per_family, int64_t* launches_per_family) {
  for (int i = 0; i < CBG_K_COUNT; ++i) { ms_per_family[i] = 0.0; launches_per_family[i] = 0; }
  CBG_CUDA_OK(cudaDeviceSynchronize());
  for (size_t i = 0; i + 1 < g_prof_marks.size(); i += 2) {
    const ProfMark& a = g_prof_marks[i];
    const ProfMark& b = g_prof_marks[i + 1];
    if (a.is_end || !b.is_end || a.family != b.family) continue;   // unmatched bracket (error path)
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, a.ev, b.ev) == cudaSuccess) {
      ms_per_family[a.family] += ms;
      launches_per_family[a.family] += 1;
    }
  }
  for (auto& m : g_prof_marks) cudaEventDestroy(m.ev);
  g_prof_marks.clear();
  return 0;
}

int64_t cbg_blob_global_floats(void) { return cbg_layout::kGlobalFloats; }
int64_t cbg_blob_layer_floats(void) { return cbg_layout::kLayerFloats; }
int32_t cbg_blob_num_fields(int32_t section) { return section == 0 ? (int)CBG_GF_COUNT : (section == 1 ? (int)CBG_LF_COUNT : -1); }
const char* cbg_blob_field_name(int32_t section, int32_t idx) {
  if (section == 0 && idx >= 0 && idx < CBG_GF_COUNT) return kGlobalFields[idx].name;
  if (section == 1 && idx >= 0 && idx < CBG_LF_COUNT) return kLayerFields[idx].name;
  return nullptr;
}
int64_t cbg_blob_field_size(int32_t section, int32_t idx) {
  if (section == 0 && idx >= 0 && idx < CBG_GF_COUNT) return kGlobalFields[idx].size;
  if (section == 1 && idx >= 0 && idx < CBG_LF_COUNT) return kLayerFields[idx].size;
  return -1;
}
int64_t cbg_blob_field_offset(int32_t section, int32_t idx) {
  if (section == 0 && idx >= 0 && idx < CBG_GF_COUNT) return cbg_layout::global_offset(idx);
  if (section == 1 && idx >= 0 && idx < CBG_LF_COUNT) return cbg_layout::layer_offset(idx);
  return -1;
}

int64_t cbg_rcache_bytes(int64_t n_nodes, int32_t num_layers) {
  if (n_nodes < 0 || num_layers < 0) return -1;
  return (int64_t)2 * num_layers * n_nodes * (CBG_KMAX * CBG_H) * (int64_t)sizeof(float);
}

int64_t cbg_workspace_bytes(int64_t n_nodes, int64_t n_gen) {
  if (n_nodes < 0 || n_gen < 0) return -1;
  return (int64_t)carve(nullptr, n_nodes, n_gen).bytes;
}

int32_t cbg_build_neighbors_f32(const float* x, const int32_t* graph_ptr, int32_t n_graphs, int64_t n_nodes,
                                int32_t max_graph_nodes, int32_t mode, int32_t k, float r_max, int32_t* nbr,
                                void* workspace, size_t workspace_bytes, void* stream) {
  Workspace ws;
  if (int rc = check_ws(workspace, workspace_bytes, n_nodes, 0, &ws)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  // flags are irrelevant for the neighbour search: pack with zeros
  CBG_CUDA_OK(cudaMemsetAsync(ws.nbr, 0, (size_t)n_nodes, st));   // reuse as a zero flag array
  if (int rc = cbg_launch_pack_x4(x, (const unsigned char*)ws.nbr, (const unsigned char*)ws.nbr, n_nodes, ws.x4, st)) return rc;
  return cbg_launch_knn(ws.x4, graph_ptr, n_graphs, max_graph_nodes, mode, k, r_max, 0, nullptr, nbr, st);
}

int32_t cbg_edge_gate_f32(const float* blob, const float* x, const int32_t* nbr, int64_t n_nodes, float* ew,
                          void* workspace, size_t workspace_bytes, void* stream) {
  Workspace ws;
  if (int rc = check_ws(workspace, workspace_bytes, n_nodes, 0, &ws)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  CBG_CUDA_OK(cudaMemsetAsync(ws.nbr, 0, (size_t)n_nodes, st));
  if (int rc = cbg_launch_pack_x4(x, (const unsigned char*)ws.nbr, (const unsigned char*)ws.nbr, n_nodes, ws.x4, st)) return rc;
  return cbg_launch_edge_gate(blob, ws.x4, nbr, n_nodes, nullptr, nullptr, ew, st);
}

int32_t cbg_denoiser_forward_f32(const float* blob, int32_t num_layers, int32_t num_classes, const float* x,
                                 const float* h, const int32_t* graph_ptr, int32_t n_graphs,
                                 int32_t max_graph_nodes, const uint8_t* lig_flag, const uint8_t* gen_flag,
                                 const int32_t* gen_idx, int32_t n_gen, const int32_t* cls_idx, int32_t n_cls,
                                 int64_t n_nodes, int32_t mode, int32_t k, float r_max, int32_t stop_after_layers,
                                 float* x_out, float* h_out, float* logits_out, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  Workspace ws;
  if (int rc = check_ws(workspace, workspace_bytes, n_nodes, n_gen, &ws)) return rc;
  if (num_layers < 0) { cbg_set_error("num_layers < 0"); return 1; }
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = cbg_launch_pack_x4(x, lig_flag, gen_flag, n_nodes, ws.x4, st)) return rc;
  CBG_CUDA_OK(cudaMemcpyAsync(ws.h, h, (size_t)n_nodes * CBG_H * 4, cudaMemcpyDeviceToDevice, st));
  // no classified rows, R-cache, pruning or static lists: every node's x and h are outputs
  cbg_sample_plan p{};
  p.blob = blob; p.num_classes = num_classes;
  p.num_layers = (stop_after_layers >= 0 && stop_after_layers < num_layers) ? stop_after_layers : num_layers;
  p.graph_ptr = graph_ptr; p.n_graphs = n_graphs; p.max_graph_nodes = max_graph_nodes; p.n_nodes = n_nodes;
  p.gen_node = gen_idx; p.n_gen = n_gen; p.mode = mode; p.k = k; p.r_max = r_max;
  if (int rc = run_denoiser(p, ws, st)) return rc;
  if (x_out) { if (int rc = cbg_launch_unpack_x(ws.x4, n_nodes, x_out, st)) return rc; }
  if (h_out) CBG_CUDA_OK(cudaMemcpyAsync(h_out, ws.h, (size_t)n_nodes * CBG_H * 4, cudaMemcpyDeviceToDevice, st));
  if (logits_out) {
    const int rows = cls_idx ? n_cls : (int)n_nodes;
    if (int rc = cbg_launch_classifier(blob, ws.h, cls_idx, rows, num_classes, logits_out, st)) return rc;
  }
  return 0;
}

int32_t cbg_denoiser_forward_host_f32(const float* blob_host, int64_t blob_floats, int64_t blob_version,
                                      int32_t num_layers, int32_t num_classes, const float* x_host,
                                      const float* h_host, const int32_t* graph_ptr_host, int32_t n_graphs,
                                      const uint8_t* lig_flag_host, const uint8_t* gen_flag_host, int64_t n_nodes,
                                      int32_t mode, int32_t k, float r_max, float* x_out_host, float* h_out_host,
                                      float* logits_out_host) {
  if (n_nodes <= 0 || n_graphs <= 0) { cbg_set_error("empty batch"); return 1; }
  if (num_classes < 1 || num_classes > CBG_MAXCLS) { cbg_set_error("num_classes=%d outside [1,%d]", num_classes, CBG_MAXCLS); return 1; }
  if (blob_floats != cbg_layout::kGlobalFloats + (long long)num_layers * cbg_layout::kLayerFloats) {
    cbg_set_error("blob has %lld floats, expected %lld", (long long)blob_floats,
                  cbg_layout::kGlobalFloats + (long long)num_layers * cbg_layout::kLayerFloats);
    return 1;
  }
  // host-side graph statistics and the generated-node list
  int max_graph_nodes = 0;
  for (int g = 0; g < n_graphs; ++g) {
    const int n = graph_ptr_host[g + 1] - graph_ptr_host[g];
    if (n < 0) { cbg_set_error("graph_ptr not monotone"); return 1; }
    if (n > max_graph_nodes) max_graph_nodes = n;
  }
  if (graph_ptr_host[0] != 0 || graph_ptr_host[n_graphs] != n_nodes) { cbg_set_error("graph_ptr must span [0, n_nodes]"); return 1; }
  std::vector<int> gen_idx;
  for (long long i = 0; i < n_nodes; ++i) if (gen_flag_host[i]) gen_idx.push_back((int)i);
  const int n_gen = (int)gen_idx.size();

  HostCache* cp = host_cache();
  if (!cp) { cbg_set_error("no current CUDA device"); return 2; }
  HostCache& g_cache = *cp;
  if (g_cache.blob_version != blob_version || g_cache.blob_floats != blob_floats || g_cache.blob_host != (const void*)blob_host) {
    if (g_cache.blob) CBG_CUDA_OK(cudaFree(g_cache.blob));
    g_cache.blob = nullptr;
    g_cache.blob_version = -1;
    CBG_CUDA_OK(cudaMalloc((void**)&g_cache.blob, (size_t)blob_floats * 4));
    CBG_CUDA_OK(cudaMemcpy(g_cache.blob, blob_host, (size_t)blob_floats * 4, cudaMemcpyHostToDevice));
    g_cache.blob_floats = blob_floats;
    g_cache.blob_version = blob_version;
    g_cache.blob_host = (const void*)blob_host;
  }
  const size_t ws_bytes = carve(nullptr, n_nodes, n_gen).bytes;
  size_t off = ws_bytes;
  auto region = [&](size_t nbytes) { size_t o = off; off += align256(nbytes); return o; };
  const size_t o_x = region((size_t)n_nodes * 12), o_h = region((size_t)n_nodes * CBG_H * 4);
  const size_t o_gp = region((size_t)(n_graphs + 1) * 4), o_lf = region((size_t)n_nodes), o_gf = region((size_t)n_nodes);
  const size_t o_gi = region((size_t)(n_gen > 0 ? n_gen : 1) * 4);
  const size_t o_xo = region((size_t)n_nodes * 12), o_ho = region((size_t)n_nodes * CBG_H * 4);
  const size_t o_lo = region((size_t)n_nodes * num_classes * 4);
  if (int rc = cache_reserve(g_cache, off)) return rc;
  char* d = (char*)g_cache.dev;
  cudaStream_t st = 0;
  CBG_CUDA_OK(cudaMemcpyAsync(d + o_x, x_host, (size_t)n_nodes * 12, cudaMemcpyHostToDevice, st));
  CBG_CUDA_OK(cudaMemcpyAsync(d + o_h, h_host, (size_t)n_nodes * CBG_H * 4, cudaMemcpyHostToDevice, st));
  CBG_CUDA_OK(cudaMemcpyAsync(d + o_gp, graph_ptr_host, (size_t)(n_graphs + 1) * 4, cudaMemcpyHostToDevice, st));
  CBG_CUDA_OK(cudaMemcpyAsync(d + o_lf, lig_flag_host, (size_t)n_nodes, cudaMemcpyHostToDevice, st));
  CBG_CUDA_OK(cudaMemcpyAsync(d + o_gf, gen_flag_host, (size_t)n_nodes, cudaMemcpyHostToDevice, st));
  if (n_gen) CBG_CUDA_OK(cudaMemcpyAsync(d + o_gi, gen_idx.data(), (size_t)n_gen * 4, cudaMemcpyHostToDevice, st));
  if (int rc = cbg_denoiser_forward_f32(g_cache.blob, num_layers, num_classes, (const float*)(d + o_x),
                                        (const float*)(d + o_h), (const int32_t*)(d + o_gp), n_graphs,
                                        max_graph_nodes, (const uint8_t*)(d + o_lf), (const uint8_t*)(d + o_gf),
                                        (const int32_t*)(d + o_gi), n_gen, nullptr, 0, n_nodes, mode, k, r_max, -1,
                                        (float*)(d + o_xo), (float*)(d + o_ho), (float*)(d + o_lo), d, ws_bytes, st))
    return rc;
  if (x_out_host) CBG_CUDA_OK(cudaMemcpyAsync(x_out_host, d + o_xo, (size_t)n_nodes * 12, cudaMemcpyDeviceToHost, st));
  if (h_out_host) CBG_CUDA_OK(cudaMemcpyAsync(h_out_host, d + o_ho, (size_t)n_nodes * CBG_H * 4, cudaMemcpyDeviceToHost, st));
  if (logits_out_host) CBG_CUDA_OK(cudaMemcpyAsync(logits_out_host, d + o_lo, (size_t)n_nodes * num_classes * 4, cudaMemcpyDeviceToHost, st));
  CBG_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

int32_t cbg_node_proj_f32(const float* blob_layer, int32_t sublayer, int32_t impl, const float* h,
                          const int32_t* row_idx, int32_t n_rows, int64_t n_nodes, float* planes, void* stream) {
  if (sublayer < 0 || sublayer > 1 || (impl != 0 && impl != 1 && impl != 2 && impl != 11 && impl != 12 && impl != 14)) { cbg_set_error("bad sublayer/impl"); return 1; }
  float* out[CBG_NPLANES];
  for (int p = 0; p < CBG_NPLANES; ++p) out[p] = planes + (size_t)p * n_nodes * CBG_H;
  const NodeGemmArgs g = node_gemm_args(blob_layer, (SubLayer)sublayer, Planes::kAll, h, row_idx, n_rows, out);
  if (impl == 0) return cbg_launch_node_gemm(g, (cudaStream_t)stream);
  if (impl == 2) return cbg_launch_node_gemm_f16(g, (cudaStream_t)stream);
  return cbg_launch_node_gemm_tc(g, (cudaStream_t)stream, impl == 12 ? 2 : (impl == 14 ? 4 : (impl == 11 ? 1 : 0)));
}

int32_t cbg_sample_begin_f32(const cbg_sample_plan* plan, const float* x_nodes, const uint8_t* lig_flag,
                             const uint8_t* gen_flag, void* stream) {
  if (!plan) { cbg_set_error("null plan"); return 1; }
  Workspace ws;
  if (int rc = check_ws(plan->workspace, plan->workspace_bytes, plan->n_nodes, plan->n_gen, &ws)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = cbg_launch_pack_x4(x_nodes, lig_flag, gen_flag, plan->n_nodes, ws.x4, st)) return rc;
  if (plan->rcache || plan->static_lists) {
    // static-only neighbour lists and their gates: atoms without gen_flag never move (SURVEY.md Appendix B)
    if (int rc = cbg_launch_knn(ws.x4, plan->graph_ptr, plan->n_graphs, plan->max_graph_nodes, CBG_MODE_KNN, CBG_KMAX,
                                0.f, 1, nullptr, ws.snbr, st)) return rc;
    if (int rc = cbg_launch_edge_gate(plan->blob, ws.x4, ws.snbr, plan->n_nodes, nullptr, nullptr, ws.sew, st)) return rc;
  }
  if (plan->rcache) {
    // step-invariant first-Linear terms of the static edges, for the fp32 SIMT X2H kernels
    const int64_t need = cbg_rcache_bytes(plan->n_nodes, plan->num_layers);
    if ((int64_t)plan->rcache_bytes < need) { cbg_set_error("rcache too small: have %zu bytes, need %lld", plan->rcache_bytes, (long long)need); return 1; }
    if (int rc = cbg_launch_rcache(plan->blob + cbg_layout::kGlobalFloats, plan->num_layers, ws.x4, ws.snbr,
                                   (int)plan->n_nodes, plan->rcache, st)) return rc;
  }
  return 0;
}

int32_t cbg_sample_prune_counts_host(const cbg_sample_plan* plan, int32_t* counts_host, void* stream) {
  if (!plan || !counts_host) { cbg_set_error("cbg_sample_prune_counts_host: null argument"); return 1; }
  Workspace ws;
  if (int rc = check_ws(plan->workspace, plan->workspace_bytes, plan->n_nodes, plan->n_gen, &ws)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  CBG_CUDA_OK(cudaMemcpyAsync(counts_host, ws.cnt, sizeof(int32_t) * (size_t)(plan->num_layers + 1), cudaMemcpyDeviceToHost, st));
  CBG_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

int32_t cbg_sample_step_f32(const cbg_sample_plan* plan, const cbg_step_coef* coef, const float* x_t,
                            const float* c_t, const float* pos_noise, const float* type_uniform, float* x_next,
                            float* c_next, int64_t* v_next, float* x0_pred, float* logits, void* stream) {
  Workspace ws;
  if (int rc = open_plan(plan, coef != nullptr, "null plan/coef", &ws)) return rc;
  NvtxRange nvtx_step("cbg:sample_step");
  cudaStream_t st = (cudaStream_t)stream;
  const int K = plan->num_classes;
  if (int rc = cbg_launch_step_init(x_t, c_t, plan->lig_node, plan->n_lig, K, plan->emb_wt, plan->h_lig_bias,
                                    plan->h_static, plan->n_nodes, ws.x4, ws.h, st)) return rc;
  if (int rc = run_denoiser(*plan, ws, st)) return rc;
  // classifier on ligand rows only (SURVEY.md A11); logits scratch lives in the w buffer (free after the layers)
  float* lg = logits ? logits : ws.w;
  if (int rc = cbg_launch_classifier(plan->blob, ws.h, plan->lig_node, plan->n_lig, K, lg, st)) return rc;
  ReverseArgs r{};
  r.x0 = (const float*)ws.x4; r.x0_stride = 4; r.x0_idx = plan->lig_node;
  r.logits = lg; r.x_t = x_t; r.c_t = c_t; r.gen = plan->gen_lig; r.pos_noise = pos_noise; r.type_u = type_uniform;
  r.c0 = coef->pos_c0; r.ct = coef->pos_ct;
  r.lac_prev = coef->log_alphas_cumprod_prev; r.l1mac_prev = coef->log_one_minus_alphas_cumprod_prev;
  r.la = coef->log_alpha; r.l1ma = coef->log_one_minus_alpha;
  r.n_lig = plan->n_lig; r.num_classes = K; r.x_next = x_next; r.c_next = c_next; r.v_next = (long long*)v_next;
  if (int rc = cbg_launch_reverse(r, coef->pos_logvar, coef->pos_nonzero, st)) return rc;
  if (x0_pred) {   // predicted ligand coordinates (testing / trajectory inspection)
    if (int rc = cbg_launch_gather_x(ws.x4, plan->lig_node, plan->n_lig, x0_pred, st)) return rc;
  }
  return 0;
}

// ---- the same step, replayed from a CUDA graph ---------------------------------------------------------------------
// Shapes and device pointers of a plan do not change over the T steps (the pruning / neighbour-list lengths live on the
// device), so the ~85 launches, fork/join events and memsets of a step are captured ONCE per plan and replayed with one
// cudaGraphLaunch per step.  What changes per step - the trajectory slots, the noise tensors, eight schedule
// coefficients - goes through a StepIO block in the workspace that the first and the last kernel of the graph read; it
// is refreshed by one small H2D copy (from a ring of pinned host slots) in front of every launch.
namespace {
constexpr int kIoRing = 64;
struct StepGraph {
  unsigned long long key = 0;
  int dev = -1;
  cudaStream_t stream = nullptr;
  cudaGraphExec_t exec = nullptr;
  cudaGraph_t graph = nullptr;
  long long kernel_nodes = 0;
  int warm = 0;                      // eager steps seen for this plan (the first one also performs one-time kernel setup)
  StepIO* pinned = nullptr;          // [kIoRing]
  cudaEvent_t ev[kIoRing] = {};
  bool ev_used[kIoRing] = {};
  int next = 0;
  unsigned long long stamp = 0;
};
std::vector<StepGraph*> g_graphs;
unsigned long long g_graph_clock = 0;

unsigned long long fnv1a(const void* p, size_t n, unsigned long long h = 1469598103934665603ull) {
  const unsigned char* b = (const unsigned char*)p;
  for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 1099511628211ull; }
  return h;
}
void destroy_graph(StepGraph* g) {
  if (g->exec) cudaGraphExecDestroy(g->exec);
  if (g->graph) cudaGraphDestroy(g->graph);
  for (int i = 0; i < kIoRing; ++i) if (g->ev[i]) cudaEventDestroy(g->ev[i]);
  if (g->pinned) cudaFreeHost(g->pinned);
  delete g;
}
}  // namespace

int32_t cbg_sample_step_graph_f32(const cbg_sample_plan* plan, const cbg_step_coef* coef, const float* x_t,
                                  const float* c_t, const float* pos_noise, const float* type_uniform, float* x_next,
                                  float* c_next, int64_t* v_next, void* stream) {
  Workspace ws;
  if (int rc = open_plan(plan, coef != nullptr, "null plan/coef", &ws)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int dev = -1;
  CBG_CUDA_OK(cudaGetDevice(&dev));
  if (g_cbg_prof_on)      // per-kernel event profiling brackets every launch: not capturable, run eagerly
    return cbg_sample_step_f32(plan, coef, x_t, c_t, pos_noise, type_uniform, x_next, c_next, v_next, nullptr, nullptr, stream);
  unsigned long long key = fnv1a(plan, sizeof(*plan));
  key = fnv1a(&st, sizeof(st), key);
  StepGraph* g = nullptr;
  for (StepGraph* c : g_graphs) if (c->key == key && c->dev == dev && c->stream == st) { g = c; break; }
  if (!g) {
    if (g_graphs.size() >= 8) {      // evict the least recently used entry
      size_t lru = 0;
      for (size_t i = 1; i < g_graphs.size(); ++i) if (g_graphs[i]->stamp < g_graphs[lru]->stamp) lru = i;
      destroy_graph(g_graphs[lru]);
      g_graphs.erase(g_graphs.begin() + (long)lru);
    }
    g = new StepGraph();
    g->key = key; g->dev = dev; g->stream = st;
    g_graphs.push_back(g);
  }
  g->stamp = ++g_graph_clock;
  if (g->warm < 1) {                 // first step of a plan: eager (sets kernel attributes, validates the arguments)
    g->warm += 1;
    return cbg_sample_step_f32(plan, coef, x_t, c_t, pos_noise, type_uniform, x_next, c_next, v_next, nullptr, nullptr, stream);
  }
  const int K = plan->num_classes;
  if (!g->exec) {
    CBG_CUDA_OK(cudaMallocHost((void**)&g->pinned, sizeof(StepIO) * kIoRing));
    for (int i = 0; i < kIoRing; ++i) CBG_CUDA_OK(cudaEventCreateWithFlags(&g->ev[i], cudaEventDisableTiming));
    const long long launches0 = g_cbg_launches;
    // capture on a private stream (the caller's may be the legacy default stream, which cannot be captured); the
    // instantiated graph is launched into the caller's stream
    cudaStream_t cs = nullptr;
    CBG_CUDA_OK(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
    CBG_CUDA_OK(cudaStreamBeginCapture(cs, cudaStreamCaptureModeRelaxed));
    int rc = cbg_launch_step_init_io(ws.io, plan->lig_node, plan->n_lig, K, plan->emb_wt, plan->h_lig_bias, plan->h_static,
                                     plan->n_nodes, ws.x4, ws.h, cs);
    if (!rc) rc = run_denoiser(*plan, ws, cs);
    if (!rc) rc = cbg_launch_classifier(plan->blob, ws.h, plan->lig_node, plan->n_lig, K, ws.w, cs);
    if (!rc) {
      ReverseArgs r{};
      r.x0 = (const float*)ws.x4; r.x0_stride = 4; r.x0_idx = plan->lig_node;
      r.logits = ws.w; r.gen = plan->gen_lig; r.n_lig = plan->n_lig; r.num_classes = K;
      rc = cbg_launch_reverse_io(r, ws.io, cs);
    }
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(cs, &graph);
    cudaStreamDestroy(cs);
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (ce != cudaSuccess) { cbg_set_error("cudaStreamEndCapture -> %s", cudaGetErrorString(ce)); return 2; }
    g->graph = graph;
    g->kernel_nodes = g_cbg_launches - launches0;      // the launchers counted their (captured) launches
    g_cbg_launches = launches0;
    CBG_CUDA_OK(cudaGraphInstantiate(&g->exec, graph, 0));
  }
  const int slot = g->next++ % kIoRing;
  if (g->ev_used[slot]) CBG_CUDA_OK(cudaEventSynchronize(g->ev[slot]));      // the copy that read this slot 64 steps ago
  StepIO& io = g->pinned[slot];
  io.x_t = x_t; io.c_t = c_t; io.pos_noise = pos_noise; io.type_u = type_uniform;
  io.x_next = x_next; io.c_next = c_next; io.v_next = (long long*)v_next;
  io.c0 = coef->pos_c0; io.ct = coef->pos_ct;
  io.lac_prev = coef->log_alphas_cumprod_prev; io.l1mac_prev = coef->log_one_minus_alphas_cumprod_prev;
  io.la = coef->log_alpha; io.l1ma = coef->log_one_minus_alpha;
  io.logvar = coef->pos_logvar; io.nonzero = coef->pos_nonzero;
  CBG_CUDA_OK(cudaMemcpyAsync(ws.io, &io, sizeof(StepIO), cudaMemcpyHostToDevice, st));
  CBG_CUDA_OK(cudaEventRecord(g->ev[slot], st));
  g->ev_used[slot] = true;
  CBG_CUDA_OK(cudaGraphLaunch(g->exec, st));
  g_cbg_launches += g->kernel_nodes;
  return 0;
}

int64_t cbg_sample_step_graph_nodes(const cbg_sample_plan* plan, void* stream) {
  if (!plan) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long key = fnv1a(plan, sizeof(*plan));
  key = fnv1a(&st, sizeof(st), key);
  for (StepGraph* c : g_graphs) if (c->key == key && c->exec) return c->kernel_nodes;
  return 0;
}

namespace {
// the launch arguments of the DiffSBDD / DiffBP reverse kernels, shared by the steps and the test hooks
SbddArgs sbdd_args(float4* x4, const int* graph_ptr, int n_graphs, const int* lig_node, int n_lig, int K,
                   const cbg_sbdd_coef& coef, const float* logits, const float* x_t, const float* c_t,
                   const float* x_noise, const float* c_noise, float* x_next, float* c_next) {
  SbddArgs r{};
  r.x4 = x4; r.graph_ptr = graph_ptr; r.lig_node = lig_node; r.n_lig = n_lig;
  r.num_classes = K; r.n_graphs = n_graphs; r.logits = logits; r.x_t = x_t; r.c_t = c_t;
  r.x_noise = x_noise; r.c_noise = c_noise; r.a = coef.a; r.b = coef.b; r.s = coef.s; r.mode = coef.mode;
  r.x_next = x_next; r.c_next = c_next;
  return r;
}
BpArgs bp_args(const float4* x4, const int* graph_ptr, int n_graphs, const int* lig_node, int n_lig, int K,
               const cbg_bp_coef& coef, const float* x_pred, const float* logits, const float* x_t, const float* c_t,
               const unsigned char* gen, const float* pos_noise, const float* type_u, float* x_next, float* c_next,
               int64_t* v_next, float* eps_out) {
  BpArgs r{};
  r.x4 = x4; r.graph_ptr = graph_ptr; r.lig_node = lig_node; r.n_lig = n_lig; r.num_classes = K;
  r.n_graphs = n_graphs; r.x_pred = x_pred; r.logits = logits; r.x_t = x_t; r.c_t = c_t; r.gen = gen;
  r.pos_noise = pos_noise; r.type_u = type_u; r.abar = coef.alpha_cumprod; r.beta = coef.beta;
  r.nonzero = coef.nonzero; r.prob = coef.change_prob; r.x_next = x_next; r.c_next = c_next;
  r.v_next = (long long*)v_next; r.eps_out = eps_out;
  return r;
}
// argument checks of the per-graph reverse hooks (before any device work)
int check_graph_hook(const char* fn, bool ptrs_ok, int n_graphs, int n_lig, int num_classes) {
  if (!ptrs_ok) { cbg_set_error("%s: null argument", fn); return 1; }
  if (n_graphs < 0 || n_lig < 0) { cbg_set_error("%s: n_graphs=%d n_lig=%d", fn, n_graphs, n_lig); return 1; }
  if (num_classes < 1 || num_classes > CBG_MAXCLS) {
    cbg_set_error("%s: num_classes=%d outside [1,%d]", fn, num_classes, CBG_MAXCLS);
    return 1;
  }
  return 0;
}
}  // namespace

int32_t cbg_sbdd_step_f32(const cbg_sample_plan* plan, const cbg_sbdd_coef* coef, const float* x_t, const float* c_t,
                          const float* x_noise, const float* c_noise, float* x_next, float* c_next,
                          float* x_pred, float* logits, void* stream) {
  Workspace ws;
  if (int rc = open_plan(plan, coef != nullptr, "null plan/coef", &ws)) return rc;
  if (plan->rcache || plan->static_lists) { cbg_set_error("DiffSBDD moves the pocket every step: the plan must not carry static lists / an R-cache"); return 1; }
  if (coef->mode != 0 && coef->mode != 1) { cbg_set_error("cbg_sbdd_coef.mode must be 0 or 1"); return 1; }
  cudaStream_t st = (cudaStream_t)stream;
  const int K = plan->num_classes;
  if (int rc = cbg_launch_step_init(x_t, c_t, plan->lig_node, plan->n_lig, K, plan->emb_wt, plan->h_lig_bias,
                                    plan->h_static, plan->n_nodes, ws.x4, ws.h, st)) return rc;
  if (int rc = run_denoiser(*plan, ws, st)) return rc;
  float* lg = logits ? logits : ws.w;
  if (int rc = cbg_launch_classifier(plan->blob, ws.h, plan->lig_node, plan->n_lig, K, lg, st)) return rc;
  if (x_pred) {
    if (int rc = cbg_launch_gather_x(ws.x4, plan->lig_node, plan->n_lig, x_pred, st)) return rc;
  }
  return cbg_launch_sbdd_reverse(sbdd_args(ws.x4, plan->graph_ptr, plan->n_graphs, plan->lig_node, plan->n_lig, K, *coef,
                                           lg, x_t, c_t, x_noise, c_noise, x_next, c_next), st);
}

int32_t cbg_sbdd_reverse_f32(float* x4, const int32_t* graph_ptr, int32_t n_graphs, const int32_t* lig_node, int32_t n_lig,
                             int32_t num_classes, const cbg_sbdd_coef* coef, const float* logits, const float* x_t,
                             const float* c_t, const float* x_noise, const float* c_noise, float* x_next, float* c_next,
                             void* stream) {
  if (int rc = check_graph_hook("cbg_sbdd_reverse_f32", x4 && graph_ptr && lig_node && coef && logits && x_t && c_t &&
                                x_noise && c_noise && x_next && c_next, n_graphs, n_lig, num_classes)) return rc;
  if (coef->mode != 0 && coef->mode != 1) { cbg_set_error("cbg_sbdd_reverse_f32: mode=%d is not 0 or 1", coef->mode); return 1; }
  return cbg_launch_sbdd_reverse(sbdd_args((float4*)x4, graph_ptr, n_graphs, lig_node, n_lig, num_classes, *coef, logits,
                                           x_t, c_t, x_noise, c_noise, x_next, c_next), (cudaStream_t)stream);
}

int32_t cbg_bp_step_f32(const cbg_sample_plan* plan, const float* com_blob, int32_t com_layers, const cbg_bp_coef* coef,
                        const float* x_t, const float* c_t, const float* pos_noise, const float* type_uniform,
                        float* x_next, float* c_next, int64_t* v_next, float* eps_out, float* logits, void* stream) {
  Workspace ws;
  if (int rc = open_plan(plan, coef && com_blob, "null plan/coef/com_blob", &ws)) return rc;
  if (com_layers < 0 || com_layers > 16) { cbg_set_error("com_layers=%d outside [0,16]", com_layers); return 1; }
  cudaStream_t st = (cudaStream_t)stream;
  const int K = plan->num_classes, n_lig = plan->n_lig;
  if (int rc = cbg_launch_step_init(x_t, c_t, plan->lig_node, n_lig, K, plan->emb_wt, plan->h_lig_bias,
                                    plan->h_static, plan->n_nodes, ws.x4, ws.h, st)) return rc;
  const BpScratch s = bp_scratch(ws, n_lig, K);
  float* lg = logits ? logits : s.logits;
  if (int rc = run_bp_denoiser(*plan, com_blob, com_layers, ws, x_t, lg, s.x_pred, st)) return rc;
  return cbg_launch_bp_reverse(bp_args(ws.x4, plan->graph_ptr, plan->n_graphs, plan->lig_node, n_lig, K, *coef, s.x_pred,
                                       lg, x_t, c_t, plan->gen_lig, pos_noise, type_uniform, x_next, c_next, v_next,
                                       eps_out), st);
}

int32_t cbg_bp_reverse_f32(const float* x4, const int32_t* graph_ptr, int32_t n_graphs, const int32_t* lig_node,
                           int32_t n_lig, int32_t num_classes, const cbg_bp_coef* coef, const float* x_pred,
                           const float* logits, const float* x_t, const float* c_t, const uint8_t* gen,
                           const float* pos_noise, const float* type_uniform, float* x_next, float* c_next,
                           int64_t* v_next, float* eps_out, void* stream) {
  if (int rc = check_graph_hook("cbg_bp_reverse_f32", x4 && graph_ptr && lig_node && coef && x_pred && logits && x_t &&
                                c_t && gen && pos_noise && type_uniform && x_next && c_next && v_next,
                                n_graphs, n_lig, num_classes)) return rc;
  return cbg_launch_bp_reverse(bp_args((const float4*)x4, graph_ptr, n_graphs, lig_node, n_lig, num_classes, *coef, x_pred,
                                       logits, x_t, c_t, gen, pos_noise, type_uniform, x_next, c_next, v_next, eps_out),
                               (cudaStream_t)stream);
}

int32_t cbg_bp_eval_loss_f32(const cbg_sample_plan* plan, const float* com_blob, int32_t com_layers,
                             const cbg_bp_eval_coef* coefs, int32_t n_rep, const float* x0, const int64_t* v0,
                             const float* pos_noise, const float* type_uniform, float* xt, int64_t* vt, uint8_t* mask,
                             float* vec, float* c_pred, float* rep_loss, void* stream) {
  NvtxRange nvtx_eval("cbg:bp_eval_loss");
  cudaStream_t st = (cudaStream_t)stream;
  Workspace ws;
  BpEvalArgs e{};
  if (int rc = open_eval(plan, com_blob && coefs && x0 && v0 && pos_noise && type_uniform && xt && vt && mask && vec &&
                         c_pred && rep_loss, "cbg_bp_eval_loss_f32: null argument", n_rep, 1, x0, v0, &ws, &e.b, st)) return rc;
  if (com_layers < 0 || com_layers > 16) { cbg_set_error("com_layers=%d outside [0,16]", com_layers); return 1; }
  for (int r = 0; r < n_rep; ++r) e.coef.c[r] = coefs[r];
  e.n_rep = n_rep; e.pos_noise = pos_noise; e.type_u = type_uniform;
  e.xt = xt; e.vt = (long long*)vt; e.mask = mask; e.vec = vec; e.c_pred = c_pred; e.rep_loss = rep_loss;
  // scratch: the X2H planes are free once the denoiser is done (the CoM head uses the H2X planes)
  const BpScratch s = bp_scratch(ws, plan->n_lig, plan->num_classes);
  e.logits = s.logits; e.x_pred = s.x_pred;
  e.xs = (float4*)ws.plane[0]; e.thr = (int2*)ws.plane[1]; e.graph_part = ws.plane[2];
  if (int rc = cbg_launch_bp_eval_noise(e, st)) return rc;
  if (int rc = run_bp_denoiser(*plan, com_blob, com_layers, ws, xt, s.logits, s.x_pred, st)) return rc;
  return cbg_launch_bp_eval_loss(e, st);
}

int32_t cbg_reverse_step_f32(const cbg_step_coef* coef, const float* x0_pred, const float* logits, const float* x_t,
                             const float* c_t, const uint8_t* gen, const float* pos_noise, const float* type_uniform,
                             int32_t n, int32_t num_classes, float* x_next, float* c_next, int64_t* v_next,
                             void* stream) {
  if (!(coef && x0_pred && logits && x_t && c_t && gen && pos_noise && type_uniform && x_next && c_next && v_next)) {
    cbg_set_error("cbg_reverse_step_f32: null argument");
    return 1;
  }
  if (n < 0) { cbg_set_error("cbg_reverse_step_f32: n=%d", n); return 1; }
  if (num_classes < 1 || num_classes > CBG_MAXCLS) { cbg_set_error("num_classes=%d outside [1,%d]", num_classes, CBG_MAXCLS); return 1; }
  ReverseArgs r{};
  r.x0 = x0_pred; r.x0_stride = 3; r.x0_idx = nullptr;
  r.logits = logits; r.x_t = x_t; r.c_t = c_t; r.gen = gen; r.pos_noise = pos_noise; r.type_u = type_uniform;
  r.c0 = coef->pos_c0; r.ct = coef->pos_ct;
  r.lac_prev = coef->log_alphas_cumprod_prev; r.l1mac_prev = coef->log_one_minus_alphas_cumprod_prev;
  r.la = coef->log_alpha; r.l1ma = coef->log_one_minus_alpha;
  r.n_lig = n; r.num_classes = num_classes; r.x_next = x_next; r.c_next = c_next; r.v_next = (long long*)v_next;
  return cbg_launch_reverse(r, coef->pos_logvar, coef->pos_nonzero, (cudaStream_t)stream);
}

int32_t cbg_eval_loss_f32(const cbg_sample_plan* plan, const cbg_eval_coef* coefs, int32_t n_rep, const float* x0,
                          const int64_t* v0, const float* pos_noise, const float* type_uniform, float* xt, int64_t* vt,
                          float* x_pred, float* c_pred, float* graph_loss, float* rep_loss, void* stream) {
  NvtxRange nvtx_eval("cbg:eval_loss");
  cudaStream_t st = (cudaStream_t)stream;
  Workspace ws;
  EvalArgs e{};
  if (int rc = open_eval(plan, coefs && x0 && v0 && pos_noise && type_uniform && xt && vt && x_pred && c_pred && graph_loss &&
                         rep_loss, "cbg_eval_loss_f32: null argument", n_rep, 1, x0, v0, &ws, &e.b, st)) return rc;
  for (int r = 0; r < n_rep; ++r) e.coef.c[r] = coefs[r];
  e.n_rep = n_rep; e.pos_noise = pos_noise; e.type_u = type_uniform;
  e.xt = xt; e.vt = (long long*)vt; e.x_pred = x_pred; e.c_pred = c_pred;
  e.logits = ws.w;                  // classifier scratch: the attention-weight buffer is free after the layers
  e.graph_cnt = (int*)ws.ew;        // so is the edge-gate buffer (n_nodes * 32 >= n_graphs entries)
  e.graph_loss = graph_loss; e.rep_loss = rep_loss;
  if (int rc = cbg_launch_eval_noise(e, st)) return rc;
  if (int rc = run_denoiser(*plan, ws, st)) return rc;
  if (int rc = cbg_launch_classifier(plan->blob, ws.h, plan->lig_node, plan->n_lig, plan->num_classes, ws.w, st)) return rc;
  return cbg_launch_eval_loss(e, st);
}

int32_t cbg_sbdd_eval_loss_f32(const cbg_sample_plan* plan, const cbg_sbdd_eval_coef* coefs, int32_t n_t,
                               const float* x0, const int64_t* v0, const float* x_rec, const float* x_t_noise,
                               const float* c_t_noise, const float* x_0_noise, const float* c_0_noise, float* vec_pos,
                               float* vec_atom, float* terms, float* t_loss, void* stream) {
  NvtxRange nvtx_eval("cbg:sbdd_eval_loss");
  cudaStream_t st = (cudaStream_t)stream;
  Workspace ws;
  SbddEvalArgs e{};
  if (int rc = open_eval(plan, coefs && x0 && v0 && x_t_noise && c_t_noise && x_0_noise && c_0_noise && vec_pos && vec_atom &&
                         terms && t_loss && (x_rec || plan->n_nodes == plan->n_lig), "cbg_sbdd_eval_loss_f32: null argument",
                         n_t, 2, x0, v0, &ws, &e.b, st)) return rc;
  if (plan->rcache || plan->static_lists) { cbg_set_error("DiffSBDD moves the pocket with every noised copy: the plan must not carry static lists / an R-cache"); return 1; }
  if ((plan->n_nodes - plan->n_lig) % (2 * n_t)) { cbg_set_error("plan (n_nodes=%lld) is not %d replicas of one batch", (long long)plan->n_nodes, 2 * n_t); return 1; }
  for (int j = 0; j < n_t; ++j) e.coef.c[j] = coefs[j];
  e.n_t = n_t; e.n_nodes = plan->n_nodes; e.x_rec = x_rec;
  e.x_t_noise = x_t_noise; e.c_t_noise = c_t_noise; e.x_0_noise = x_0_noise; e.c_0_noise = c_0_noise;
  e.logits = ws.w;                  // classifier scratch: the attention-weight buffer is free after the layers
  e.vec_pos = vec_pos; e.vec_atom = vec_atom; e.terms = terms; e.t_loss = t_loss;
  if (int rc = cbg_launch_sbdd_eval_noise(e, st)) return rc;
  if (int rc = run_denoiser(*plan, ws, st)) return rc;
  if (int rc = cbg_launch_classifier(plan->blob, ws.h, plan->lig_node, plan->n_lig, plan->num_classes, ws.w, st)) return rc;
  return cbg_launch_sbdd_eval_loss(e, st);
}

// ---- row f3: device-side batch construction ---------------------------------------------------------------------
int32_t cbg_pocket_stats_f32(const float* prot_pos, const int32_t* prot_ptr, int32_t n_pockets, const float* ctx_pos,
                             const int32_t* ctx_ptr, int32_t centre_mode, float* space_size, float* centre, void* stream) {
  if (n_pockets < 0 || (n_pockets > 0 && (!prot_pos || !prot_ptr || !space_size || !centre))) { cbg_set_error("cbg_pocket_stats_f32: null argument"); return 1; }
  if (centre_mode != 0 && centre_mode != 1) { cbg_set_error("centre_mode must be 0 (pocket mean) or 1 (context mean)"); return 1; }
  if (centre_mode == 1 && (!ctx_ptr || !ctx_pos)) { cbg_set_error("centre_mode 1 needs ctx_pos and ctx_ptr"); return 1; }
  return cbg_launch_pocket_stats(prot_pos, prot_ptr, n_pockets, ctx_pos, ctx_ptr, centre_mode, space_size, centre, (cudaStream_t)stream);
}

int32_t cbg_sample_ligand_sizes(const cbg_size_prior* prior, const float* space_size, int32_t n_pockets, int32_t repeat,
                                const double* u, const int32_t* ctx_ptr, const int32_t* extra, int32_t* n_lig,
                                int32_t* lig_ptr, void* stream) {
  if (!prior || !prior->bounds || !prior->bin_ptr || !prior->values || !prior->cdf || prior->n_bounds < 0) { cbg_set_error("cbg_sample_ligand_sizes: bad size prior"); return 1; }
  if (n_pockets < 0 || repeat < 0 || !space_size || !u || !n_lig || !lig_ptr) { cbg_set_error("cbg_sample_ligand_sizes: null argument"); return 1; }
  if (ctx_ptr && !extra) { cbg_set_error("context tasks need the extra[] draws"); return 1; }
  return cbg_launch_ligand_sizes(prior->bounds, prior->n_bounds, prior->bin_ptr, prior->values, prior->cdf, space_size,
                                 n_pockets, repeat, u, ctx_ptr, extra, n_lig, lig_ptr, (cudaStream_t)stream);
}

int32_t cbg_build_batch_f32(const cbg_batch_spec* b, void* stream) {
  if (!b) { cbg_set_error("cbg_build_batch_f32: null spec"); return 1; }
  if (!b->prot_pos || !b->prot_element || !b->prot_backbone || !b->prot_aa || !b->prot_ptr || !b->centre || !b->lig_ptr ||
      !b->pos_noise || !b->protein_pos || !b->protein_atom_feature || !b->protein_aa_type || !b->protein_element_batch ||
      !b->protein_translation || !b->ligand_pos || !b->ligand_atom_type || !b->ligand_element_batch) {
    cbg_set_error("cbg_build_batch_f32: null argument"); return 1;
  }
  if (b->type_dist != CBG_TYPE_UNIFORM && b->type_dist != CBG_TYPE_ABSORBING) { cbg_set_error("unknown type_dist"); return 1; }
  if (b->type_dist == CBG_TYPE_UNIFORM && (!b->type_u || b->num_classes <= 0)) { cbg_set_error("uniform types need type_u and num_classes"); return 1; }
  if (b->pos_dist != CBG_POS_GAUSSIAN && b->pos_dist != CBG_POS_ZERO_MEAN_GAUSSIAN) { cbg_set_error("unknown pos_dist"); return 1; }
  if (b->ctx_ptr && (!b->ctx_pos || !b->ctx_type)) { cbg_set_error("ctx_ptr needs ctx_pos and ctx_type"); return 1; }
  if (b->ctx_ptr && b->pos_dist == CBG_POS_ZERO_MEAN_GAUSSIAN) { cbg_set_error("zero_mean_gaussian is a de-novo option"); return 1; }
  return cbg_launch_build_batch(b->prot_pos, b->prot_element, b->prot_backbone, b->prot_aa, b->prot_ptr, b->n_pockets, b->repeat,
                                b->centre, b->ctx_pos, b->ctx_type, b->ctx_ptr, b->lig_ptr, b->pos_noise, b->type_u,
                                b->num_classes, b->type_dist, b->pos_dist, b->protein_pos, b->protein_atom_feature,
                                (long long*)b->protein_aa_type, (long long*)b->protein_element_batch, b->protein_translation,
                                b->ligand_pos, (long long*)b->ligand_atom_type, (long long*)b->ligand_element_batch,
                                b->ligand_ctx_flag, b->ligand_gen_flag, (cudaStream_t)stream);
}

}  // extern "C"
