// Fused equivariant message-passing kernels (the dominant kernels of the hot path).
//
// Reference semantics (as written, per edge e = (j -> i), 32 in-edges per node i):
//   kv   = [onehot(type) | onehot(type) (x) g(|x_i - x_j|) | h_i | h_j]          (340 wide)
//   X2H: k = MLP_k(kv), v = MLP_v(kv) * e_w, q = MLP_q(h)/sqrt(8) (node GEMM)
//        alpha = softmax_j(<q_i, k_ij>) per head ; h_i += sum_j alpha_ij v_ij
//        (repo/modules/attention/x2h_attention.py:43-97)
//   H2X: k = MLP_xk(kv), v = MLP_xv(kv) * e_w  [16 heads]
//        dx_i = mean_heads sum_j alpha_ij v_ij (x_i - x_j)
//        (repo/modules/attention/h2x_attention.py:34-73; x += dx * gen_flag, unitransformer.py:182)
//
// What the kernels do instead (exact algebra, nothing of size [E,*] except alpha*e_w):
//   * first Linear via the node planes: pre = Pi[i] + Pj[j] + c[type] + Wrf[type] g(d)
//   * logits through the query-folded matrix U_i[f][hd] = sum_{f' in hd} q_i[f'] W1k[f'][f]:
//       <q_i, W1k a + b1k>_hd = a . U_i[:,hd] + const(i,hd)     (const cancels in the softmax)
//   * values through linearity of the second Linear:
//       sum_j w_ij (W1v a_ij + b1v) = W1v (sum_j w_ij a_ij) + b1v sum_j w_ij   per head
//   32 in-edges of a node = one warp; in-warp softmax/aggregation, no atomics, fixed
//   summation order (deterministic).
//
// Thread mapping: a warp owns one destination node at a time.  Geometry is computed with
// lane = edge; the MLP math with lane = 4 consecutive features (f = 4*lane .. 4*lane+3) for
// groups of 4 edges; per-(edge, head) contractions are finished with a halving butterfly
// that leaves lane l with head l/2 and edges 4g + 2*(l%2), 4g + 2*(l%2) + 1.  The butterfly is
// select-free for its four head steps because every lane keeps its per-head operand (U, W1xv) in a
// lane-permuted order (physical slot hp <-> head hp ^ (lane >> 1)).
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include "cbg_kernels.cuh"

namespace {

// warps per CTA are a template parameter (8 / 12 / 16): more warps = better latency hiding at the
// price of a tighter register budget (255 / 168 / 128 per thread); picked at run time, see below.
constexpr long long kOffX2hK = cbg_layout::layer_offset(CBG_LF_X2H_K_WRF);
constexpr long long kOffX2hV = cbg_layout::layer_offset(CBG_LF_X2H_V_WRF);
constexpr long long kOffH2x = cbg_layout::layer_offset(CBG_LF_H2X_K_WRF);
constexpr long long kOffX2hKRbf = cbg_layout::layer_offset(CBG_LF_X2H_K_RBF);
constexpr long long kOffX2hVRbf = cbg_layout::layer_offset(CBG_LF_X2H_V_RBF);

struct __align__(16) EdgeMeta {   // per-warp scratch, 3456 B; indexed by the PERMUTED edge position
  float g[CBG_NRBF][32];          // g[m][e]
  float rel[3][32];               // x_i - x_j
  float ew[32];                   // e_w (0 for padded slots)
  int j[32];                      // source node (i itself for padded slots)
  int t[32];                      // edge type 0..3
  int slot[32];                   // index into the node's static-neighbour list (-1: not a static edge)
};

struct MlpSmem {                  // first-layer weights of one edge MLP in shared memory
  const float* wrf;               // [4][20][128]
  const float* c;                 // [4][128]
};

// lane = edge: geometry, RBF, type.  The 32 slots of the node are re-ordered as
//   [static edges (both endpoints have gen_flag == 0) | other valid edges | padding],
// each class keeping its nearest-first order; every edge kernel applies the same permutation, so
// positions agree between x2h_k (writes w) and x2h_v (reads w).  Static edges never change over the
// diffusion steps (their endpoints never move), which is what the R-cache below exploits; the p-th
// static edge of the list is the p-th entry of the node's static-only kNN list (prefix property).
// Returns the validity mask in permuted positions.
// fstat (optional): per-node flag "all 32 slots hold static edges" (written by the edge gate once per step when the
// R-cache is on).  For such a node the permutation is the identity and every edge is served from the R-cache, so only
// j, e_w and the slot index are ever read: the coordinate gathers, the RBF and the type computation are skipped.
__device__ __forceinline__ unsigned edge_setup(EdgeMeta& M, int i, int lane, const float4* __restrict__ x4,
                                               const int* __restrict__ nbr, const float* __restrict__ ew,
                                               const float* s_rbf, const unsigned char* __restrict__ fstat = nullptr) {
  if (fstat != nullptr && fstat[i]) {                     // warp-uniform
    M.j[lane] = nbr[(size_t)i * CBG_KMAX + lane];
    M.ew[lane] = ew[(size_t)i * CBG_KMAX + lane];
    M.slot[lane] = lane;
    __syncwarp();
    return 0xffffffffu;
  }
  const float4 xi = x4[i];
  const int jn = nbr[(size_t)i * CBG_KMAX + lane];
  const bool valid = jn >= 0;
  const int j = valid ? jn : i;
  const float4 xj = x4[j];
  const float rx = xi.x - xj.x, ry = xi.y - xj.y, rz = xi.z - xj.z;
  const float d = sqrtf(rx * rx + ry * ry + rz * rz);
  const int fi = node_flags(xi), fj = node_flags(xj);
  const bool is_static = valid && ((fi | fj) & 2) == 0;
  const unsigned vm = __ballot_sync(CBG_FULL, valid);
  const unsigned sm = __ballot_sync(CBG_FULL, is_static);
  const unsigned lt = (1u << lane) - 1u;
  const int n_static = __popc(sm), n_valid = __popc(vm);
  const int rank_s = __popc(sm & lt);
  const int pos = is_static ? rank_s
                            : (valid ? n_static + __popc(vm & ~sm & lt) : n_valid + __popc(~vm & lt));
  const float coeff = s_rbf[20];
#pragma unroll
  for (int m = 0; m < CBG_NRBF; ++m) {
    const float u = d - s_rbf[m];
    M.g[m][pos] = expf(coeff * u * u);
  }
  M.rel[0][pos] = rx; M.rel[1][pos] = ry; M.rel[2][pos] = rz;
  M.ew[pos] = valid ? ew[(size_t)i * CBG_KMAX + lane] : 0.f;
  M.j[pos] = j;
  // unitransformer.py:88-99: 0 lig->lig, 1 lig src/prot dst, 2 prot src/lig dst, 3 prot->prot
  M.t[pos] = ((fj & 1) ? 0 : 2) + ((fi & 1) ? 0 : 1);
  M.slot[pos] = is_static ? rank_s : -1;
  __syncwarp();
  return (n_valid >= 32) ? 0xffffffffu : ((1u << n_valid) - 1u);
}

// pull the next node's R block (16 KB, contiguous) towards L2 while this node computes
__device__ __forceinline__ void prefetch_rc(const float* rc_base, int i_next, int lane) {
  if (rc_base == nullptr) return;
  const char* b = reinterpret_cast<const char*>(rc_base + (size_t)i_next * (CBG_KMAX * CBG_H));
#pragma unroll
  for (int r = 0; r < 4; ++r) asm volatile("prefetch.global.L2 [%0];" ::"l"(b + (size_t)(lane + 32 * r) * 128));
}

// number of entries of the node list of this launch (host bound, optionally clipped by a device count)
__device__ __forceinline__ int list_length(const EdgeArgs& p) {
  int n = p.n_nodes;
  if (p.n_nodes_dev) { const int nd = *p.n_nodes_dev; n = nd < n ? nd : n; }
  return n;
}

// Node scheduling of the X2H kernels.  With a ticket counter (EdgeArgs::ticket, zeroed before the launch) every warp
// draws its next node from a global counter: nodes differ in cost (generated atoms and their neighbourhood run the RBF
// path, static nodes only stream the R-cache), so a static round-robin leaves SMs idle at the end of a launch.  The
// draw for the following node is issued before the current one is processed, which hides the atomic's latency.
struct NodeSched {
  int* ticket;
  int stride, pending, nn;
  __device__ __forceinline__ int first(const EdgeArgs& p, int warp_global, int total_warps, int lane) {
    ticket = p.ticket; stride = total_warps; pending = 0; nn = 0;
    if (ticket == nullptr) return warp_global;
    int v = 0;
    if (lane == 0) v = atomicAdd(ticket, 1);
    return __shfl_sync(CBG_FULL, v, 0);
  }
  __device__ __forceinline__ void draw(int n, int lane) {            // request the node that follows n
    if (ticket != nullptr) { if (lane == 0) pending = atomicAdd(ticket, 1); }
    else pending = n + stride;
  }
  __device__ __forceinline__ int next(int lane) {                    // first use waits for the atomic
    nn = ticket != nullptr ? __shfl_sync(CBG_FULL, pending, 0) : pending;
    return nn;
  }
};

// All-lane sums of 4 per-lane values, result in every lane: transposed butterfly (each step halves
// the number of live values), three plain steps, four broadcasts: 10 SHFL instead of 20.
__device__ __forceinline__ void allreduce4(float (&s)[4], int lane) {
  const bool u1 = (lane & 16) != 0;
  float k0 = u1 ? s[2] : s[0], k1 = u1 ? s[3] : s[1];
  const float d0 = u1 ? s[0] : s[2], d1 = u1 ? s[1] : s[3];
  k0 += __shfl_xor_sync(CBG_FULL, d0, 16);
  k1 += __shfl_xor_sync(CBG_FULL, d1, 16);
  const bool u2 = (lane & 8) != 0;
  float k = u2 ? k1 : k0;
  const float d = u2 ? k0 : k1;
  k += __shfl_xor_sync(CBG_FULL, d, 8);
  k += __shfl_xor_sync(CBG_FULL, k, 4);
  k += __shfl_xor_sync(CBG_FULL, k, 2);
  k += __shfl_xor_sync(CBG_FULL, k, 1);
  s[0] = __shfl_sync(CBG_FULL, k, 0);     // lanes 0-7 hold value 0, 8-15 value 1, 16-23 value 2, 24-31 value 3
  s[1] = __shfl_sync(CBG_FULL, k, 8);
  s[2] = __shfl_sync(CBG_FULL, k, 16);
  s[3] = __shfl_sync(CBG_FULL, k, 24);
}

// First Linear + LayerNorm + ReLU of one edge MLP for the 4 edges e0..e0+3.
// a[ee] = relu(LN(Pi + Pj[j] + c[t] + Wrf[t] g)) restricted to this lane's 4 features.
// rc: this node's block of the R-cache ([32 static slots][128], R = c[t] + Wrf[t] g(d) of the static
// edge) or nullptr.  Groups whose 4 edges are all static skip the RBF mat-vec and stream R instead.
__device__ __forceinline__ void first_layer4(const EdgeMeta& M, int e0, int lane, const float4 pi,
                                             const float* __restrict__ pj_plane, const MlpSmem W,
                                             const float4 gamma, const float4 beta, float4 (&a)[4],
                                             const float* __restrict__ rc) {
  int t[4];
  const bool cached = (rc != nullptr) && (M.slot[e0 + 3] >= 0);   // static edges come first: slot[e0+3]>=0 => all 4
  if (cached) {
#pragma unroll
    for (int ee = 0; ee < 4; ++ee) {
      const int j = M.j[e0 + ee];
      const float4 pj = ldg4(pj_plane + (size_t)j * CBG_H + 4 * lane);
      const float4 r = ldg4(rc + M.slot[e0 + ee] * CBG_H + 4 * lane);
      a[ee] = add4(add4(pi, pj), r);
    }
  } else {
#pragma unroll
  for (int ee = 0; ee < 4; ++ee) {
    const int j = M.j[e0 + ee];
    t[ee] = M.t[e0 + ee];
    const float4 pj = ldg4(pj_plane + (size_t)j * CBG_H + 4 * lane);
    const float4 c = ld4(W.c + t[ee] * CBG_H + 4 * lane);
    a[ee] = add4(add4(pi, pj), c);
  }
  const bool uniform = (t[0] == t[1]) && (t[0] == t[2]) && (t[0] == t[3]);   // warp-uniform
  if (uniform) {
    const float* w = W.wrf + t[0] * (CBG_NRBF * CBG_H) + 4 * lane;
#pragma unroll
    for (int m = 0; m < CBG_NRBF; ++m) {
      const float4 wv = ld4(w + m * CBG_H);
      const float4 gv = ld4(&M.g[m][e0]);
      fma4(a[0], wv, gv.x); fma4(a[1], wv, gv.y); fma4(a[2], wv, gv.z); fma4(a[3], wv, gv.w);
    }
  } else {   // mixed edge types in the group (rare): compact code, per-edge weight rows
#pragma unroll 1
    for (int m = 0; m < CBG_NRBF; ++m) {
      const float4 gv = ld4(&M.g[m][e0]);
      const float gs[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
      for (int ee = 0; ee < 4; ++ee)
        fma4(a[ee], ld4(W.wrf + (t[ee] * CBG_NRBF + m) * CBG_H + 4 * lane), gs[ee]);
    }
  }
  }
  // LayerNorm(128, eps=1e-5) over the feature dim (4 per lane x 32 lanes), two-pass
  float s[4];
#pragma unroll
  for (int ee = 0; ee < 4; ++ee) s[ee] = (a[ee].x + a[ee].y) + (a[ee].z + a[ee].w);
  allreduce4(s, lane);
#pragma unroll
  for (int ee = 0; ee < 4; ++ee) {
    a[ee] = add4s(a[ee], -(s[ee] * (1.f / 128.f)));
    s[ee] = dot4(a[ee], a[ee]);
  }
  allreduce4(s, lane);
#pragma unroll
  for (int ee = 0; ee < 4; ++ee) {
    const float rstd = 1.f / sqrtf(s[ee] * (1.f / 128.f) + 1e-5f);
    a[ee] = ln_relu4(a[ee], rstd, gamma, beta);
  }
}

// Query-folded key matrix, lane-permuted: Up[c][hp] = U[c][hp ^ (lane>>1)] with
// U[c][hd] = sum_{d<8} q[hd*8+d] * W1[hd*8+d][4*lane+c]   (W1 natural [f_out][f_in] in smem).
__device__ __forceinline__ void build_u(const float* __restrict__ q_i, const float* s_w1, int lane,
                                        float (&U)[4][CBG_HEADS]) {
  const int hx = lane >> 1;
#pragma unroll
  for (int hp = 0; hp < CBG_HEADS; ++hp) {
    const int hd = hp ^ hx;
    const float4 q0 = ldg4(q_i + hd * 8), q1 = ldg4(q_i + hd * 8 + 4);
    const float qv[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
    float4 u = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int d = 0; d < 8; ++d) fma4(u, ld4(s_w1 + (hd * 8 + d) * CBG_H + 4 * lane), qv[d]);
    U[0][hp] = u.x; U[1][hp] = u.y; U[2][hp] = u.z; U[3][hp] = u.w;
  }
}

// Streaming head contraction + warp reduction.  For the 4 edges of a group and the 16 lane-permuted head
// slots hp, leaf(hp)[ee] = a[ee] . W(hp) (this lane's 4 features) must be summed over all lanes.  The
// halving butterfly  level 0: hp vs hp+8 (xor 16), 1: hp+4 (xor 8), 2: hp+2 (xor 4), 3: hp+1 (xor 2)  is
// evaluated depth first, so a partial result is shuffled as soon as its two halves exist: only ~24
// values are live instead of 64 and the shuffles overlap the FMAs of the next leaves.  Because slot hp
// holds head hp ^ (lane>>1), every lane keeps its lower half and sends its upper half: no selects.
template <int LVL, int HP, class Leaf>
struct HeadReduce {
  static __device__ __forceinline__ void run(const Leaf& leaf, float (&out)[4]) {
    float lo[4], hi[4];
    HeadReduce<LVL + 1, HP, Leaf>::run(leaf, lo);
    HeadReduce<LVL + 1, HP + (8 >> LVL), Leaf>::run(leaf, hi);
#pragma unroll
    for (int ee = 0; ee < 4; ++ee) out[ee] = lo[ee] + __shfl_xor_sync(CBG_FULL, hi[ee], 16 >> LVL);
  }
};
// level 3 evaluates its two leaves (head slots HP, HP+1) together so the dot products can use packed FMAs
template <int HP, class Leaf>
struct HeadReduce<3, HP, Leaf> {
  static __device__ __forceinline__ void run(const Leaf& leaf, float (&out)[4]) {
    float lo[4], hi[4];
    leaf.template eval2<HP>(lo, hi);
#pragma unroll
    for (int ee = 0; ee < 4; ++ee) out[ee] = lo[ee] + __shfl_xor_sync(CBG_FULL, hi[ee], 2);
  }
};
// last step: split on the high edge bit (lane bit 0).  r0, r1 = totals for head lane>>1 and edges
// 2*(lane&1), 2*(lane&1)+1 of the group.
template <class Leaf>
__device__ __forceinline__ void reduce_heads(const Leaf& leaf, int lane, float& r0, float& r1) {
  float f[4];
  HeadReduce<0, 0, Leaf>::run(leaf, f);
  const bool up = (lane & 1) != 0;
  const float s0 = up ? f[0] : f[2], s1 = up ? f[1] : f[3];
  const float k0 = up ? f[2] : f[0], k1 = up ? f[3] : f[1];
  r0 = k0 + __shfl_xor_sync(CBG_FULL, s0, 1);
  r1 = k1 + __shfl_xor_sync(CBG_FULL, s1, 1);
}

// leaf = a[ee] . Up[:,hp] with the lane-permuted, query-folded key matrix in registers
struct ULeaf {
  const float4 (&a)[4];
  const float (&U)[4][CBG_HEADS];
  template <int HP>
  __device__ __forceinline__ void eval2(float (&lo)[4], float (&hi)[4]) const {
#pragma unroll
    for (int ee = 0; ee < 4; ++ee) {
      float2 t = fmul2(make_float2(U[0][HP], U[0][HP + 1]), make_float2(a[ee].x, a[ee].x));
      t = ffma2(make_float2(U[1][HP], U[1][HP + 1]), make_float2(a[ee].y, a[ee].y), t);
      t = ffma2(make_float2(U[2][HP], U[2][HP + 1]), make_float2(a[ee].z, a[ee].z), t);
      t = ffma2(make_float2(U[3][HP], U[3][HP + 1]), make_float2(a[ee].w, a[ee].w), t);
      lo[ee] = t.x;
      hi[ee] = t.y;
    }
  }
};
// leaf = a[ee] . W[head][:] with the weight rows in shared memory ([16][128], lane-permuted head slot)
struct SmemLeaf {
  const float4 (&a)[4];
  const float* w;      // base of the [16][128] matrix
  int lane;
  template <int HP>
  __device__ __forceinline__ void eval2(float (&lo)[4], float (&hi)[4]) const {
    const float4 w0 = ld4(w + (HP ^ (lane >> 1)) * CBG_H + 4 * lane);
    const float4 w1 = ld4(w + ((HP + 1) ^ (lane >> 1)) * CBG_H + 4 * lane);
#pragma unroll
    for (int ee = 0; ee < 4; ++ee) { lo[ee] = dot4(a[ee], w0); hi[ee] = dot4(a[ee], w1); }
  }
};

__device__ __forceinline__ void contract_heads(const float4 (&a)[4], const float (&U)[4][CBG_HEADS], int lane,
                                               float& r0, float& r1) {
  reduce_heads(ULeaf{a, U}, lane, r0, r1);
}

// edge handled by this lane for value i (0/1) of group g under the reduce_heads mapping
__device__ __forceinline__ int lane_edge(int g, int lane, int i) { return 4 * g + 2 * (lane & 1) + i; }

// in-warp segment softmax over the 32 edges of head lane>>1: 16 logits per lane (8 groups x 2
// edges), the other 16 live in lane^1.  Returns alpha in place.
__device__ __forceinline__ void softmax32(float (&lg)[8][2], int lane, unsigned vmask) {
  float mx = -INFINITY;
#pragma unroll
  for (int g = 0; g < 8; ++g)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const bool valid = (vmask >> lane_edge(g, lane, i)) & 1u;
      if (!valid) lg[g][i] = -INFINITY;
      mx = fmaxf(mx, lg[g][i]);
    }
  mx = fmaxf(mx, __shfl_xor_sync(CBG_FULL, mx, 1));
  float sum = 0.f;
#pragma unroll
  for (int g = 0; g < 8; ++g)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      lg[g][i] = (mx == -INFINITY) ? 0.f : expf(lg[g][i] - mx);
      sum += lg[g][i];
    }
  sum += __shfl_xor_sync(CBG_FULL, sum, 1);
  const float inv = (sum > 0.f) ? sum : 1.f;
#pragma unroll
  for (int g = 0; g < 8; ++g)
#pragma unroll
    for (int i = 0; i < 2; ++i) lg[g][i] = lg[g][i] / inv;
}

// ------------------------------------------------------------------------------------------------
// X2H, part 1: attention weights  w[i][e][hd] = softmax_e(<q_i, k_ie>) * e_w[i][e]
// smem: K_WRF | K_C | K_LN | K_W1 | K_RBF  (contiguous in the blob) + per-warp EdgeMeta
constexpr int kX2hKFloats = 4 * 20 * 128 + 4 * 128 + 256 + 128 * 128 + 32;
constexpr int x2hk_smem(int w) { return kX2hKFloats * 4 + w * (int)sizeof(EdgeMeta); }

template <int kWarps>
__global__ void __launch_bounds__(kWarps * 32, 1) x2h_k_kernel(EdgeArgs p) {
  extern __shared__ __align__(16) float smem[];
  const float* s_wrf = smem;
  const float* s_c = s_wrf + 4 * 20 * 128;
  const float* s_ln = s_c + 4 * 128;
  const float* s_w1 = s_ln + 256;
  const float* s_rbf = s_w1 + 128 * 128;
  EdgeMeta* metas = reinterpret_cast<EdgeMeta*>(smem + kX2hKFloats);
  block_copy_f4(smem, p.layer + kOffX2hK, kX2hKFloats);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  EdgeMeta& M = metas[warp];
  const MlpSmem W{s_wrf, s_c};
  const float4 gamma = ld4(s_ln + 4 * lane), beta = ld4(s_ln + 128 + 4 * lane);

  const int n_list = list_length(p);
  NodeSched sch;
  for (int n = sch.first(p, blockIdx.x * kWarps + warp, gridDim.x * kWarps, lane); n < n_list; n = sch.nn) {
    sch.draw(n, lane);
    const int i = p.node_idx ? p.node_idx[n] : n;
    const unsigned vmask = edge_setup(M, i, lane, p.x4, p.nbr, p.ew, s_rbf, p.fstat);
    const float* rc = p.rc_k ? p.rc_k + (size_t)i * (CBG_KMAX * CBG_H) : nullptr;
    {
      const int nn = sch.next(lane);
      if (nn < n_list) prefetch_rc(p.rc_k, p.node_idx ? p.node_idx[nn] : nn, lane);
    }
    float U[4][CBG_HEADS];
    build_u(p.q + (size_t)i * CBG_H, s_w1, lane, U);
    const float4 pi = ldg4(p.pi_k + (size_t)i * CBG_H + 4 * lane);
    float lg[8][2];
#pragma unroll 1
    for (int g = 0; g < 8; ++g) {
      float4 a[4];
      first_layer4(M, 4 * g, lane, pi, p.pj_k, W, gamma, beta, a, rc);
      float r0, r1;
      contract_heads(a, U, lane, r0, r1);
#pragma unroll
      for (int gg = 0; gg < 8; ++gg) if (gg == g) { lg[gg][0] = r0; lg[gg][1] = r1; }
    }
    softmax32(lg, lane, vmask);
    float* wout = p.w + (size_t)i * (CBG_KMAX * CBG_HEADS);
#pragma unroll
    for (int g = 0; g < 8; ++g)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int e = lane_edge(g, lane, i);
        wout[e * CBG_HEADS + (lane >> 1)] = lg[g][i] * M.ew[e];
      }
    __syncwarp();   // M is rewritten by the next node's setup
  }
}

// ------------------------------------------------------------------------------------------------
// X2H, part 2: h_i += W1v (sum_e w_ie a_ie) + b1v sum_e w_ie   (per head)
// smem: V_WRF | V_C | V_LN | V_W1 | V_B1 | V_RBF + per-warp (EdgeMeta, wbuf[32][16])
constexpr int kX2hVFloats = 4 * 20 * 128 + 4 * 128 + 256 + 128 * 128 + 128 + 32;
constexpr int x2hv_smem(int w) { return kX2hVFloats * 4 + w * ((int)sizeof(EdgeMeta) + 32 * 16 * 4); }

template <int kWarps>
__global__ void __launch_bounds__(kWarps * 32, 1) x2h_v_kernel(EdgeArgs p) {
  extern __shared__ __align__(16) float smem[];
  const float* s_wrf = smem;
  const float* s_c = s_wrf + 4 * 20 * 128;
  const float* s_ln = s_c + 4 * 128;
  const float* s_w1 = s_ln + 256;
  const float* s_b1 = s_w1 + 128 * 128;
  const float* s_rbf = s_b1 + 128;
  EdgeMeta* metas = reinterpret_cast<EdgeMeta*>(smem + kX2hVFloats);
  float* wbufs = reinterpret_cast<float*>(metas + kWarps);
  block_copy_f4(smem, p.layer + kOffX2hV, kX2hVFloats);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  EdgeMeta& M = metas[warp];
  float* wbuf = wbufs + warp * (32 * 16);
  const MlpSmem W{s_wrf, s_c};
  const float4 gamma = ld4(s_ln + 4 * lane), beta = ld4(s_ln + 128 + 4 * lane);

  const int n_list = list_length(p);
  NodeSched sch;
  for (int n = sch.first(p, blockIdx.x * kWarps + warp, gridDim.x * kWarps, lane); n < n_list; n = sch.nn) {
    sch.draw(n, lane);
    const int i = p.node_idx ? p.node_idx[n] : n;
    edge_setup(M, i, lane, p.x4, p.nbr, p.ew, s_rbf, p.fstat);
    const float* rc = p.rc_v ? p.rc_v + (size_t)i * (CBG_KMAX * CBG_H) : nullptr;
    {
      const int nn = sch.next(lane);
      if (nn < n_list) prefetch_rc(p.rc_v, p.node_idx ? p.node_idx[nn] : nn, lane);
    }
    {
      const float* wsrc = p.w + (size_t)i * (CBG_KMAX * CBG_HEADS);
#pragma unroll
      for (int r = 0; r < 4; ++r) st4(wbuf + 4 * (lane + 32 * r), ld4(wsrc + 4 * (lane + 32 * r)));
    }
    __syncwarp();
    const float4 pi = ldg4(p.pi_v + (size_t)i * CBG_H + 4 * lane);
    float4 S[CBG_HEADS];
#pragma unroll
    for (int hd = 0; hd < CBG_HEADS; ++hd) S[hd] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
    for (int g = 0; g < 8; ++g) {
      float4 a[4];
      first_layer4(M, 4 * g, lane, pi, p.pj_v, W, gamma, beta, a, rc);
#pragma unroll
      for (int ee = 0; ee < 4; ++ee) {
        const float* wr = wbuf + (4 * g + ee) * 16;
        const float4 w0 = ld4(wr), w1 = ld4(wr + 4), w2 = ld4(wr + 8), w3 = ld4(wr + 12);
        const float wv[16] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w,
                              w2.x, w2.y, w2.z, w2.w, w3.x, w3.y, w3.z, w3.w};
#pragma unroll
        for (int hd = 0; hd < CBG_HEADS; ++hd) fma4(S[hd], a[ee], wv[hd]);
      }
    }
    // out[f'] = W1v[f'][:] . S[head(f')][:]  -> 128 partials per lane in two halves of 64.
    // Partial index = dp*8 + hh with f' = half*64 + hh*8 + (dp ^ (lane>>2)): the three steps over the
    // within-head bits are select-free (lane-permuted rows of W1v), the two steps over head bits
    // use selects.  Lane l ends with hh = 2*(l&3) + {0,1}, d = l>>2.
    const float* hin = p.h + (size_t)i * CBG_H;
    const int dx3 = lane >> 2;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      // g[hh] = sum over lanes of W1v[f(dp,hh)] . S[half*8+hh], reduced over the three within-head bits
      // (dp vs dp+4: xor 16, dp+2: xor 8, dp+1: xor 4) depth first, then the two head-bit steps with selects
      float part[8];
#pragma unroll
      for (int hh = 0; hh < 8; ++hh) {
        const float4 sv = S[half * 8 + hh];
        float lv[8];
#pragma unroll
        for (int dp = 0; dp < 8; ++dp) {
          const int f = half * 64 + hh * 8 + (dp ^ dx3);
          const float4 wv = ld4(s_w1 + f * CBG_H + 4 * lane);
          lv[dp] = dot4(wv, sv);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) lv[k] += __shfl_xor_sync(CBG_FULL, lv[k + 4], 16);
#pragma unroll
        for (int k = 0; k < 2; ++k) lv[k] += __shfl_xor_sync(CBG_FULL, lv[k + 2], 8);
        part[hh] = lv[0] + __shfl_xor_sync(CBG_FULL, lv[1], 4);
      }
      {   // hh bit 2 <-> lane bit 1
        const bool up = (lane & 2) != 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float send = up ? part[k] : part[k + 4];
          const float keep = up ? part[k + 4] : part[k];
          part[k] = keep + __shfl_xor_sync(CBG_FULL, send, 2);
        }
      }
      {   // hh bit 1 <-> lane bit 0
        const bool up = (lane & 1) != 0;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const float send = up ? part[k] : part[k + 2];
          const float keep = up ? part[k + 2] : part[k];
          part[k] = keep + __shfl_xor_sync(CBG_FULL, send, 1);
        }
      }
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int hh = 2 * (lane & 3) + k;
        const int hd = half * 8 + hh;
        const int f = half * 64 + hh * 8 + dx3;
        float sw = 0.f;
#pragma unroll
        for (int e = 0; e < 32; ++e) sw += wbuf[e * 16 + hd];
        p.h[(size_t)i * CBG_H + f] = hin[f] + (part[k] + s_b1[f] * sw);
      }
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// H2X for the generated nodes only (x moves only where gen_flag, unitransformer.py:182):
//   dx_i = (1/16) sum_hd sum_e alpha_ie^hd e_w (W1xv[hd] . a_v,ie + b1xv[hd]) (x_i - x_j)
// smem: K_WRF|K_C|K_LN|K_W1 | V_WRF|V_C|V_LN|V_W1(16x128)|V_B1(32) | RBF + per-warp EdgeMeta
constexpr int kH2xFloats = (4 * 20 * 128 + 4 * 128 + 256 + 128 * 128) + (4 * 20 * 128 + 4 * 128 + 256 + 16 * 128 + 32) + 32;
constexpr int h2x_smem(int w) { return kH2xFloats * 4 + w * (int)sizeof(EdgeMeta); }

template <int kWarps>
__global__ void __launch_bounds__(kWarps * 32, 1) h2x_kernel(EdgeArgs p) {
  extern __shared__ __align__(16) float smem[];
  const float* k_wrf = smem;
  const float* k_c = k_wrf + 4 * 20 * 128;
  const float* k_ln = k_c + 4 * 128;
  const float* k_w1 = k_ln + 256;
  const float* v_wrf = k_w1 + 128 * 128;
  const float* v_c = v_wrf + 4 * 20 * 128;
  const float* v_ln = v_c + 4 * 128;
  const float* v_w1 = v_ln + 256;        // [16][128]
  const float* v_b1 = v_w1 + 16 * 128;   // [32]
  const float* s_rbf = v_b1 + 32;
  EdgeMeta* metas = reinterpret_cast<EdgeMeta*>(smem + kH2xFloats);
  block_copy_f4(smem, p.layer + kOffH2x, kH2xFloats);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  EdgeMeta& M = metas[warp];
  const MlpSmem WK{k_wrf, k_c}, WV{v_wrf, v_c};
  const float4 kga = ld4(k_ln + 4 * lane), kbe = ld4(k_ln + 128 + 4 * lane);
  const float4 vga = ld4(v_ln + 4 * lane), vbe = ld4(v_ln + 128 + 4 * lane);
  const float b1 = v_b1[lane >> 1];      // this lane's head under the reduce_heads mapping

  for (int n = blockIdx.x * kWarps + warp; n < p.n_nodes; n += gridDim.x * kWarps) {
    const int i = p.node_idx[n];
    const unsigned vmask = edge_setup(M, i, lane, p.x4, p.nbr, p.ew, s_rbf, p.fstat);
    float U[4][CBG_HEADS];
    build_u(p.q + (size_t)i * CBG_H, k_w1, lane, U);
    const float4 pik = ldg4(p.pi_k + (size_t)i * CBG_H + 4 * lane);
    const float4 piv = ldg4(p.pi_v + (size_t)i * CBG_H + 4 * lane);
    float lg[8][2], vx[8][2];
#pragma unroll 1
    for (int g = 0; g < 8; ++g) {
      float4 a[4];
      first_layer4(M, 4 * g, lane, pik, p.pj_k, WK, kga, kbe, a, nullptr);
      float r0, r1;
      contract_heads(a, U, lane, r0, r1);
      // dynamic g: keep the register arrays statically indexed
#pragma unroll
      for (int gg = 0; gg < 8; ++gg) if (gg == g) { lg[gg][0] = r0; lg[gg][1] = r1; }
      first_layer4(M, 4 * g, lane, piv, p.pj_v, WV, vga, vbe, a, nullptr);
      reduce_heads(SmemLeaf{a, v_w1, lane}, lane, r0, r1);
#pragma unroll
      for (int gg = 0; gg < 8; ++gg) if (gg == g) { vx[gg][0] = r0 + b1; vx[gg][1] = r1 + b1; }
    }
    softmax32(lg, lane, vmask);
    float ax = 0.f, ay = 0.f, az = 0.f;
#pragma unroll
    for (int g = 0; g < 8; ++g)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int e = lane_edge(g, lane, i);
        const float coef = M.ew[e] * lg[g][i] * vx[g][i];
        ax = fmaf(coef, M.rel[0][e], ax);
        ay = fmaf(coef, M.rel[1][e], ay);
        az = fmaf(coef, M.rel[2][e], az);
      }
    ax = warp_sum(ax); ay = warp_sum(ay); az = warp_sum(az);
    if (lane == 0) st4(p.dx + 4 * (size_t)n, make_float4(ax * (1.f / 16.f), ay * (1.f / 16.f), az * (1.f / 16.f), 0.f));
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// R-cache build (once per batch): R[i][s][:] = c[t] + Wrf[t] g(|x_i - x_j|) for the s-th entry j of
// node i's static-only neighbour list.  blockIdx.y selects (layer, k|v MLP).
constexpr int kRcFloats = 4 * 20 * 128 + 4 * 128;   // Wrf | c (contiguous in the blob)
constexpr int kRcSmem = (kRcFloats + 32) * 4 + 8 * (20 * 32 + 32) * 4;

__global__ void __launch_bounds__(256) rcache_kernel(const float* __restrict__ layers, long long layer_stride,
                                                     const float4* __restrict__ x4, const int* __restrict__ snbr,
                                                     int n_nodes, float* __restrict__ rcache) {
  extern __shared__ __align__(16) float smem[];
  const int which = blockIdx.y & 1, layer = blockIdx.y >> 1;
  const float* L = layers + (size_t)layer * layer_stride;
  const float* wsrc = L + (which ? kOffX2hV : kOffX2hK);
  const float* rbf_src = L + (which ? kOffX2hVRbf : kOffX2hKRbf);
  float* s_wrf = smem;
  float* s_c = smem + 4 * 20 * 128;
  float* s_rbf = smem + kRcFloats;
  block_copy_f4(smem, wsrc, kRcFloats);
  if (threadIdx.x < 32) s_rbf[threadIdx.x] = rbf_src[threadIdx.x];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* g = smem + kRcFloats + 32 + warp * (20 * 32 + 32);   // g[m][s]
  int* ts = reinterpret_cast<int*>(g + 20 * 32);
  float* out_base = rcache + (size_t)blockIdx.y * n_nodes * (CBG_KMAX * CBG_H);
  for (int i = blockIdx.x * 8 + warp; i < n_nodes; i += gridDim.x * 8) {
    const float4 xi = x4[i];
    if (node_flags(xi) & 2) continue;                   // moving centre: no static edges
    const int jn = snbr[(size_t)i * CBG_KMAX + lane];
    const int j = jn >= 0 ? jn : i;
    const float4 xj = x4[j];
    const float rx = xi.x - xj.x, ry = xi.y - xj.y, rz = xi.z - xj.z;
    const float d = sqrtf(rx * rx + ry * ry + rz * rz);
    const float coeff = s_rbf[20];
#pragma unroll
    for (int m = 0; m < CBG_NRBF; ++m) { const float u = d - s_rbf[m]; g[m * 32 + lane] = expf(coeff * u * u); }
    ts[lane] = ((node_flags(xj) & 1) ? 0 : 2) + ((node_flags(xi) & 1) ? 0 : 1);
    __syncwarp();
    float* out = out_base + (size_t)i * (CBG_KMAX * CBG_H);
    for (int s0 = 0; s0 < 32; s0 += 4) {
      float4 a[4];
#pragma unroll
      for (int ee = 0; ee < 4; ++ee) a[ee] = ld4(s_c + ts[s0 + ee] * CBG_H + 4 * lane);
#pragma unroll 4
      for (int m = 0; m < CBG_NRBF; ++m) {
        const float4 gv = ld4(g + m * 32 + s0);
        const float gs[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
        for (int ee = 0; ee < 4; ++ee)
          fma4(a[ee], ld4(s_wrf + (ts[s0 + ee] * CBG_NRBF + m) * CBG_H + 4 * lane), gs[ee]);
      }
#pragma unroll
      for (int ee = 0; ee < 4; ++ee) st4(out + (s0 + ee) * CBG_H + 4 * lane, a[ee]);
    }
    __syncwarp();
  }
}

int g_num_sms = 0;
int g_edge_warps = 12;
int g_h2x_impl = -1;       // -1: follow g_edge_impl; CBG_H2X_IMPL=simt|tc overrides
int g_edge_impl = 6;       // 6 (default): wgmma tile kernels (x2h_tc.cu); 0: the fp32 SIMT kernels above (tested alternative, R-cache capable)
int g_h2x_warps = 12;

template <int W>
int set_attrs() {
  CBG_CUDA_OK(cudaFuncSetAttribute(x2h_k_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, x2hk_smem(W)));
  CBG_CUDA_OK(cudaFuncSetAttribute(x2h_v_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, x2hv_smem(W)));
  CBG_CUDA_OK(cudaFuncSetAttribute(h2x_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, h2x_smem(W)));
  return 0;
}

int edge_grid(int n_nodes, int warps) {
  const int need = (n_nodes + warps - 1) / warps;
  return need < g_num_sms ? need : g_num_sms;
}

template <int W>
int launch_x2h(const EdgeArgs& a, cudaStream_t st) {
  const int grid = edge_grid(a.n_nodes, W);
  EdgeArgs av = a;
  if (av.ticket) av.ticket += 1;          // the second kernel has its own work counter
  CBG_PROF_BEGIN(CBG_K_X2H_K, st);
  x2h_k_kernel<W><<<grid, W * 32, x2hk_smem(W), st>>>(a);
  CBG_LAUNCHED(CBG_K_X2H_K, st);
  CBG_PROF_BEGIN(CBG_K_X2H_V, st);
  x2h_v_kernel<W><<<grid, W * 32, x2hv_smem(W), st>>>(av);
  CBG_LAUNCHED(CBG_K_X2H_V, st);
  return 0;
}

template <int W>
int launch_h2x(const EdgeArgs& a, cudaStream_t st) {
  CBG_PROF_BEGIN(CBG_K_H2X, st);
  h2x_kernel<W><<<edge_grid(a.n_nodes, W), W * 32, h2x_smem(W), st>>>(a);
  CBG_LAUNCHED(CBG_K_H2X, st);
  return 0;
}

}  // namespace

int cbg_edge_init(void) {
  static bool done_dev[CBG_MAX_DEVICES] = {};
  bool& done = cbg_dev_flag(done_dev);
  if (done) return 0;
  int dev = 0;
  CBG_CUDA_OK(cudaGetDevice(&dev));
  CBG_CUDA_OK(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
  if (const char* e = getenv("CBG_EDGE_WARPS")) {
    const int w = atoi(e);
    if (w == 8 || w == 12 || w == 16) g_edge_warps = w;
  }
  if (const char* e = getenv("CBG_EDGE_IMPL")) {
    if (strcmp(e, "simt") == 0 || strcmp(e, "0") == 0) g_edge_impl = 0;
    else if (strcmp(e, "6") == 0 || strcmp(e, "tc") == 0) g_edge_impl = 6;
  }
  if (const char* e = getenv("CBG_H2X_IMPL")) {
    if (strcmp(e, "simt") == 0 || strcmp(e, "0") == 0) g_h2x_impl = 0;
    else if (strcmp(e, "6") == 0 || strcmp(e, "tc") == 0) g_h2x_impl = 6;
  }
  if (const char* e = getenv("CBG_H2X_WARPS")) {
    const int w = atoi(e);
    if (w == 8 || w == 12 || w == 16) g_h2x_warps = w;
  }
  if (int rc = set_attrs<8>()) return rc;
  if (int rc = set_attrs<12>()) return rc;
  if (int rc = set_attrs<16>()) return rc;
  done = true;
  return 0;
}

int cbg_launch_rcache(const float* layers, int num_layers, const float4* x4, const int* snbr, int n_nodes,
                      float* rcache, cudaStream_t st) {
  if (n_nodes <= 0 || num_layers <= 0) return 0;
  if (int rc = cbg_edge_init()) return rc;
  static bool attr_dev[CBG_MAX_DEVICES] = {};
  bool& attr = cbg_dev_flag(attr_dev);
  if (!attr) {
    CBG_CUDA_OK(cudaFuncSetAttribute(rcache_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kRcSmem));
    attr = true;
  }
  dim3 grid((unsigned)((n_nodes + 7) / 8 < 4 * g_num_sms ? (n_nodes + 7) / 8 : 4 * g_num_sms), 2 * num_layers);
  CBG_PROF_BEGIN(CBG_K_MISC, st);
  rcache_kernel<<<grid, 256, kRcSmem, st>>>(layers, cbg_layout::kLayerFloats, x4, snbr, n_nodes, rcache);
  CBG_LAUNCHED(CBG_K_MISC, st);
  return 0;
}

int cbg_launch_x2h(const EdgeArgs& a, cudaStream_t st) {
  if (a.n_nodes <= 0) return 0;
  if (int rc = cbg_edge_init()) return rc;
  if (g_edge_impl == 6) return cbg_launch_x2h_tc(a, st);       // wgmma tile kernels (x2h_tc.cu)
  switch (g_edge_warps) {
    case 8: return launch_x2h<8>(a, st);
    case 16: return launch_x2h<16>(a, st);
    default: return launch_x2h<12>(a, st);
  }
}

int cbg_launch_h2x(const EdgeArgs& a, cudaStream_t st) {
  if (a.n_nodes <= 0) return 0;
  if (int rc = cbg_edge_init()) return rc;
  // default: the wgmma tile kernel (x2h_tc.cu, needs the compact w scratch); the fp32 SIMT kernel below stays as the
  // independent cross-check (cbg_set_edge_impl(0) or CBG_H2X_IMPL=simt)
  if ((g_h2x_impl < 0 ? g_edge_impl : g_h2x_impl) == 6 && a.w != nullptr) return cbg_launch_h2x_tc(a, st);
  switch (g_h2x_warps) {
    case 8: return launch_h2x<8>(a, st);
    case 16: return launch_h2x<16>(a, st);
    default: return launch_h2x<12>(a, st);
  }
}

// testing hook (include/cbg_b200.h): pick the X2H edge-kernel implementation and the SIMT kernels' warps per CTA
int cbg_edge_set_impl(int impl, int warps) {
  if (int rc = cbg_edge_init()) return rc;
  if (impl != 0 && impl != 6) { cbg_set_error("edge impl must be 6 (wgmma, default) or 0 (fp32 SIMT)"); return 1; }
  if (warps != 0 && warps != 8 && warps != 12 && warps != 16) { cbg_set_error("warps per CTA must be 8, 12 or 16"); return 1; }
  g_edge_impl = impl;
  if (warps && impl == 0) g_edge_warps = warps;
  return 0;
}
