// gnnx_internal.cuh -- structures shared by the plan (k-hop extraction) kernels, the persistent
// explainer kernel and the C-ABI host code.  sm_90a (H100) only.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gnnx.h"

#define GX_MAX_LEVELS 8  // n_hops <= 7
#define GX_NONE16 0xFFFFu
#define GX_MAX_LAYERS 7  // num_gc_layers of a model variant (explain_var.cu): n_hops = num_gc_layers < GX_MAX_LEVELS; the tuned kernels build the reference default 3
#define GX_MAX_GANG 160   // CTAs that may share one task in explain_gang.cu (<= number of SMs)
#define GX_GRID_CAP (132 * 8)  // CTAs of a grid-stride launch: 8 per SM of an H100 (132 SMs)
#define GX_WP_SMEM_MAX 2048  // floats: pred_model (C x (2h+e) + C) is kept in shared memory up to this size

// One explained node ("task").  Counts are produced by khop_count_kernel, offsets by the host
// prefix sums, the packed arrays by khop_fill_kernel.
struct GxTask {
  int32_t node;     // global node id
  int32_t n;        // |k-hop set|
  int32_t e_d;      // directed entries of the induced sub-adjacency (self loops dropped)
  int32_t npairs;   // e_d / 2 undirected edges
  int32_t npairs_in;  // pairs with at least one endpoint in a row the forward computes (< n2): listed first
  int32_t idx_new;  // rank of `node` among its ascending neighbours (explain.py:496)
  int32_t gt_label; // label[node]
  int32_t n1, n2;   // level-order prefix sizes: |dist<=L-2|, |dist<=L-1| for L=3 -> |dist<=1|, |dist<=2|
  int32_t e1;       // directed entries whose source row is < n2 (what the forward ever gathers)
  int32_t status;   // 0 ok; 1 node not inside its own neighbourhood
  int32_t n_norm;   // the n of the reference's dense tensors (1/n^2 factors, M0 std): n in node mode, max_nodes in graph mode
  int32_t flags;    // graph mode: bit 0 = some row of the padded graph has no edge (its constant embedding joins the max-pool)
  int32_t loops;    // node mode: members with a self loop (the diagonal of the reference's sub_adj; not among the e_d entries)
  int32_t cum[GX_MAX_LEVELS + 1];  // cum[t] = #nodes with dist <= t (dist measured from `node`)
  int32_t smem_bytes;              // shared-memory footprint of this task in the explainer kernel
  int64_t node_off;  // into nbrs / lo2gid
  int64_t rp_off;    // into sub_rowptr / irowptr (= node_off + task index: n+1 entries per task)
  int64_t edge_off;  // into sub_col / icol / m0 / edge_mask
  int64_t pair_off;  // into the pair arrays
};

// Device-resident plan arrays (all int32).
struct GxPlanArrays {
  GxTask* tasks;
  int32_t* nbrs;        // [total_n] ascending global ids (canonical order)
  int32_t* lo2gid;      // [total_n] global id of the node with level-order id i
  int32_t* sub_rowptr;  // [total_n + count] canonical CSR, task-local
  int32_t* sub_col;     // [total_e]
  int32_t* irowptr;     // [total_n + count] level-order CSR, task-local
  int32_t* icol;        // [total_e] level-order ids; per row partitioned by level of the neighbour
  int32_t* cs2is;       // [total_e] canonical slot -> internal slot (task-local)
  int32_t* is2cs;       // [total_e] internal slot -> canonical slot
  int32_t* pair_i;      // [total_e/2] i < j, level-order ids
  int32_t* pair_j;
  int32_t* pair_pij;    // position of j in internal row i (absolute, task-local)
  int32_t* pair_pji;
  int32_t* pair_oij;    // canonical edge slot of (i,j) (task-local index into the edge arrays)
  int32_t* pair_oji;
};

struct GxGraphDev {
  int64_t N;
  int32_t nnz;
  const int32_t* rowptr;
  const int32_t* col;
  const float* feat;  // [N*d]
  int32_t d;
  const int32_t* label;
  const int32_t* pred_label;
};

struct GxModelDev {
  int32_t d, hid, emb, C, L;
  int32_t bn;          // --bn: per-node standardisation after every hidden ReLU (models.py:222-228)
  int32_t variant;     // 1: num_layers != 3 or bn or att -> every task runs in explain_var.cu with the UNPADDED widths hid / emb
  int32_t att;         // --method att: every layer scales the masked adjacency by s_ij = P_i . P_j, P = H_{l-1} Wa_l (models.py:62-68)
  const float* W[GX_MAX_LAYERS];   // row-major (in,out)
  const float* Wt[GX_MAX_LAYERS];  // row-major (out,in) (default model only)
  const float* b[GX_MAX_LAYERS];   // never NULL on device (zeros when --nobias)
  const float* Wp;     // (C, 2*hid+emb)
  const float* bp;
};
// att models: layer l's attention weights (conv_*.att_weight, row-major (in, in)) follow its conv weights in the model buffer, so the
// struct (a kernel argument of every explainer kernel) keeps its size
__host__ __device__ inline const float* gx_att_weight(const GxModelDev& m, int l) {
  return m.W[l] + (l == 0 ? m.d : m.hid) * (l == m.L - 1 ? m.emb : m.hid);
}

// MLP prediction head (gx_set_model_head, models.py:193-207): k hidden Linear + ReLU layers of widths w[0 .. k-1], then Linear(., C).
// The k + 1 Linears lie back to back at W, each as its row-major (out, in) weight followed by its out biases, so that the head is one
// block (staged in shared memory with one copy when it fits).  k = 0: no head, pred_model is GxModelDev's Wp / bp.  A separate kernel
// argument of the variant, dense and forward kernels: GxModelDev is also an argument of the tuned kernels, which never see a head.
struct GxHeadDev {
  int32_t k;
  int32_t w[GX_MAX_HEAD_LAYERS];
  const float* W;
};
__host__ __device__ inline int gx_head_in(const GxHeadDev& hd, int PD, int j) { return j == 0 ? PD : hd.w[j - 1]; }
__host__ __device__ inline int gx_head_out(const GxHeadDev& hd, int C, int j) { return j == hd.k ? C : hd.w[j]; }
// words of Linear 0 .. j-1 in the block (j = k + 1: the whole head; k = 0: C (PD + 1), pred_model's weight and bias)
__host__ __device__ inline int gx_head_off(const GxHeadDev& hd, int PD, int C, int j) {
  int o = 0;
  for (int i = 0; i < j; ++i) o += gx_head_out(hd, C, i) * (gx_head_in(hd, PD, i) + 1);
  return o;
}
__host__ __device__ inline int gx_head_words(const GxHeadDev& hd, int PD, int C) { return gx_head_off(hd, PD, C, hd.k + 1); }
__host__ __device__ inline int gx_head_act_words(const GxHeadDev& hd) { int s = 0; for (int j = 0; j < hd.k; ++j) s += hd.w[j]; return s; }
__host__ __device__ inline int gx_head_max_width(const GxHeadDev& hd) { int s = 0; for (int j = 0; j < hd.k; ++j) s = hd.w[j] > s ? hd.w[j] : s; return s; }

struct GxHparamsDev {
  int32_t iters;     // forward/backward/update iterations executed: num_epochs - 1 (the last epoch's backward is unobservable), num_epochs when a trace is requested
  int32_t out_iter;  // the mask (and the optimiser state) is emitted after this many updates: num_epochs - 1
  float one_minus_b1, b2, one_minus_b2, eps;
  float c_size, c_feat_size, c_ent, c_lap;
  const float2* adam_tab;  // [iters] Adam: (step_size_t = lr_t/(1-b1^t), sqrt(1-b2^t)) for t = start_step + 1 .., computed in double on the host; other optimisers: (lr_t, 0).  lr_t follows the scheduler
  int32_t init;
  int32_t flags;  // GX_HP_* bits
  int32_t opt;    // GX_OPT_*; the tuned kernels build Adam only (others: explain_var.cu + outer_pairs_kernel)
  int32_t mode;   // 0: mask optimisation; 1: gradient baseline (explain(model="grad")): one forward/backward on the unmasked subgraph
  uint64_t seed;
};

#define GX_HP_IEEE_EDGE 1  // edge phase with IEEE exp/div/sqrt instead of the hardware approximations (test knob)
#define GX_HP_NODE_GENERIC 2   // explain_node.cu: never the narrow instantiation (test / A-B knob)

// Optional trace / optimiser-state buffers of gx_explain_io (device pointers, nullptr = unused).
struct GxExtra {
  float* trace;        // [count][epochs][GX_TRACE_COLS]: the explainer kernels write raw per-epoch terms, trace_finalize_kernel assembles the columns
  float* trace_pred;   // [count][epochs][C]
  double* tr_outer;    // [count][epochs][4]: (sum S, sum H(S), sum a (y_i-y_j)^2, sum 2a after the step) over the outer pairs
  int32_t epochs;      // trace rows per task (= num_epochs of the call)
  const float* adam_m_in; const float* adam_v_in; const float* feat_state_in;
  float* mask_param_out; float* adam_m_out; float* adam_v_out; float* feat_state_out;
};

// ---------------------------------------------------------------------------------------------
// Shared-memory layout of one task in the explainer kernel.  Computed identically on host
// (classification of tasks into launch classes) and device (carve-up).
// ---------------------------------------------------------------------------------------------
__host__ __device__ inline int gx_round_up(int x, int m) { return (x + m - 1) / m * m; }

struct GxLayout {
  // float arrays (offsets in 4-byte words)
  int X, U, Yh1, q1, Yh2, q2, dZ2, a, y, W1s, W1t, W2s, W2t, W3s, bs, sF, F, mF, vF, gFp, zs, dE, dZ3, logit, Wp;
  // index arrays (offsets in 4-byte words; element type IdxT)
  int icol, irp, llist, cnt1, llistB;
  int total_words;
  int dp;
};

// Shared-memory footprint of one task.  np_in = pairs with an endpoint in rows < n2: their optimiser state and
// their indices live in a per-CTA global slab that stays in L2 (read once per epoch, in the pair phase, so
// shared memory would only buy latency the phase already hides); pairs between two outermost nodes never
// touch the forward and are optimised by a separate elementwise kernel.
// idx_bytes = sizeof(IdxT) (2 or 4).  hid/emb must be multiples of 4.
__host__ __device__ inline GxLayout gx_make_layout(int n, int n1, int n2, int e1, int d,
                                                   int hid, int emb, int C, int nwarps,
                                                   int idx_bytes, int cs = 1) {
  GxLayout L;
  const int dp = gx_round_up(d, 4);
  L.dp = dp;
  int o = 0;
  auto takef = [&](int words) { int r = o; o += gx_round_up(words, 4); return r; };
  auto takei = [&](int elems) { int r = o; o += gx_round_up((elems * idx_bytes + 3) / 4, 4); return r; };
  L.X = takef(n * dp);
  L.U = takef(n2 * dp);      // A_m X in the forward; overwritten row by row with dZ1 (.) sF in the backward
  L.Yh1 = takef(n2 * hid);
  L.q1 = takef(n2);
  L.Yh2 = takef(n1 * hid);
  L.q2 = takef(n1);
  L.dZ2 = takef(n1 * hid);
  L.a = takef(e1);
  L.y = takef(n);            // float(pred_label) per node (Laplacian regulariser)
  L.W1s = takef(dp * hid);   // [dp][hid]   rows >= d are zero
  L.W1t = takef(hid * dp);   // [hid][dp]   transposed
  L.W2s = takef(hid * hid);
  L.W2t = takef(hid * hid);
  L.W3s = takef(hid * emb);
  L.bs = takef(2 * hid + emb);
  L.sF = takef(dp);
  L.F = takef(dp);
  L.mF = takef(dp);
  L.vF = takef(dp);
  L.gFp = takef(nwarps * cs * dp);   // per-warp dL/dsF partials of every CTA of the cluster (cs = cluster size)
  L.zs = takef(nwarps * 128);
  L.dE = takef(2 * hid);
  L.dZ3 = takef(hid);
  L.logit = takef(C < 32 ? 32 : C);
  L.Wp = takef(C * (2 * hid + emb + 1) <= GX_WP_SMEM_MAX ? C * (2 * hid + emb + 1) : 0);  // pred_model weights + bias when small
  L.icol = takei(e1);
  L.irp = takei(n2 + 1);
  L.llist = takei(n2);
  L.cnt1 = takei(n2);        // per row: number of leading columns < n1 (the only ones that carry dZ2)
  L.llistB = takei(n2);      // rows whose < n1 prefix is long (split across a whole warp in the backward)
  L.total_words = o;
  return L;
}

// Global-memory slab of one task in the streaming kernel (explain_stream.cu: tasks whose state does not fit
// shared memory).  Offsets in 4-byte words; the CSR / pair index arrays are read straight from the plan.
struct GxStreamLayout {
  int64_t a, gE, P, dP, Yh1, q1, dY1, Yh2, q2, dZ2, lapg, cnt1, cnt2, gFp, gFb, longlist, trw, xlo;
  int64_t total_words;
  int dp;
};
__host__ __device__ inline GxStreamLayout gx_make_stream_layout(int n, int n1, int n2, int e_d, int np_in, int d, int hid, int nwarps) {
  GxStreamLayout L;
  const int dp = gx_round_up(d, 4);
  L.dp = dp;
  int64_t o = 0;
  auto take = [&](int64_t words) { int64_t r = o; o += (words + 3) / 4 * 4; return r; };
  L.a = take(e_d);                     // masked-adjacency value of every internal slot (rows >= n2: only their < n2 prefix is live)
  L.gE = take(e_d);                    // layer-1 edge-gradient dot <dY1[col], P[row]> of every live slot (0 elsewhere)
  L.P = take((int64_t)n * hid);        // (X . sF) W1 of every node
  L.dP = take((int64_t)n * hid);       // A_m^T dY1 of every node
  L.Yh1 = take((int64_t)n2 * hid); L.q1 = take(n2); L.dY1 = take((int64_t)n2 * hid);
  L.Yh2 = take((int64_t)n1 * hid); L.q2 = take(n1); L.dZ2 = take((int64_t)n1 * hid);
  L.lapg = take(np_in);               // per inner pair: its (epoch-invariant) Laplacian-regulariser gradient
  L.cnt1 = take(n2);                   // per row < n2: leading columns < n1
  L.cnt2 = take(n);                    // per row: leading columns < n2
  L.gFp = take((int64_t)nwarps * dp);
  // explain_gang.cu: dL/dsF partials of the 128-node blocks, rows sliced over a whole CTA, per-warp trace partials of a gang
  L.gFb = take((int64_t)((n + 127) / 128) * dp);
  L.longlist = take(n);
  L.trw = take(GX_MAX_GANG * 32 * 4);
  L.xlo = take((int64_t)(n + 16) * (gx_round_up(d, 8) + 4));   // the task's feature rows in level order, padded to the shared-memory tile pitch
  L.total_words = o;
  return L;
}

// Global-memory slab of one task in the model-variant kernel (explain_var.cu); hidden-width arrays have row stride vw = 32 * ceil(width / 32).
// Graph mode computes every one of its n rows with an edge at every layer (n2 = n, e1 = e_d) and has no Laplacian term (np_in = 0).
// Attention models (att != 0, e_d = all directed slots of the task) add the per-layer projections and edge weights; for any other
// model these arrays take zero words.
// Wide inputs (wide != 0: d > 128) contract layer 1 as A_m (X (sigmoid(F) (.) W1)): U and dZ1 take zero words, the masked adjacency
// covers all e_d slots (dP gathers over the rows beyond n2), and the feature-mask state and the hid-wide products P, dY1, dP and G
// live here.  For d <= 128 these arrays take zero words.
struct GxVarLayout {
  int64_t a, U, dZ1, lapg, Yh, H, dZ, q, istd;
  int64_t P, s, as, t, cw, dHa;
  int64_t fm, XB, dY1, dP, G;
  int64_t total_words;
};
__host__ __device__ inline GxVarLayout gx_make_var_layout(int n, int n2, int e1, int np_in, int d, int L, int vw = 32, int att = 0,
                                                          int e_d = 0, int wide = 0) {
  GxVarLayout Lo;
  const int dp = gx_round_up(d, 4);
  int64_t o = 0;
  auto take = [&](int64_t words) { int64_t r = o; o += (words + 3) / 4 * 4; return r; };
  (void)n;
  Lo.a = take(wide ? e_d : e1);               // masked adjacency of the rows the forward visits (level-order rows < n2; wide: every row)
  Lo.U = take(wide ? 0 : (int64_t)n2 * dp);   // A_m X
  Lo.dZ1 = take(wide ? 0 : (int64_t)n2 * dp); // dL/d(A_m X') (.) sigmoid(feat_mask)
  Lo.lapg = take(np_in);
  Lo.Yh = take((int64_t)L * n2 * vw);         // per layer: normalised pre-activations (row stride vw = 32 * ceil(width / 32))
  Lo.H = take((int64_t)L * n2 * vw);          // per layer: relu (+ standardisation) output = input of the next layer / the readout
  Lo.dZ = take((int64_t)(L - 1) * n2 * vw);   // layers 2..L: dL/d(A_m H_{l-1})
  Lo.q = take((int64_t)L * n2);
  Lo.istd = take((int64_t)L * n2);
  const int64_t at = att ? 1 : 0;
  Lo.P = take(at * ((int64_t)n * dp + (int64_t)(L - 1) * n2 * vw));   // per layer: P = H_{l-1} Wa on the layer's input rows (layer 1: n rows, stride dp)
  Lo.s = take(at * L * e1);                   // per layer and slot: s_ij = P_i . P_j
  Lo.as = take(at * L * e1);                  // per layer and slot: the aggregation weight a_ij s_ij
  Lo.t = take(at * L * e1);                   // per layer and slot of a row of the layer: t_ij = dL/dZ_i . H_{l-1}[j]
  Lo.cw = take(at * e_d);                     // the current layer's a_ij (t_ij + t_ji) on every slot (rows beyond n2 included)
  Lo.dHa = take(at * n2 * vw);                // dL/dP Wa^T of the layer above: the attention's share of dL/dH
  const int64_t wd = wide ? 1 : 0;
  Lo.fm = take(wd * 5 * dp);                  // sigmoid(F), F, the optimiser's two moments, dL/dsigmoid(F) (dp words each)
  Lo.XB = take(wd * n * vw);                  // P = X (sigmoid(F) (.) W1) of every row of the task
  Lo.dY1 = take(wd * n2 * vw);                // dL/dY of layer 1's rows
  Lo.dP = take(wd * n * vw);                  // A_m^T dY1 of every row
  Lo.G = take(wd * dp * vw);                  // X^T dP (d, hid)
  Lo.total_words = o;
  return Lo;
}

// Shared-memory footprint of one graph-mode task (all `na` rows with at least one edge are computed at every layer).
struct GxLayoutG {
  int X, U, Yh1, Yh2, Yh3, q, dZ2, dZ3, a, W1s, W1t, W2s, W2t, W3s, W3t, bs, cst, emb, dE, sF, F, mF, vF, gFp, zs, logit, Wp;
  int arg, icol, irp, pi, pj, ppij, ppji;
  int total_words;
  int dp;
};
__host__ __device__ inline GxLayoutG gx_make_layout_graph(int na, int e_d, int np, int d, int hid, int emb, int C, int nwarps) {
  GxLayoutG L;
  const int dp = gx_round_up(d, 4);
  L.dp = dp;
  int o = 0;
  auto takef = [&](int words) { int r = o; o += gx_round_up(words, 4); return r; };
  auto takei = [&](int elems) { int r = o; o += gx_round_up((elems * 2 + 3) / 4, 4); return r; };
  L.X = takef(na * dp); L.U = takef(na * dp);
  L.Yh1 = takef(na * hid); L.Yh2 = takef(na * hid); L.Yh3 = takef(na * emb);
  L.q = takef(3 * na);
  L.dZ2 = takef(na * hid); L.dZ3 = takef(na * hid);
  L.a = takef(e_d);
  L.W1s = takef(dp * hid); L.W1t = takef(hid * dp); L.W2s = takef(hid * hid); L.W2t = takef(hid * hid);
  L.W3s = takef(hid * emb); L.W3t = takef(emb * hid);
  L.bs = takef(2 * hid + emb);
  L.cst = takef(2 * hid + emb);   // embedding of an edge-less row: relu(normalize(b_l)) / normalize(b_3)
  L.emb = takef(2 * hid + emb);
  L.dE = takef(2 * hid + emb);
  L.sF = takef(dp); L.F = takef(dp); L.mF = takef(dp); L.vF = takef(dp);
  L.gFp = takef(nwarps * dp);
  L.zs = takef(nwarps * 128);
  L.logit = takef(C < 32 ? 32 : C);
  L.Wp = takef(C * (2 * hid + emb + 1) <= GX_WP_SMEM_MAX ? C * (2 * hid + emb + 1) : 0);
  L.arg = takef(2 * hid + emb);   // int: arg-max row of every pooled feature (-1: the edge-less constant)
  L.icol = takei(e_d); L.irp = takei(na + 1);
  L.pi = takei(np); L.pj = takei(np); L.ppij = takei(np); L.ppji = takei(np);
  L.total_words = o;
  return L;
}

// Global-memory slab of one task in the unconstrained kernel (explain_dense.cu): the dense n x n state and the per-layer activations of
// all n rows.  Hc / dZc hold, per row, the layer inputs X = H_0, H_1 .. H_L and the matching dL/d(A_m H_{l-1}) side by side: column
// offset 0 for X / dZ_1 (width d), off1 + (l - 1) vw for H_l / dZ_{l+1} (vw = 32 * ceil(width / 32)), so that every pair gradient
// sum_l dZ_l H_{l-1}^T is ONE product dZc Hc^T over the first k_pair columns; padding columns stay zero.
constexpr int GX_DENSE_MAX_N = 4096;   // 16.7 M mask parameters per task, the bound of graph mode's max_nodes
struct GxDenseLayout {
  int64_t M, m, v, a, G, Hc, dZc, Z, Yh, q, istd;
  int64_t total_words;
  int off1, kh, k_pair, zw;
};
__host__ __device__ inline GxDenseLayout gx_make_dense_layout(int n, int d, int L, int vw) {
  GxDenseLayout Lo;
  Lo.off1 = gx_round_up(d, 8);
  Lo.k_pair = Lo.off1 + (L - 1) * vw;
  Lo.kh = Lo.k_pair + vw;
  Lo.zw = Lo.off1 > vw ? Lo.off1 : vw;
  const int64_t nn = (int64_t)n * n;
  int64_t o = 0;
  auto take = [&](int64_t words) { int64_t r = o; o += (words + 3) / 4 * 4; return r; };
  Lo.M = take(nn); Lo.m = take(nn); Lo.v = take(nn);   // mask parameter and optimiser state of every directed entry (i, j) at i * n + j
  Lo.a = take(nn);                                      // masked adjacency sym(sigmoid(M)) (.) (1 - I)
  Lo.G = take(nn);                                      // pair-gradient product dZc Hc^T
  Lo.Hc = take((int64_t)n * Lo.kh);
  Lo.dZc = take((int64_t)n * Lo.kh);
  Lo.Z = take((int64_t)n * Lo.zw);                      // output of the current aggregation product
  Lo.Yh = take((int64_t)L * n * vw);                    // per layer: normalised pre-activations
  Lo.q = take((int64_t)L * n);
  Lo.istd = take((int64_t)L * n);
  Lo.total_words = o;
  return Lo;
}

// ---------------------------------------------------------------------------------------------
#define GX_CUDA_CHECK(expr)                                                      \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      gx_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                   __LINE__);                                                        \
      return GX_ERR_CUDA;                                                            \
    }                                                                                \
  } while (0)

void gx_set_error(const char* fmt, ...);

// kernel launchers (defined in khop.cu / explain_node.cu)
struct GxSlotWs {
  uint32_t* bm;     // [slots * W]   membership bitmap (must be all-zero between tasks)
  int32_t* wpref;   // [slots * (W+1)]
  uint8_t* dist;    // [slots * N]
  int32_t* q;       // [slots * (N+1)]
  int32_t* loc;     // [slots * N]  level-order id by canonical id
  int32_t* cof;     // [slots * N]  canonical id by level-order id
  int32_t* pbase;   // [slots * (N+1)]
  int32_t W;        // words per bitmap
  int32_t slots;
};

cudaError_t gx_launch_khop_count(const GxGraphDev& g, const int32_t* nodes_dev, int count, int k,
                                 int row_lvl, GxSlotWs ws, GxTask* tasks, cudaStream_t s);
cudaError_t gx_launch_khop_fill(const GxGraphDev& g, int count, int k, GxSlotWs ws, GxPlanArrays plan,
                                cudaStream_t s);
cudaError_t gx_launch_hop_rows(const GxGraphDev& g, const int32_t* nodes_dev, int count, int k,
                               GxSlotWs ws, uint8_t* out_rows, cudaStream_t s);

struct GxExplainLaunch {
  const int32_t* order;  // [ntasks] task ids of this launch class, most expensive first
  int32_t ntasks;
  int32_t* counter;      // device work-queue counter (zeroed)
  int32_t smem_bytes;    // dynamic shared memory per CTA (shared-memory classes)
  int32_t threads;
  int32_t grid;
  int32_t cluster = 1;   // CTAs per task (thread-block cluster size): 1, 2 or 4 (explain_node.cu cluster class)
  int32_t gang = 1;      // explain_gang.cu: co-resident CTAs per task (grid = gangs * gang)
  unsigned long long* gang_bars = nullptr;   // [gangs] barrier counters, zeroed
  int32_t* gang_mail = nullptr;              // [gangs * 2]
  float* gws;            // per-CTA global slab of the streaming class
  int64_t gws_stride_words;
  float* pws;            // per-CTA pair-state slab: 8 floats per inner pair (M,m,v,S of both directions)
  int64_t pws_stride_words;
  float* dbg;            // debug dump buffer (device) or NULL
  GxExtra x;             // optional trace / optimiser-state buffers
};
cudaError_t gx_launch_explain(const GxExplainLaunch& cfg, const GxGraphDev& g, const GxModelDev& m,
                              const GxHparamsDev& hp, const GxPlanArrays& plan, const float* m0,
                              float* out_mask, float* out_feat, cudaStream_t s);
cudaError_t gx_launch_explain_stream(const GxExplainLaunch& cfg, const GxGraphDev& g, const GxModelDev& m,
                                     const GxHparamsDev& hp, const GxPlanArrays& plan, const float* m0,
                                     float* out_mask, float* out_feat, cudaStream_t s);
cudaError_t gx_launch_explain_gang(const GxExplainLaunch& cfg, const GxGraphDev& g, const GxModelDev& m,
                                   const GxHparamsDev& hp, const GxPlanArrays& plan, const float* m0,
                                   float* out_mask, float* out_feat, cudaStream_t s);
int gx_gang_smem_bytes(int d, int hid, int C);
cudaError_t gx_launch_model_forward(const GxGraphDev& g, const GxModelDev& m, const GxHeadDev& hd, float* H, float* pred, float* emb_out, float* P,
                                    cudaStream_t s);
constexpr int GX_STREAM_THREADS = 768;  // 24 warps: 80 registers per thread, 5 KB of cp.async staging per warp
int gx_explain_max_smem();
struct GxGraphBatchDev {
  int32_t num_graphs, max_nodes, d;
  const int32_t* rowptr;  // [G*max_nodes+1], global edge offsets
  const int32_t* col;     // node id within the graph
  const float* feat;      // [G*max_nodes*d]
  const int32_t* label;   // [G]
};
cudaError_t gx_launch_graph_plan(const GxGraphBatchDev& gb, int count, GxPlanArrays plan, cudaStream_t s);
// grad_label: hp.mode == 1 only, one loss label per task (-1: the forward's arg-max)
cudaError_t gx_launch_explain_graphs(const GxExplainLaunch& cfg, const GxGraphBatchDev& gb, const GxModelDev& m,
                                     const GxHparamsDev& hp, const GxPlanArrays& plan, const float* m0, float* out_mask,
                                     float* out_feat, const int32_t* grad_label, cudaStream_t s);
// explain_var.cu: the model and optimiser variants, node mode (graph_mode 0, g) or graph mode (gb)
cudaError_t gx_launch_explain_var(const GxExplainLaunch& cfg, int graph_mode, const GxGraphDev& g, const GxGraphBatchDev& gb,
                                  const GxModelDev& m, const GxHeadDev& hd, const GxHparamsDev& hp, const GxPlanArrays& plan, const float* m0,
                                  float* out_mask, float* out_feat, cudaStream_t s);
int gx_var_smem_bytes(int graph_mode, int d, int L, int hid, int emb, int C, int att = 0, const GxHeadDev& hd = GxHeadDev{});
constexpr int GX_VAR_WIDE_MIN = 129;    // input widths from here on run the variant kernel's wide path (layer 1 contracted as A_m (X B))
constexpr int GX_VAR_WIDE_MAX = 4096;   // the largest input width the wide path builds
int gx_var_ctas_per_sm(int graph_mode, const GxModelDev& m, const GxHeadDev& hd);
int gx_var_row_stride(int hid, int emb);
// explain_dense.cu: Explainer.explain(..., unconstrained=True), node mode (graph_mode 0, g) or graph mode (gb); m0 / out_dense are dense
// (dense_off[t] = the offset of task t's n_t^2 block), out_mask holds the sub-adjacency slots, x.trace / x.trace_pred optional.
struct GxDenseIo {
  const int64_t* dense_off;
  const float* m0;
  float* out_mask;
  float* out_dense;
  float* trace;
  float* trace_pred;
  int32_t epochs;
};
cudaError_t gx_launch_explain_dense(const GxExplainLaunch& cfg, int graph_mode, const GxGraphDev& g, const GxGraphBatchDev& gb,
                                    const GxModelDev& m, const GxHeadDev& hd, const GxHparamsDev& hp, const GxPlanArrays& plan,
                                    const GxDenseIo& io, cudaStream_t s);
int gx_dense_smem_bytes(int d, int L, int hid, int emb, int C, const GxHeadDev& hd = GxHeadDev{});
int gx_dense_ctas_per_sm(const GxModelDev& m, const GxHeadDev& hd);
cudaError_t gx_launch_outer_pairs(const GxHparamsDev& hp, const GxGraphDev& g, const GxPlanArrays& plan, int count,
                                  const float* m0, float* out_mask, const GxExtra& x, cudaStream_t s);
cudaError_t gx_launch_denoise_topk(const GxPlanArrays& plan, int count, const float* edge_mask, int k2, int cap, float* out_thr,
                                   int32_t* out_cnt, int32_t* out_slots, float* out_vals, cudaStream_t s);
cudaError_t gx_launch_denoise_topk_edges(const GxPlanArrays& plan, int count, const float* edge_mask, int k2, int cap, float* out_thr,
                                         int32_t* out_cnt, int32_t* out_uv, float* out_vals, cudaStream_t s);
// comm.cu
struct GxComm;
int gx_comm_impl_unique_id(char* id128);
int gx_comm_impl_init(GxComm** out, int world, int rank, const char* id128);
void gx_comm_impl_destroy(GxComm* c);
int gx_comm_impl_world(const GxComm* c);
int gx_comm_impl_rank(const GxComm* c);
int gx_comm_impl_allgather(GxComm* c, const float* send, float* recv, size_t slot_floats, cudaStream_t s);
cudaError_t gx_launch_unshard(const float* gathered, int items, const int64_t* src, const int64_t* dst, const int32_t* sz, float* out, cudaStream_t s);
// trace.cu
cudaError_t gx_launch_trace_finalize(const GxHparamsDev& hp, const GxPlanArrays& plan, int count, const GxExtra& x, cudaStream_t s);
cudaError_t gx_launch_offedge(const GxHparamsDev& hp, const GxPlanArrays& plan, int count, int epochs, const int64_t* dense_off,
                              const float* m0_dense, double* out, cudaStream_t s);
cudaError_t gx_launch_offedge_graphs(const GxHparamsDev& hp, const GxPlanArrays& plan, const GxGraphBatchDev& gb, int count, int epochs,
                                     const float* m0_dense, double* out, cudaStream_t s);
cudaError_t gx_launch_densify(const GxPlanArrays& plan, int count, const int64_t* dense_off,
                              const float* edge_mask, double* out, cudaStream_t s);
// densify_graphs.cu: gids[count] and val_off[count] (start of graph t's packed slots in values) are device arrays
cudaError_t gx_launch_densify_graphs(const GxGraphBatchDev& gb, const int32_t* gids, int count, const int64_t* val_off,
                                     const float* values, double* out, cudaStream_t s);
