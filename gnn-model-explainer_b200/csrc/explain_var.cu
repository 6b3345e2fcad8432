// explain_var.cu -- K2v: the mask-optimisation kernel for the model and optimiser VARIANTS of the reference (SURVEY 8 row f3), node
// mode and graph-classification mode:
//   num_gc_layers = 2 .. 7 (explainer_main.py:57-66, explain.py:64: n_hops = num_gc_layers; models.py:193-220,230-267) and
//   --bn (models.py:222-228: a FRESH BatchNorm1d(n) in train mode on the (1, n, h) activations = per-node standardisation over
//   the feature axis, eps 1e-5, biased variance, applied after the ReLU of every hidden layer; the readout concatenates the
//   standardised activations, models.py:241-260), hidden / output widths up to 256 (the tuned kernels stop at 32), d <= 128, and
//   the optimisers of utils/train_utils.py:7-23 (Adam, SGD momentum 0.95, RMSprop, Adagrad; step / cos schedulers).
// Node mode computes exactly what oracle/kernel_spec.py specifies (parameters on the directed edges, layer l only on the rows within
// L - l hops of the explained node, inner / outer pair split) and reads out row 0 (the explained node in level order).
// Graph mode replaces Explainer.explain(node_idx=0, graph_idx=g, graph_mode=True) (explain.py:80-85,137-146,209-211; loss :740-808
// with lap_loss = 0) on a GcnEncoderGraph (models.py:269-316), as explain_graph.cu generalised to L layers:
//   * no receptive-field pruning: every row with at least one edge is computed at every layer; rows WITHOUT an edge (padding,
//     isolated nodes) all hold one per-layer constant, bn(relu(normalize(b_l))) / normalize(b_L), independent of the masks -- it joins
//     every max-pool and never carries gradient to M or F;
//   * readout = per-layer column max over the padded rows (the constant first, then the rows in ascending order; the first maximum
//     takes the gradient), concatenation, Linear, softmax, -log p[graph label];
//   * every edge gets SDDMM terms from all L layers; the 1/n^2 of the entropy term and the std of M0 use the PADDED size.
// These options are rare, so the kernel is written for clarity, not speed: one persistent CTA per task, state in a per-CTA global slab
// (GxVarLayout, L2 resident for the reference's graph sizes), one warp per row with lane = feature, one thread per undirected edge in
// the edge phase.  Phases per epoch (one __syncthreads each): F1 .. FL | (graph mode: pool) | S | BL .. B1 | P.  The default model
// (3 layers, no bn) with Adam never comes here.
// Attention models (kAtt, --method att, models.py:62-68) weight every layer's masked adjacency by s_ij = P_i . P_j, P = H_{l-1} Wa_l
// (unnormalised, no softmax; every layer starts from the masked adjacency).  Per layer the forward adds a projection and an edge
// phase before the gather (Fl = Pl | Sl | gather with a s); the backward adds, after the row phase, t_ij = dL/dZ_i . H_{l-1}[j] per
// slot, the pair weights a_ij (t_ij + t_ji), and dL/dP = sum_j a_ij (t_ij + t_ji) P_j, whose dL/dP Wa^T joins dL/dH_{l-1} (layer 1:
// dL/dsF).  The edge phase then uses dL/da_ij + dL/da_ji = sum_l s_ij (t_ij + t_ji) from the stored s and t.
// Wide inputs (kWide, 128 < d <= 4096) contract layer 1 in the other order, A_m (X (sF (.) W1)) (DESIGN section 13), so that every per-edge
// step is hid-wide and the d-wide work is two products per epoch on the tensor cores:
//   F0  P = X B with B = sF (.) W1 formed on the fly (3xTF32 mma.sync), every row of the task;
//   F1  y_i = b1 + sum_j a_ij P_j, then the usual row epilogue;
//   B1  dY1 of layer 1's rows, then dP_j = sum_i a_ij dY1_i over every row j (the leading columns of j that are layer-1 rows);
//   B0  G = X^T dP (3xTF32), dL/dsF_f = sum_c W1_fc G_fc;
//   P   layer 1's pair term <dY1_i, P_j> + <dY1_j, P_i> replaces the d-wide dots.
// The feature-mask state and the products live in the task slab and W1 is read through L2, so shared memory does not grow with d.
// Hidden / output widths of 129 .. 256 (kBlk, KW = 8, no attention; DESIGN section 15) take each layer's product over the row block
// instead of row by row, so that a 256 x 256 weight read through L2 is not re-read per row:
//   Fl  gather Z = A_m H_{l-1} (layer 1: U = A_m X) of the layer's rows, then Y = b + Z W_l (rows_product, FP32) into Yh(l), then the
//       row epilogue (normalise, ReLU, bn) in place; Z lives in dZ(l), which the backward overwrites;
//   Bl  the row backward writes dY over the row's Yh(l), then dZ_l = dY W_l^T over the block (layer 1: into dZ1, then dL/dsF's partials
//       and dZ1 (.) sF row by row, as var_first_layer_dz).
// The slab and shared-memory carve-ups are the narrow ones with 256-float rows.
#include "explain_var_common.cuh"
#include "mma_tf32.cuh"

namespace {

struct VarArgs {
  const int32_t* order;
  int32_t ntasks;
  int32_t* counter;
  float* gws;
  int64_t gws_stride_words;
  float* pws;
  int64_t pws_stride_words;
  GxGraphDev g;          // node mode
  GxGraphBatchDev gb;    // graph mode
  GxModelDev m;
  GxHparamsDev hp;
  GxPlanArrays plan;
  const float* m0;
  float* out_mask;
  float* out_feat;
  GxHeadDev hd;          // MLP prediction head (k = 0: none)
};

// ---------------------------------------------------------------------------------------------------------------- attention layers
// Forward of one attention layer (every thread calls; ends with __syncthreads).  P = H_{l-1} Wa (row stride ldp) on the layer's
// nin input rows, H_0 = X (.) sF from the feature rows on layer 1 (Hp == nullptr), else Hp (row stride vw); then s_ij = P_i . P_j and
// a_ij s_ij on the slots of the rows < min(nin, nsrows) (the rows with stored slots) whose column is an input row.  s_ij and s_ji
// are the same products summed in the same order, so they are equal.
__device__ __forceinline__ void att_forward_edges(int win, int ldp, int nin, int nsrows, int d, const float* feat, const int32_t* __restrict__ lo2gid,
                                                  const float* sF, const float* Hp, int vw, const float* Wa, const int32_t* __restrict__ irp,
                                                  const int32_t* __restrict__ icol, const float* a, float* P, float* s, float* as, float* zs,
                                                  int warp, int nwarps, int lane) {
  for (int i = warp; i < nin; i += nwarps) {
    if (Hp == nullptr) {
      const float* const x = feat + (int64_t)lo2gid[i] * d;
      for (int f = lane; f < d; f += 32) zs[f] = __ldg(x + f) * sF[f];   // x * sigmoid(feat_mask) (explain.py:707)
    } else {
      for (int f = lane; f < win; f += 32) zs[f] = Hp[(int64_t)i * vw + f];
    }
    __syncwarp();
    for (int c = lane; c < win; c += 32) {
      float p = 0.f;
      for (int f = 0; f < win; ++f) p = fmaf(zs[f], Wa[f * win + c], p);
      P[(int64_t)i * ldp + c] = p;
    }
    __syncwarp();
  }
  __syncthreads();
  const int srows = nin < nsrows ? nin : nsrows;
  for (int i = warp; i < srows; i += nwarps) {
    const float* const Pi = P + (int64_t)i * ldp;
    for (int e = irp[i] + lane; e < irp[i + 1]; e += 32) {
      const int j = icol[e];
      if (j >= nin) continue;
      const float* const Pj = P + (int64_t)j * ldp;
      float sv = 0.f;
      for (int f = 0; f < win; ++f) sv = fmaf(Pi[f], Pj[f], sv);
      s[e] = sv;
      as[e] = a[e] * sv;
    }
  }
  __syncthreads();
}

// Backward of one attention layer after its row phase (every thread calls; ends with __syncthreads).  D = dL/dZ of the layer's nrow
// rows: dZ1 = dL/dZ (.) sF (row stride dp) dotted with the raw feature rows on layer 1 (Hp == nullptr), else dZ_l dotted with
// Hp = H_{l-1} (row stride vw).
//   t_ij = D_i . H_{l-1}[j] on every slot of the layer's rows;
//   cw_ij = cw_ji = a_ij (t_ij + t_ji) per pair (t only where the row is a row of the layer);
//   dL/dP_i = sum_j cw_ij P_j on the nin input rows (a row beyond the layer's rows has only its leading columns inside them);
//   dL/dP_i Wa^T -> dHa (the layer below adds it to dL/dH) or, on layer 1, dL/dsF += X (.) dL/dP Wa^T into this warp's partials gFw.
__device__ __forceinline__ void att_backward_edges(int win, int ldp, int nrow, int nin, int nsrows, int np, int d, const float* feat,
                                                   const int32_t* __restrict__ lo2gid, const float* D, const float* Hp, int vw, const float* Wa,
                                                   const int32_t* __restrict__ irp, const int32_t* __restrict__ icol, const float* a,
                                                   const int32_t* __restrict__ pi, const int32_t* __restrict__ pj, const int32_t* __restrict__ ppij,
                                                   const int32_t* __restrict__ ppji, const float* P, float* t, float* cw, float* dHa, float* gFw,
                                                   float* zs, int tid, int nt, int warp, int nwarps, int lane) {
  const int dp = gx_round_up(d, 4);
  for (int i = warp; i < nrow; i += nwarps) {
    const float* const Di = D + (int64_t)i * (Hp == nullptr ? dp : vw);
    for (int e = irp[i] + lane; e < irp[i + 1]; e += 32) {
      const int j = icol[e];
      float tv = 0.f;
      if (Hp == nullptr) {
        const float* const x = feat + (int64_t)lo2gid[j] * d;
        for (int f = 0; f < d; ++f) tv = fmaf(Di[f], __ldg(x + f), tv);
      } else {
        const float* const h = Hp + (int64_t)j * vw;
        for (int f = 0; f < win; ++f) tv = fmaf(Di[f], h[f], tv);
      }
      t[e] = tv;
    }
  }
  __syncthreads();
  for (int p = tid; p < np; p += nt) {
    const int i = pi[p], j = pj[p];
    const float tij = i < nrow ? t[ppij[p]] : 0.f, tji = j < nrow ? t[ppji[p]] : 0.f;
    const float c = (i < nsrows ? a[ppij[p]] : a[ppji[p]]) * (tij + tji);
    cw[ppij[p]] = c;
    cw[ppji[p]] = c;
  }
  __syncthreads();
  for (int i = warp; i < nin; i += nwarps) {
    const int r0 = irp[i], r1 = irp[i + 1];
    for (int c0 = 0; c0 < win; c0 += 32) {
      const int c = c0 + lane;
      float v = 0.f;
      if (c < win)
        for (int e = r0; e < r1; ++e) {
          const int j = icol[e];
          if (i >= nrow && j >= nrow) break;   // columns are partitioned by level
          v = fmaf(cw[e], P[(int64_t)j * ldp + c], v);
        }
      if (c < win) zs[c] = v;
    }
    __syncwarp();
    // [dL/dP_i Wa^T]_f = sum_c dL/dP_i[c] Wa[f][c]: lanes over c (consecutive words of Wa's row f), one warp sum per f; lane f % 32
    // owns entry f, as in the row phase
    const float* const x = Hp == nullptr ? feat + (int64_t)lo2gid[i] * d : nullptr;
    for (int f = 0; f < win; ++f) {
      float q = 0.f;
      for (int c = lane; c < win; c += 32) q = fmaf(zs[c], Wa[f * win + c], q);
      q = warp_sum(q);
      if (lane == (f & 31)) {
        if (Hp == nullptr) gFw[f] = fmaf(q, __ldg(x + f), gFw[f]);
        else dHa[(int64_t)i * vw + f] = q;
      }
    }
    __syncwarp();
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------------------------- wide inputs
// C = A B (M x N, row stride ldc) on the tensor cores, 3xTF32 (mma_tf32.cuh): one 16 x 8 tile per warp at a time, the k steps of a tile
// in ascending order, so the product is deterministic.  a(r, k) and b(k, c) return the operands and 0 outside the matrices.
template <typename FA, typename FB>
__device__ __forceinline__ void wide_mma(int M, int N, int K, FA a, FB b, float* C, int ldc, int warp, int nwarps, int lane) {
  const int g = lane >> 2, t = lane & 3;
  const int tn = (N + 7) / 8, tiles = (M + 15) / 16 * tn;
  for (int tile = warp; tile < tiles; tile += nwarps) {
    const int m0 = tile / tn * 16, n0 = tile % tn * 8;
    float c[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k0 = 0; k0 < K; k0 += 8) {
      uint32_t ah[4], al[4], bh0, bl0, bh1, bl1;
      tf32_split(a(m0 + g, k0 + t), ah[0], al[0]);
      tf32_split(a(m0 + g + 8, k0 + t), ah[1], al[1]);
      tf32_split(a(m0 + g, k0 + t + 4), ah[2], al[2]);
      tf32_split(a(m0 + g + 8, k0 + t + 4), ah[3], al[3]);
      tf32_split(b(k0 + t, n0 + g), bh0, bl0);
      tf32_split(b(k0 + t + 4, n0 + g), bh1, bl1);
      mma_tf32(c, al, bh0, bh1);   // the small terms first
      mma_tf32(c, ah, bl0, bl1);
      mma_tf32(c, ah, bh0, bh1);
    }
    const int r = m0 + g, col = n0 + 2 * t;
    if (r < M && col < N) C[(int64_t)r * ldc + col] = c[0];
    if (r < M && col + 1 < N) C[(int64_t)r * ldc + col + 1] = c[1];
    if (r + 8 < M && col < N) C[(int64_t)(r + 8) * ldc + col] = c[2];
    if (r + 8 < M && col + 1 < N) C[(int64_t)(r + 8) * ldc + col + 1] = c[3];
  }
}

// ------------------------------------------------------------------------------------------------------------ hidden widths 129 .. 256
// C = bias + A B (M x N, row stride ldc; bias == nullptr: 0) in FP32 on the CUDA cores: a warp takes 8 rows x 32 columns at a time
// (lane = column, one accumulator per row), k in ascending order.  Each output is the chain fmaf(a(r, k), b(k, c), .) from the bias that
// var_dense / var_hidden_dz / var_first_layer_dz compute for a single row, so the row-block path does the narrow path's arithmetic, and a
// B row is read once per 8 rows.  a(r, k) and b(k, c) return the operands and 0 outside the matrices.
template <typename FA, typename FB>
__device__ __forceinline__ void rows_product(int M, int N, int K, FA a, FB b, const float* bias, float* C, int ldc, int warp, int nwarps, int lane) {
  constexpr int RB = 8;
  const int tn = (N + 31) / 32, tiles = (M + RB - 1) / RB * tn;
  for (int tile = warp; tile < tiles; tile += nwarps) {
    const int r0 = tile / tn * RB, c = tile % tn * 32 + lane;
    float acc[RB];
#pragma unroll
    for (int r = 0; r < RB; ++r) acc[r] = bias != nullptr && c < N ? bias[c] : 0.f;
    for (int k = 0; k < K; ++k) {
      const float bk = b(k, c);
#pragma unroll
      for (int r = 0; r < RB; ++r) acc[r] = fmaf(a(r0 + r, k), bk, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < RB; ++r)
      if (r0 + r < M && c < N) C[(int64_t)(r0 + r) * ldc + c] = acc[r];
  }
}

// The minimum-blocks bound 0 is the compiler's default: node mode is capped at 128 registers (some instantiations spill); graph mode
// lets the small default-width model fit two CTAs per SM.
template <bool kGraph, bool kBn, int KW, bool kAtt, bool kWide, bool kBlk = false>
__global__ void __launch_bounds__(kVarThreads, kGraph ? (KW == 1 && !kBn ? 2 : 1) : 0) explain_var_kernel(const VarArgs A) {
  static_assert(!kBlk || (KW == 8 && !kAtt), "the row-block path is built for widths 129 .. 256 without attention");
  extern __shared__ __align__(16) float sm[];
  __shared__ int s_task;
  constexpr int NT = kVarThreads, nwarps = NT / 32;
  constexpr int VW = 32 * KW;   // row stride of every hidden-width array
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const GxModelDev& m = A.m;
  const GxHparamsDev& hp = A.hp;
  const int d = m.d, C = m.C, L = m.L, hid = m.hid, embw = m.emb;
  const int dp = gx_round_up(d, 4);
  const int PD = hid * (L - 1) + embw;
  const bool ieee = (hp.flags & GX_HP_IEEE_EDGE) != 0;
  const GxHeadDev& hd = A.hd;
  const VarSmem S = var_smem_of<kWide>(d, L, hid, embw, C, nwarps, kAtt ? 1 : 0, hd);
  float* const sF = sm + S.sF; float* const Fm = sm + S.F; float* const mF = sm + S.mF; float* const vF = sm + S.vF;
  float* const zs = sm + S.zs + warp * S.zlen;
  float* const gFp = sm + S.gFp;
  float* const emb = sm + S.emb; float* const dEmb = sm + S.dEmb; float* const logit = sm + S.logit;
  float* const cst = sm + S.total;                                              // graph mode (gx_var_smem_bytes)
  int* const arg = reinterpret_cast<int*>(sm + S.total + gx_round_up(PD, 4));   // graph mode
  const bool wp_smem = gx_head_words(hd, PD, C) <= GX_WP_SMEM_MAX;
  const float* const Wpp = wp_smem ? sm + S.Wp : m.Wp;
  const float* const bpp = wp_smem ? sm + S.Wp + C * PD : m.bp;
  auto win_of = [&](int l) { return l == 0 ? d : hid; };            // l = 0 .. L-1
  auto wout_of = [&](int l) { return l == L - 1 ? embw : hid; };

  const float* Wl[GX_MAX_LAYERS];   // conv weights: shared memory when they fit, else global (L2 resident)
  var_stage_model<kWide>(m, hd, S, sm, Wl, tid, NT);
  const float* Wal[kAtt ? GX_MAX_LAYERS : 1];  // attention weights (kAtt), staged like Wl
  if constexpr (kAtt) var_stage_att(m, S, sm, Wal, tid, NT);
  if constexpr (kGraph) {
    __syncthreads();
    // embedding of a row without edges: Y = 0 W + b, the same activation as any row; depends on the model only
    if (warp == 0) {
      for (int l = 1; l <= L; ++l) {
        const int wout = wout_of(l - 1);
        float y[KW], yh[KW], h[KW], is;
        var_dense<KW>(zs, 0, Wl[l - 1], wout, sm + S.b[l - 1], y, lane);
        var_activate<kBn, KW>(y, wout, l < L, yh, h, &is, lane);
#pragma unroll
        for (int k = 0; k < KW; ++k)
          if (lane + 32 * k < wout) cst[hid * (l - 1) + lane + 32 * k] = h[k];
      }
    }
  }
  float* const slab = A.gws + (int64_t)blockIdx.x * A.gws_stride_words;
  float2* const MM = reinterpret_cast<float2*>(A.pws + (int64_t)blockIdx.x * A.pws_stride_words);

  for (;;) {
    int task_id;
    if (!var_next_task(A, s_task, tid, task_id)) break;
    const GxTask* __restrict__ Tp = A.plan.tasks + task_id;
    // graph mode: n = the rows with an edge, n2 = n, e1 = e_d, npairs_in = npairs (gx_plan_graphs)
    const int n = Tp->n, n2 = kGraph ? n : Tp->n2, e1 = Tp->e1, np = Tp->npairs_in;
    const int gt = Tp->gt_label;
    const int64_t node_off = Tp->node_off, rp_off = Tp->rp_off, edge_off = Tp->edge_off, pair_off = Tp->pair_off;
    int R[GX_MAX_LAYERS + 1];   // node mode: R[l] = rows of layer l (1-based): nodes within L - l hops; R[0] = n
    if constexpr (!kGraph) {
      R[0] = n;
      for (int l = 1; l <= L; ++l) R[l] = Tp->cum[L - l] < n ? Tp->cum[L - l] : n;
    }
    auto rows = [&](int l) { if constexpr (kGraph) return n; else return R[l]; };
    auto rin = [&](int l) { if constexpr (kGraph) return n; else return R[l - 1]; };   // input rows of layer l
    const GxVarLayout Lo = gx_make_var_layout(n, n2, e1, kGraph ? 0 : np, d, L, VW, kAtt ? 1 : 0, Tp->e_d, kWide ? 1 : 0);
    // layer 1's input rows: the graph's features (node mode), this graph's padded rows (graph mode); both indexed by lo2gid
    const float* const feat = kGraph ? A.gb.feat + (int64_t)Tp->node * A.gb.max_nodes * d : A.g.feat;
    const int32_t* __restrict__ lo2gid = A.plan.lo2gid + node_off;
    const int32_t* __restrict__ irp = A.plan.irowptr + rp_off;
    const int32_t* __restrict__ icol = A.plan.icol + edge_off;
    const int32_t* __restrict__ pi = A.plan.pair_i + pair_off; const int32_t* __restrict__ pj = A.plan.pair_j + pair_off;
    const int32_t* __restrict__ ppij = A.plan.pair_pij + pair_off; const int32_t* __restrict__ ppji = A.plan.pair_pji + pair_off;
    const int32_t* __restrict__ poij = A.plan.pair_oij + pair_off; const int32_t* __restrict__ poji = A.plan.pair_oji + pair_off;
    float* const a = slab + Lo.a; float* const U = slab + Lo.U; float* const dZ1 = slab + Lo.dZ1; float* const lapg = slab + Lo.lapg;
    auto Yh = [&](int l) { return slab + Lo.Yh + (int64_t)(l - 1) * n2 * VW; };     // l = 1..L: normalised pre-activation
    auto Hh = [&](int l) { return slab + Lo.H + (int64_t)(l - 1) * n2 * VW; };      // l = 1..L: what the next layer / the readout sees
    auto dZ = [&](int l) { return slab + Lo.dZ + (int64_t)(l - 2) * n2 * VW; };     // l = 2..L: dL/d(A_m H_{l-1}) (width hid)
    auto qn = [&](int l) { return slab + Lo.q + (int64_t)(l - 1) * n2; };
    auto istd = [&](int l) { return slab + Lo.istd + (int64_t)(l - 1) * n2; };
    // attention (kAtt): P of layer l (row stride dp on layer 1, VW above), per-slot s, a s and t of layer l
    auto Pl = [&](int l) { return slab + Lo.P + (l == 1 ? 0 : (int64_t)n * dp + (int64_t)(l - 2) * n2 * VW); };
    auto sl = [&](int l) { return slab + Lo.s + (int64_t)(l - 1) * e1; };
    auto asl = [&](int l) { return slab + Lo.as + (int64_t)(l - 1) * e1; };
    auto tl = [&](int l) { return slab + Lo.t + (int64_t)(l - 1) * e1; };
    float* const cw = slab + Lo.cw; float* const dHa = slab + Lo.dHa;
    float2* const mm = MM + np; float2* const vv = mm + np; float2* const SS = vv + np;
    // the feature-mask state: shared memory, or the slab for wide inputs (kWide), which also holds P = X B, dY1, dP = A_m^T dY1,
    // G = X^T dP and dL/dsF
    float* const fsF = kWide ? slab + Lo.fm : sF; float* const fF = kWide ? slab + Lo.fm + dp : Fm;
    float* const fmF = kWide ? slab + Lo.fm + 2 * dp : mF; float* const fvF = kWide ? slab + Lo.fm + 3 * dp : vF;
    float* const gFw = slab + Lo.fm + 4 * dp;
    float* const XB = slab + Lo.XB; float* const dY1 = slab + Lo.dY1; float* const dP = slab + Lo.dP; float* const Gw = slab + Lo.G;
    const float* const W1 = m.W[0];
    auto xat = [=](int r, int f) { return r < n && f < d ? __ldg(feat + (int64_t)lo2gid[r] * d + f) : 0.f; };   // X of the task, level order
    const float nn = (float)Tp->n_norm * (float)Tp->n_norm;
    const float ent_over_nn = hp.c_ent / nn;
    const float lap_over_nn = hp.c_lap / nn;

    for (int f = tid; f < dp; f += NT) {
      fsF[f] = 0.5f; fF[f] = 0.f; fmF[f] = 0.f; fvF[f] = 0.f;   // feat_mask = 0 (explain.py:633-643)
      if (hp.out_iter == 0 && f < d && A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = 0.5f;
    }
    {
      const float m0_std = sqrtf(2.0f / (float)Tp->n_norm);  // gain('relu') * sqrt(2/(n+n)) (explain.py:647-651), n = the padded size in graph mode
      for (int p = tid; p < np; p += NT) {
        const int oij = poij[p], oji = poji[p];
        const float Mi = var_init_param(hp, A.m0, edge_off + oij, (uint32_t)Tp->node, (uint32_t)oij, m0_std);
        const float Mj = var_init_param(hp, A.m0, edge_off + oji, (uint32_t)Tp->node, (uint32_t)oji, m0_std);
        MM[p] = make_float2(Mi, Mj);
        mm[p] = make_float2(0.f, 0.f);
        vv[p] = make_float2(0.f, 0.f);
        const float Si = sigmoid_f(Mi), Sj = sigmoid_f(Mj);
        SS[p] = make_float2(Si, Sj);
        const float a0 = 0.5f * (Si + Sj);  // explain.py:665-678
        const int i = pi[p], j = pj[p];
        if (kGraph || kWide || i < n2) a[ppij[p]] = a0;
        if (kGraph || kWide || j < n2) a[ppji[p]] = a0;
        if constexpr (!kGraph) {   // no Laplacian term in graph mode (explain.py:787-788)
          const float yd = (float)__ldg(A.g.pred_label + lo2gid[i]) - (float)__ldg(A.g.pred_label + lo2gid[j]);
          lapg[p] = lap_over_nn * yd * yd;   // d/dA_ij + d/dA_ji of y^T (D - A) y / n^2 (explain.py:780-793)
        }
        if (hp.out_iter == 0) { A.out_mask[edge_off + oij] = a0; A.out_mask[edge_off + oji] = a0; }
      }
    }
    __syncthreads();

    for (int it = 1; it <= hp.iters; ++it) {
      // ---------------------------------------------------------------- forward, layer by layer        (models.py:58-80,230-267)
      if constexpr (kWide) {   // F0: P = X (sF (.) W1) on every row of the task
        wide_mma(n, hid, d, xat, [&](int f, int c) { return f < d && c < hid ? fsF[f] * __ldg(W1 + (int64_t)f * hid + c) : 0.f; }, XB, VW,
                 warp, nwarps, lane);
        __syncthreads();
      }
      for (int l = 1; l <= L; ++l) {
        const int win = win_of(l - 1), wout = wout_of(l - 1);
        const float* const Ws = Wl[l - 1]; const float* const bsm = sm + S.b[l - 1];
        const float* ag = a;   // the aggregation weights: a, or a s on attention models
        if constexpr (kAtt) {
          att_forward_edges(win, l == 1 ? dp : VW, rin(l), kGraph ? n : n2, d, feat, lo2gid, sF, l == 1 ? nullptr : Hh(l - 1), VW,
                            Wal[l - 1], irp, icol, a, Pl(l), sl(l), asl(l), zs, warp, nwarps, lane);
          ag = asl(l);
        }
        for (int i = warp; i < rows(l); i += nwarps) {
          const int r0 = irp[i], r1 = irp[i + 1];
          if constexpr (kWide) {
            if (l == 1) {   // F1: y = b1 + sum_j a_ij P_j
              float y[KW];
#pragma unroll
              for (int k = 0; k < KW; ++k) y[k] = lane + 32 * k < wout ? bsm[lane + 32 * k] : 0.f;
              for (int e = r0; e < r1; ++e) {
                const float ae = a[e];
                const float* const Pj = XB + (int64_t)icol[e] * VW;
#pragma unroll
                for (int k = 0; k < KW; ++k)
                  if (lane + 32 * k < wout) y[k] = fmaf(ae, Pj[lane + 32 * k], y[k]);
              }
              var_row_epilogue<kBn, KW>(y, wout, l, L, i, Yh, Hh, VW, qn, istd, lane);
              continue;
            }
          }
          if constexpr (kBlk) {   // the aggregate only (layer 1: U; above: Z into dZ(l), free until the backward)
            if (l == 1) var_gather_feat(r0, r1, icol, a, feat, lo2gid, d, sF, U + (int64_t)i * dp, zs, lane);
            else var_gather_hidden<KW>(r0, r1, icol, a, Hh(l - 1), win, dZ(l) + (int64_t)i * VW, lane);
            continue;
          }
          if (l == 1) var_gather_feat(r0, r1, icol, ag, feat, lo2gid, d, sF, U + (int64_t)i * dp, zs, lane);
          else var_gather_hidden<KW>(r0, r1, icol, ag, Hh(l - 1), win, zs, lane);
          var_row_forward<kBn, KW>(zs, win, Ws, wout, bsm, l, L, i, Yh, Hh, VW, qn, istd, lane);
        }
        __syncthreads();
        if constexpr (kBlk) {
          if (!kWide || l > 1) {   // Y = b + Z W over the layer's rows into Yh(l), then the row epilogue in place
            const int nr = rows(l);
            float* const Zl = l == 1 ? U : dZ(l);
            const int ldz = l == 1 ? dp : VW;
            rows_product(nr, wout, win, [&](int r, int k) { return r < nr ? (l == 1 ? Zl[(int64_t)r * ldz + k] * sF[k] : Zl[(int64_t)r * ldz + k]) : 0.f; },
                         [&](int k, int c) { return c < wout ? Ws[k * wout + c] : 0.f; }, bsm, Yh(l), VW, warp, nwarps, lane);
            __syncthreads();
            for (int i = warp; i < nr; i += nwarps) {
              float y[KW];
#pragma unroll
              for (int k = 0; k < KW; ++k) {
                const int c = lane + 32 * k;
                y[k] = c < wout ? Yh(l)[(int64_t)i * VW + c] : 0.f;
              }
              var_row_epilogue<kBn, KW>(y, wout, l, L, i, Yh, Hh, VW, qn, istd, lane);
            }
            __syncthreads();
          }
        }
      }
      // ---------------------------------------------------------------- S: readout, softmax, dEmb   (models.py:305-314, explain.py:711)
      if constexpr (kGraph) {   // max-pool of every layer, the edge-less rows' constant first
        var_max_pool(L, hid, PD, n, Hh, VW, (Tp->flags & 1) != 0 ? cst : nullptr, -1, emb, arg, tid, NT);
        __syncthreads();
      }
      if constexpr (!kGraph) {   // node mode reads out row r = level-order id 0
        if (warp == 0)
          for (int l = 1; l <= L; ++l)
            for (int c = lane; c < wout_of(l - 1); c += 32) emb[hid * (l - 1) + c] = Hh(l)[c];
        __syncthreads();
      }
      var_readout_tail(emb, hd, wp_smem ? sm + S.Wp : hd.W, Wpp, bpp, C, PD, gt, sm + S.hx, sm + S.hg, logit, dEmb, tid, NT);
      if constexpr (!kWide)
        for (int idx = tid; idx < nwarps * dp; idx += NT) gFp[idx] = 0.f;
      __syncthreads();
      // ---------------------------------------------------------------- backward, layer by layer
      for (int l = L; l >= 1; --l) {
        const int win = win_of(l - 1), wout = wout_of(l - 1);
        const float* const Ws = Wl[l - 1];
        const int koff = hid * (l - 1);
        for (int i = warp; i < rows(l); i += nwarps) {
          // dL/dH_l[i] = (A_m^T dZ_{l+1})[i] over the neighbours that are rows of layer l+1 (a prefix of row i) + the readout's share
          float g[KW], yh[KW];
#pragma unroll
          for (int k = 0; k < KW; ++k) g[k] = 0.f;
          if (l < L) var_gather_back<KW>(irp[i], irp[i + 1], icol, kAtt ? asl(l + 1) : a, dZ(l + 1), wout, rows(l + 1), g, lane);   // columns are partitioned by level
          if constexpr (kAtt) {   // + the attention's share, dL/dP_{l+1} Wa_{l+1}^T
#pragma unroll
            for (int k = 0; k < KW; ++k)
              if (l < L && lane + 32 * k < wout) g[k] += dHa[(int64_t)i * VW + lane + 32 * k];
          }
#pragma unroll
          for (int k = 0; k < KW; ++k) {
            const int c = lane + 32 * k;
            if (c < wout && (kGraph ? arg[koff + c] == i : i == 0)) g[k] += dEmb[koff + c];
            yh[k] = Yh(l)[(int64_t)i * VW + c];
          }
          if constexpr (kBlk) {   // dY straight into the slab: over the row's Yh (read above, not read again; the product runs over the
                                  // row block below), or into dY1 on the wide input path's layer 1
            var_row_backward<kBn, KW>(g, yh, l, L, i, Hh, VW, qn, istd, wout, (kWide && l == 1 ? dY1 : Yh(l)) + (int64_t)i * VW, lane);
            continue;
          }
          var_row_backward<kBn, KW>(g, yh, l, L, i, Hh, VW, qn, istd, wout, zs, lane);
          if constexpr (kWide) {
            if (l == 1) {   // B1: keep dY1
#pragma unroll
              for (int k = 0; k < KW; ++k) dY1[(int64_t)i * VW + lane + 32 * k] = lane + 32 * k < wout ? zs[lane + 32 * k] : 0.f;
              __syncwarp();
              continue;
            }
          }
          // dZ[f] = sum_c dY[c] W[f][c]
          if (l == 1) var_first_layer_dz(zs, Ws, d, wout, U + (int64_t)i * dp, sF, gFp + warp * dp, dZ1 + (int64_t)i * dp, lane);
          else var_hidden_dz<KW>(zs, Ws, win, wout, dZ(l) + (int64_t)i * VW, lane);
          __syncwarp();
        }
        __syncthreads();
        if constexpr (kBlk) {
          if (!kWide || l > 1) {   // dZ = dY W^T over the layer's rows (layer 1: into dZ1, then dL/dsF's partials and the mask)
            const int nr = rows(l);
            const float* const dYl = Yh(l);
            rows_product(nr, win, wout, [&](int r, int c) { return r < nr ? dYl[(int64_t)r * VW + c] : 0.f; },
                         [&](int c, int f) { return f < win ? Ws[f * wout + c] : 0.f; }, nullptr, l == 1 ? dZ1 : dZ(l), l == 1 ? dp : VW,
                         warp, nwarps, lane);
            __syncthreads();
            if (l == 1) {   // as var_first_layer_dz: each warp's rows in ascending order into its own partials
              for (int i = warp; i < nr; i += nwarps)
                for (int f = lane; f < d; f += 32) {
                  const float t = dZ1[(int64_t)i * dp + f];
                  gFp[warp * dp + f] = fmaf(t, U[(int64_t)i * dp + f], gFp[warp * dp + f]);
                  dZ1[(int64_t)i * dp + f] = t * sF[f];
                }
              __syncthreads();
            }
          }
        }
        if constexpr (kWide) {
          if (l == 1) {
            // B1: dP_j = sum_i a_ij dY1_i over j's leading columns that are layer-1 rows (A_m symmetric), every row j of the task
            for (int j = warp; j < n; j += nwarps) {
              float g[KW];
#pragma unroll
              for (int k = 0; k < KW; ++k) g[k] = 0.f;
              var_gather_back<KW>(irp[j], irp[j + 1], icol, a, dY1, wout, rows(1), g, lane);
#pragma unroll
              for (int k = 0; k < KW; ++k) dP[(int64_t)j * VW + lane + 32 * k] = g[k];
            }
            __syncthreads();
            // B0: G = X^T dP, then dL/dsF_f = sum_c W1_fc G_fc
            wide_mma(d, hid, n, [&](int f, int r) { return xat(r, f); }, [&](int r, int c) { return r < n && c < hid ? dP[(int64_t)r * VW + c] : 0.f; },
                     Gw, VW, warp, nwarps, lane);
            __syncthreads();
            for (int f = warp; f < d; f += nwarps) {
              float t = 0.f;
              for (int c = lane; c < hid; c += 32) t = fmaf(__ldg(W1 + (int64_t)f * hid + c), Gw[(int64_t)f * VW + c], t);
              t = warp_sum(t);
              if (lane == 0) gFw[f] = t;
            }
            __syncthreads();
          }
        }
        if constexpr (kAtt)
          att_backward_edges(win, l == 1 ? dp : VW, rows(l), rin(l), kGraph ? n : n2, np, d, feat, lo2gid, l == 1 ? dZ1 : dZ(l),
                             l == 1 ? nullptr : Hh(l - 1), VW, Wal[l - 1], irp, icol, a, pi, pj, ppij, ppji, Pl(l), tl(l), cw, dHa,
                             gFp + warp * dp, zs, tid, NT, warp, nwarps, lane);
      }
      // ---------------------------------------------------------------- P: edge gradients, regularisers, optimiser step, next mask
      {
        const float2 tab = __ldg(hp.adam_tab + (it - 1));
        const float step = tab.x, bc2s = tab.y, bc2s_inv = 1.0f / tab.y;
        const bool last = (it == hp.out_iter);   // the mask built after this update is the one the reference returns
        for (int f = tid; f < d; f += NT) {
          float gsum = 0.f;
          if constexpr (kWide) gsum = gFw[f];
          else
            for (int w = 0; w < nwarps; ++w) gsum += gFp[w * dp + f];
          const float s = fsF[f];
          const float g = s * (1.f - s) * (gsum + hp.c_feat_size / (float)d);
          float mf = fmF[f], vf = fvF[f], Fv = fF[f];
          var_feat_update(hp, g, Fv, mf, vf, step, bc2s);
          fmF[f] = mf; fvF[f] = vf; fF[f] = Fv;
          const float sn = sigmoid_f(Fv);
          fsF[f] = sn;   // (the edge dots below use dZ1 (.) sF stored in the backward, not this value)
          if (last && A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = sn;
        }
        for (int p = tid; p < np; p += NT) {
          const int i = pi[p], j = pj[p];   // i < j in level order
          // dL/dA_ij + dL/dA_ji = sum over the layers of <dL/d(A_m H_{l-1})[i], H_{l-1}[j]> + <.. [j], .. [i]> (layer 1: feature rows)
          float Gd;
          if constexpr (kAtt) {   // sum over the layers of s_ij (t_ij + t_ji), t of the rows of the layer only
            Gd = kGraph ? 0.f : lapg[p];
            for (int l = 1; l <= L; ++l) {
              const bool ri = kGraph || i < R[l], rj = kGraph || j < R[l];
              if (!ri && !rj) continue;
              const float tij = ri ? tl(l)[ppij[p]] : 0.f, tji = rj ? tl(l)[ppji[p]] : 0.f;
              Gd = fmaf(sl(l)[ppij[p]], tij + tji, Gd);
            }
          } else if constexpr (kGraph && !kWide) {   // no Laplacian term; every row at every layer, both directions of a layer in one sum
            Gd = 0.f;
            {
              const float* xi = feat + (int64_t)lo2gid[i] * d; const float* xj = feat + (int64_t)lo2gid[j] * d;
              float t = 0.f;
              for (int f = 0; f < d; ++f) t = fmaf(dZ1[(int64_t)i * dp + f], __ldg(xj + f), t);
              for (int f = 0; f < d; ++f) t = fmaf(dZ1[(int64_t)j * dp + f], __ldg(xi + f), t);
              Gd += t;
            }
            for (int l = 2; l <= L; ++l) {
              const float* const dZl = dZ(l); const float* const Hp = Hh(l - 1);
              float t = 0.f;
              for (int f = 0; f < hid; ++f) t = fmaf(dZl[(int64_t)i * VW + f], Hp[(int64_t)j * VW + f], t);
              for (int f = 0; f < hid; ++f) t = fmaf(dZl[(int64_t)j * VW + f], Hp[(int64_t)i * VW + f], t);
              Gd += t;
            }
          } else if constexpr (!kWide) {   // only the rows of layer l, the two directions added one by one
            Gd = lapg[p];
            if (i < R[1]) {
              float t = 0.f;
              const float* xr = feat + (int64_t)lo2gid[j] * d;
              for (int f = 0; f < d; ++f) t = fmaf(dZ1[(int64_t)i * dp + f], __ldg(xr + f), t);
              Gd += t;
            }
            if (j < R[1]) {
              float t = 0.f;
              const float* xr = feat + (int64_t)lo2gid[i] * d;
              for (int f = 0; f < d; ++f) t = fmaf(dZ1[(int64_t)j * dp + f], __ldg(xr + f), t);
              Gd += t;
            }
            for (int l = 2; l <= L; ++l) {
              const float* const dZl = dZ(l); const float* const Hp = Hh(l - 1);
              if (i < R[l]) { float t = 0.f; for (int f = 0; f < hid; ++f) t = fmaf(dZl[(int64_t)i * VW + f], Hp[(int64_t)j * VW + f], t); Gd += t; }
              if (j < R[l]) { float t = 0.f; for (int f = 0; f < hid; ++f) t = fmaf(dZl[(int64_t)j * VW + f], Hp[(int64_t)i * VW + f], t); Gd += t; }
            }
          } else {   // wide inputs: as the two branches above, with layer 1's term <dY1_i, P_j> + <dY1_j, P_i> (hid-wide)
            auto dot = [&](const float* u, const float* v, int w) { float t = 0.f; for (int c = 0; c < w; ++c) t = fmaf(u[c], v[c], t); return t; };
            const float* const Yi = dY1 + (int64_t)i * VW; const float* const Yj = dY1 + (int64_t)j * VW;
            const float* const Pi = XB + (int64_t)i * VW; const float* const Pj = XB + (int64_t)j * VW;
            if constexpr (kGraph) {
              Gd = dot(Yi, Pj, hid) + dot(Yj, Pi, hid);
              for (int l = 2; l <= L; ++l) {
                const float* const dZl = dZ(l); const float* const Hp = Hh(l - 1);
                Gd += dot(dZl + (int64_t)i * VW, Hp + (int64_t)j * VW, hid) + dot(dZl + (int64_t)j * VW, Hp + (int64_t)i * VW, hid);
              }
            } else {
              Gd = lapg[p];
              for (int l = 1; l <= L; ++l) {
                const float* const dZl = l == 1 ? dY1 : dZ(l); const float* const Hp = l == 1 ? XB : Hh(l - 1);
                if (i < R[l]) Gd += dot(dZl + (int64_t)i * VW, Hp + (int64_t)j * VW, hid);
                if (j < R[l]) Gd += dot(dZl + (int64_t)j * VW, Hp + (int64_t)i * VW, hid);
              }
            }
          }
          Gd *= 0.5f;  // sym_mask = (S + S^T)/2 (explain.py:671)
          float2 Mv = MM[p];
          const float2 Sv = SS[p];
          float2 m2 = mm[p], v2 = vv[p];
          const float gi = Sv.x * (1.f - Sv.x) * (Gd + hp.c_size - ent_over_nn * Mv.x);
          const float gj = Sv.y * (1.f - Sv.y) * (Gd + hp.c_size - ent_over_nn * Mv.y);
          var_edge_update(hp, gi, Mv.x, m2.x, v2.x, step, bc2s, bc2s_inv, ieee);
          var_edge_update(hp, gj, Mv.y, m2.y, v2.y, step, bc2s, bc2s_inv, ieee);
          const float2 Sn = make_float2(sigmoid_fast(Mv.x, ieee), sigmoid_fast(Mv.y, ieee));
          MM[p] = Mv; mm[p] = m2; vv[p] = v2; SS[p] = Sn;
          const float an = 0.5f * (Sn.x + Sn.y);
          if (kGraph || kWide || i < n2) a[ppij[p]] = an;
          if (kGraph || kWide || j < n2) a[ppji[p]] = an;
          if (last) { A.out_mask[edge_off + poij[p]] = an; A.out_mask[edge_off + poji[p]] = an; }
        }
      }
      __syncthreads();
    }
  }
}

// calls f(kernel) with the instantiation for the mode and the model
template <typename F>
cudaError_t with_var_kernel(int graph_mode, const GxModelDev& m, F&& f) {
  if (var_row_kw(m.hid, m.emb) == 8) {   // widths 129 .. 256: the row-block path (attention models are refused at these widths)
    if (m.att) return cudaErrorInvalidValue;
    const bool wide = m.d >= GX_VAR_WIDE_MIN;
    auto blk = [&](auto bn) {
      constexpr bool b = decltype(bn)::value;
      if (graph_mode) return wide ? f(explain_var_kernel<true, b, 8, false, true, true>) : f(explain_var_kernel<true, b, 8, false, false, true>);
      return wide ? f(explain_var_kernel<false, b, 8, false, true, true>) : f(explain_var_kernel<false, b, 8, false, false, true>);
    };
    return m.bn ? blk(std::true_type()) : blk(std::false_type());
  }
  return var_dispatch(m, [&](auto bn, auto kw) {
    constexpr bool b = decltype(bn)::value;
    constexpr int w = decltype(kw)::value;
    if (m.att) return graph_mode ? f(explain_var_kernel<true, b, w, true, false>) : f(explain_var_kernel<false, b, w, true, false>);
    if (m.d >= GX_VAR_WIDE_MIN) return graph_mode ? f(explain_var_kernel<true, b, w, false, true>) : f(explain_var_kernel<false, b, w, false, true>);
    return graph_mode ? f(explain_var_kernel<true, b, w, false, false>) : f(explain_var_kernel<false, b, w, false, false>);
  });
}

}  // namespace

// var_smem's carve-up + in graph mode the edge-less rows' constant embedding and the arg-max row of every pooled feature (cst, arg)
int gx_var_smem_bytes(int graph_mode, int d, int L, int hid, int emb, int C, int att, const GxHeadDev& hd) {
  const int pool = graph_mode ? 2 * gx_round_up(hid * (L - 1) + emb, 4) : 0;
  const int words = d >= GX_VAR_WIDE_MIN ? var_smem_wide(d, L, hid, emb, C, kVarThreads / 32, hd).total
                                         : var_smem(d, L, hid, emb, C, kVarThreads / 32, att, hd).total;
  return (words + pool) * 4;
}
int gx_var_row_stride(int hid, int emb) { return 32 * var_row_kw(hid, emb); }

int gx_var_ctas_per_sm(int graph_mode, const GxModelDev& m, const GxHeadDev& hd) {
  const int bytes = gx_var_smem_bytes(graph_mode, m.d, m.L, m.hid, m.emb, m.C, m.att, hd);
  int n = 0;
  with_var_kernel(graph_mode, m, [&](auto kern) { n = var_ctas_per_sm(kern, bytes); return cudaSuccess; });
  return n;
}

cudaError_t gx_launch_explain_var(const GxExplainLaunch& cfg, int graph_mode, const GxGraphDev& g, const GxGraphBatchDev& gb,
                                  const GxModelDev& m, const GxHeadDev& hd, const GxHparamsDev& hp, const GxPlanArrays& plan, const float* m0,
                                  float* out_mask, float* out_feat, cudaStream_t s) {
  VarArgs args;
  fill_queue_args(args, cfg, m, hp, plan, m0, out_mask, out_feat);
  args.g = g; args.gb = gb; args.gws = cfg.gws; args.gws_stride_words = cfg.gws_stride_words; args.hd = hd;
  const int bytes = gx_var_smem_bytes(graph_mode, m.d, m.L, m.hid, m.emb, m.C, m.att, hd);
  return with_var_kernel(graph_mode, m, [&](auto kern) { return var_launch(kern, args, cfg.grid, bytes, s); });
}
