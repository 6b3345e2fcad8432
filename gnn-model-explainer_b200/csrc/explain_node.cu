// explain_node.cu -- K2: the persistent per-node mask-optimisation kernel (node mode), shared-memory resident.
//
// One CTA owns one explained node for ALL epochs: mask build A (.) sym(sigmoid(M)), the reference's
// 3-layer GCN forward ((A_m H) W + b -> row L2-normalise -> ReLU), softmax / -log p[gt], the
// size / entropy / Laplacian / feature-size regularisers, the hand-derived backward to dL/dM and
// dL/dF, and the Adam step, with every array resident in shared memory (tasks that do not fit 227 KB run in
// explain_stream.cu).  Replaces, for the default
// hyper-parameters, explainer/explain.py:137-146 (epoch loop) + :665-715 (ExplainModule.forward)
// + :740-808 (loss) + autograd + torch.optim.Adam, and models.py:58-80,230-267,363-376.
//
// What makes it cheaper than the dense reference (exact, not approximate):
//   * M, m, v live only on the E_d directed edges of the k-hop sub-adjacency: every term of
//     dL/dM_ij is local to (i,j)/(j,i), off-edge entries never reach the returned mask.
//   * Only ONE row of logits carries loss, so layer l is needed only for nodes within L-l hops
//     of the explained node; with nodes relabelled in (distance, degree) order every layer's row
//     set is a prefix [0,n_{L-l}) and the backward touches the same prefixes.
//   * dL/dF needs sum_i dZ1[i] (.) U[i] with U = A_m X kept from the forward, so the layer-1
//     transpose aggregation disappears.
//   * The returned mask is the one built in the forward of the LAST epoch (explain.py:694,209),
//     i.e. after num_epochs-1 updates; the last backward/Adam step is unobservable and skipped.
//
// Work mapping (v3; v1 was issue bound with lane=feature rows, v2's one-thread-per-row dense left most
// warps waiting at barriers):
//   * a warp is cut into groups of GW = max(d,20)/4 lanes; a group owns ONE row from start to finish:
//     it walks the row's edges with float4 shared-memory loads (lane q holds features 4q..4q+3),
//     exchanges the aggregate through a per-warp scratch row, and each lane then produces one float4
//     of the dense product (weights as float4 from shared memory), the row norm being a GW-lane
//     shuffle sum.  Rows are dealt cyclically over the warps in chunks of 32/GW, so every phase keeps
//     all warps busy; rows with more than kLongRow edges are split across a whole warp first.
//   * edge phase: one thread per undirected edge (both directions), sigmoid cached between epochs.
// Phases per epoch (one __syncthreads each): F1 | F2 | S (row r: layer 3 + readout + softmax +
// layer-3 backward, one warp) | B2 | B1 | P.
#include "explain_common.cuh"

namespace {

// Phase S: everything that concerns only the explained node's own row (level-order id 0): layer 3, the concat readout,
// softmax / -log p[gt] and the layer-3 backward (models.py:256-260,375; explain.py:714,750-753).  One warp, a large share of a
// tiny task's epoch: written for a SHORT serial chain -- compile-time trip counts, clamped lane indices instead
// of divergent `if (lane < ..)` blocks, one exp per class, the four 8-lane groups of the warp reduced with shuffles.
// kWpShared only separates the two instantiations so that the pred_model pointer keeps its address space (LDS vs LDG).
// kTrace: tr[0] = -log softmax[gt] (explain.py:750-753), tr[1] = softmax[gt]; trp (optional) receives the softmax row.
template <typename IdxT, int HID, int EMB, bool kWpShared, bool kTrace>
__device__ __forceinline__ void readout_phase(int lane, int C, int gt, const IdxT* irp, const IdxT* icol, const float* a,
                                              const float* Yh1, const float* Yh2, float* zs, const float* bs, const float* W3s,
                                              const float* Wpp, const float* bpp, float* logit, float* dE, float* dZ3,
                                              float* tr, float* trp) {
  constexpr int HS = HID, H4 = HID / 4, PD = 2 * HID + EMB;
  const int g = lane >> 3, q8 = lane & 7;
  // layer-3 aggregate of row 0: the four 8-lane groups walk its edges four apart, then sum across the groups
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  {
    const int r0 = irp[0], r1 = irp[1];
    if (q8 < H4) acc = gather_row<IdxT, true, 4>(r0 + g, r1, 4, icol, a, Yh2, HS, q8);
  }
#pragma unroll
  for (int o = 8; o <= 16; o <<= 1) {
    acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
    acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
  }
  if (lane < H4) st4(zs + 4 * lane, acc);
  __syncwarp();
  // Y3 = Z3 W3 + b3 (lane = output feature), row normalise
  const int le = lane < EMB ? lane : EMB - 1;
  const int lh = lane < HID ? lane : HID - 1;
  float y3 = bs[2 * HID + le];
#pragma unroll
  for (int f4 = 0; f4 < H4; ++f4) {
    const float4 z4 = ld4(zs + 4 * f4);
    const float* w = W3s + (4 * f4) * EMB + le;
    y3 = fmaf(z4.x, w[0], y3); y3 = fmaf(z4.y, w[EMB], y3); y3 = fmaf(z4.z, w[2 * EMB], y3); y3 = fmaf(z4.w, w[3 * EMB], y3);
  }
  if (lane >= EMB) y3 = 0.f;
  const float ss = warp_sum(y3 * y3);
  const float rq3 = 1.0f / fmaxf(sqrtf(ss), 1e-12f);   // F.normalize(p=2, dim=2), eps 1e-12
  const float yh3 = y3 * rq3;
  const float e1v = fmaxf(Yh1[lh], 0.f);  // row 0 of H1
  const float e2v = fmaxf(Yh2[lh], 0.f);  // row 0 of H2
  __syncwarp();
  if (lane < HID) { zs[lane] = e1v; zs[HID + lane] = e2v; }
  if (lane < EMB) zs[2 * HID + lane] = yh3;
  __syncwarp();
  // logits = pred_model(concat): four classes at a time, eight lanes per class
  for (int cb = 0; cb < C; cb += 4) {
    const int c = cb + g;
    const float* wp = Wpp + (c < C ? c : C - 1) * PD;
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < (PD + 7) / 8; ++k) {
      const int kk = q8 + 8 * k;
      if (kk < PD) t = fmaf(zs[kk], wp[kk], t);
    }
    t += __shfl_xor_sync(0xffffffffu, t, 1);
    t += __shfl_xor_sync(0xffffffffu, t, 2);
    t += __shfl_xor_sync(0xffffffffu, t, 4);
    if (c < C && q8 == 0) logit[c] = t + bpp[c];
  }
  __syncwarp();
  // softmax over the classes, dL/dlogits = p - onehot(gt) (explain.py:750-753)
  if (C <= 32) {
    const float v = lane < C ? logit[lane] : -INFINITY;
    const float mx = warp_max(v);
    const float ex = lane < C ? expf(v - mx) : 0.f;
    const float se = warp_sum(ex);
    if (kTrace) {
      if (lane == gt) { tr[0] = -((v - mx) - logf(se)); tr[1] = ex / se; }
      if (trp != nullptr && lane < C) trp[lane] = ex / se;
    }
    if (lane < C) logit[lane] = ex / se - (lane == gt ? 1.f : 0.f);
  } else {
    float mx = -INFINITY;
#pragma unroll 1
    for (int c = lane; c < C; c += 32) mx = fmaxf(mx, logit[c]);
    mx = warp_max(mx);
    float se = 0.f;
#pragma unroll 1
    for (int c = lane; c < C; c += 32) se += expf(logit[c] - mx);
    se = warp_sum(se);
    __syncwarp();
    if (kTrace) {
      if (lane == 0) { const float lg = logit[gt]; tr[0] = -((lg - mx) - logf(se)); tr[1] = expf(lg - mx) / se; }
      if (trp != nullptr)
        for (int c = lane; c < C; c += 32) trp[c] = expf(logit[c] - mx) / se;
      __syncwarp();
    }
#pragma unroll 1
    for (int c = lane; c < C; c += 32) logit[c] = expf(logit[c] - mx) / se - (c == gt ? 1.f : 0.f);
  }
  __syncwarp();
  // dEmb = Wp^T g ; backward of y/max(|y|,eps): dY = (dYh - Yh <Yh,dYh>)/q ; dZ3 = dY3 W3^T
  float d1 = 0.f, d2 = 0.f, d3 = 0.f;
  for (int c = 0; c < C; ++c) {
    const float gc = logit[c];
    const float* wp = Wpp + c * PD;
    d1 = fmaf(gc, wp[lh], d1); d2 = fmaf(gc, wp[HID + lh], d2); d3 = fmaf(gc, wp[2 * HID + le], d3);
  }
  if (lane < HID) { dE[lane] = d1; dE[HS + lane] = d2; }
  if (lane >= EMB) d3 = 0.f;
  const float s3 = warp_sum(yh3 * d3);
  const float dy3 = (d3 - yh3 * s3) * rq3;
  __syncwarp();
  if (lane < EMB) zs[lane] = dy3;
  __syncwarp();
  if (lane < HID) dZ3[lane] = dot_v4(zs, W3s + lane * EMB, EMB / 4);
}

// CS > 1: cluster launch class -- the CS CTAs of a thread-block cluster share one task (rows and pairs dealt over the cluster's
// warps, results stored into every CTA's copy of the state through DSMEM, hardware cluster barrier between phases; phases S and
// B2 concern a handful of rows and are computed redundantly by every CTA, which saves two cluster barriers per epoch).
// kNarrow: 4*ceil(d/4) <= HID == EMB (every default-width model with d <= HID; checked by the launcher).  The lane group is then
// GW = HID/4 lanes wide at compile time, and the loops over the input width run to the constant H4 with the run-time D4 as a
// predicate: the same arithmetic in the same order as the run-time shape, with fewer instructions and registers.
template <typename IdxT, int HID, int EMB, int NT, bool kTrace, int CS, bool kNarrow>
__global__ void __launch_bounds__(NT, 1024 / NT) explain_node_kernel(const ExplainArgs A) {
  extern __shared__ __align__(16) float smem_dyn[];
  __shared__ int s_task;
  __shared__ float s_tr[kTrace ? (NT / 32) * CS * 4 + 4 : 1];   // trace: per-warp partial sums of the edge phase + (pred loss, p[gt], feat-size term)
  __shared__ GxLayout sL;
  __shared__ int s_long[3];  // number of long rows among [0,n2), among [0,n1), and rows with a long < n1 prefix
  __shared__ long long s_clk[8];   // A.dbg only (thread 0): clock64 sums of the phases F1 F2 S B2 B1 P, the last mark, the task's start (globaltimer ns)
  static_assert(HID % 4 == 0 && EMB % 4 == 0, "hidden widths must be multiples of 4");
  static_assert(sizeof(IdxT) == 2, "the pair slab packs two indices per word");
  static_assert(!kNarrow || (CS == 1 && EMB == HID), "the narrow instantiation is for single-CTA tasks of HID == EMB models");
  constexpr IdxT kNone = IdxTraits<IdxT>::kNone;
  constexpr int HS = HID;            // row stride of the hidden-width arrays
  constexpr int H4 = HID / 4;
  constexpr int PD = 2 * HID + EMB;  // pred_model input width (concat of the three layers)
  constexpr int kF4 = kNarrow ? H4 : 0;   // compile-time bound of the loops over D4 (0: run-time trip count)
  constexpr int kGW = kNarrow ? H4 : 0;   // compile-time lane-group width (0: run-time)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nthreads = blockDim.x, nwarps = nthreads >> 5;
  const int crank = CS > 1 ? (int)cluster_ctarank() : 0;        // this CTA's rank in its cluster
  const int cid = CS > 1 ? (int)cluster_id_x() : (int)blockIdx.x;   // cluster id = index of the per-task pair-state slab
  const int cwarp = warp * CS + crank, cnwarps = nwarps * CS;   // warp id / warp count over the whole cluster (consecutive ids on different CTAs)
  Peer<CS> peer;
  peer.init(smem_dyn, (uint32_t)crank);
  float* const base = smem_dyn;
  if (CS > 1) cluster_sync_all();   // every CTA of the cluster is running before anyone stores into a peer's shared memory
  const GxModelDev& m = A.m;
  const GxHparamsDev& hp = A.hp;
  const int d = m.d, C = m.C;
  const bool ieee = (hp.flags & GX_HP_IEEE_EDGE) != 0;

  for (;;) {
    if (tid == 0 && crank == 0) peer.sti(&s_task, atomicAdd(A.counter, 1));
    phase_sync<CS>();
    const int qi = s_task;
    phase_sync<CS>();
    if (qi >= A.ntasks) break;
    const int task_id = A.order[qi];
    if (A.dbg != nullptr && tid == 0) {
      unsigned long long t_start_ns;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_start_ns));
      s_clk[7] = (long long)t_start_ns;
    }
    const GxTask* __restrict__ Tp = A.plan.tasks + task_id;
    const int n = Tp->n, n1 = Tp->n1, n2 = Tp->n2, e1 = Tp->e1, np = Tp->npairs_in;  // inner pairs only
    // gradient baseline: the loss is taken at the node's PREDICTED label (explain.py:130), otherwise at label[node] (explain.py:750-753)
    const int gt = hp.mode ? __ldg(A.g.pred_label + Tp->node) : Tp->gt_label;
    const int64_t node_off = Tp->node_off, rp_off = Tp->rp_off, edge_off = Tp->edge_off, pair_off = Tp->pair_off;
    if (tid == 0) sL = gx_make_layout(n, n1, n2, e1, d, HID, EMB, C, nwarps, (int)sizeof(IdxT), CS);
    __syncthreads();
    const int dp = sL.dp, D4 = dp / 4;
    const int32_t* __restrict__ lo2gid = A.plan.lo2gid + node_off;

    // ------------------------------------------------------------------ load
    {
      float* const X = base + sL.X; float* const W1s = base + sL.W1s; float* const W2s = base + sL.W2s; float* const W3s = base + sL.W3s;
      float* const bs = base + sL.bs; float* const sF = base + sL.sF; float* const Fm = base + sL.F; float* const mF = base + sL.mF;
      float* const vF = base + sL.vF; float* const gFp = base + sL.gFp; float* const a = base + sL.a; float* const yv = base + sL.y;
      float2* const MM = reinterpret_cast<float2*>(A.pws + (int64_t)cid * A.pws_stride_words); float2* const mm = MM + np; float2* const vv = mm + np; float2* const SS = vv + np;
      uint2* const PX = reinterpret_cast<uint2*>(SS + np);
      IdxT* const icol = reinterpret_cast<IdxT*>(base + sL.icol); IdxT* const irp = reinterpret_cast<IdxT*>(base + sL.irp);
    for (int idx = tid; idx < n * dp; idx += nthreads) {
      const int i = idx / dp, f = idx - i * dp;
      X[idx] = f < d ? __ldg(A.g.feat + (int64_t)lo2gid[i] * d + f) : 0.f;
    }
    for (int idx = tid; idx < dp * HS; idx += nthreads) {
      const int f = idx / HS, c = idx - f * HS;
      W1s[idx] = f < d ? __ldg(m.W[0] + f * HID + c) : 0.f;
    }
    for (int idx = tid; idx < HID * HS; idx += nthreads) W2s[idx] = __ldg(m.W[1] + idx);
    {
      float* const W1t = base + sL.W1t; float* const W2t = base + sL.W2t;
      for (int idx = tid; idx < HID * dp; idx += nthreads) {   // W1t[c][f] = W1[f][c], zero for f >= d
        const int c = idx / dp, f = idx - c * dp;
        W1t[idx] = f < d ? __ldg(m.Wt[0] + c * d + f) : 0.f;
      }
      for (int idx = tid; idx < HID * HID; idx += nthreads) W2t[idx] = __ldg(m.Wt[1] + idx);
    }
    for (int idx = tid; idx < HID * EMB; idx += nthreads) W3s[idx] = __ldg(m.W[2] + idx);
    for (int idx = tid; idx < HID; idx += nthreads) { bs[idx] = __ldg(m.b[0] + idx); bs[HID + idx] = __ldg(m.b[1] + idx); }
    for (int idx = tid; idx < EMB; idx += nthreads) bs[2 * HID + idx] = __ldg(m.b[2] + idx);
    if (C * (PD + 1) <= GX_WP_SMEM_MAX) {
      float* const Wps = base + sL.Wp;
      for (int idx = tid; idx < C * PD; idx += nthreads) Wps[idx] = __ldg(m.Wp + idx);
      for (int idx = tid; idx < C; idx += nthreads) Wps[C * PD + idx] = __ldg(m.bp + idx);
    }
    for (int e = tid; e < e1; e += nthreads) icol[e] = (IdxT)A.plan.icol[edge_off + e];
    for (int i = tid; i <= n2; i += nthreads) irp[i] = (IdxT)A.plan.irowptr[rp_off + i];
    for (int i = tid; i < n; i += nthreads) yv[i] = (float)__ldg(A.g.pred_label + lo2gid[i]);
    const bool resume = hp.init == GX_INIT_STATE && !hp.mode;   // optimiser state supplied by the caller (gx_explain_io)
    for (int f = tid; f < dp; f += nthreads) {
      sF[f] = hp.mode ? 1.0f : 0.5f;  // sigmoid(0): feat_mask is initialised to 0 (explain.py:633-643); gradient baseline: unmasked features
      Fm[f] = 0.f; mF[f] = 0.f; vF[f] = 0.f;
      if (resume && A.x.feat_state_in != nullptr && f < d) {
        const float* fs = A.x.feat_state_in + (int64_t)task_id * 3 * d;
        Fm[f] = fs[f]; mF[f] = fs[d + f]; vF[f] = fs[2 * d + f];
        sF[f] = sigmoid_f(fs[f]);
      }
      if (hp.out_iter == 0 && !hp.mode && f < d) {   // num_epochs == 1: the state that goes out is the state that came in
        if (A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = sF[f];
        if (A.x.feat_state_out != nullptr) {
          float* fo = A.x.feat_state_out + (int64_t)task_id * 3 * d;
          fo[f] = Fm[f]; fo[d + f] = mF[f]; fo[2 * d + f] = vF[f];
        }
      }
    }
    for (int idx = tid; idx < cnwarps * dp; idx += nthreads) gFp[idx] = 0.f;
    const float m0_std = sqrtf(2.0f / (float)n);  // gain('relu') * sqrt(2/(n+n)) (explain.py:647-651)
    for (int p = tid; p < np; p += nthreads) {
      const int i = A.plan.pair_i[pair_off + p], j = A.plan.pair_j[pair_off + p];
      const int pij = A.plan.pair_pij[pair_off + p], pji = A.plan.pair_pji[pair_off + p];
      const int oij = A.plan.pair_oij[pair_off + p], oji = A.plan.pair_oji[pair_off + p];
      float Mi, Mj;
      if (hp.mode) {
        Mi = Mj = 0.f;
      } else if (hp.init == GX_INIT_PHILOX) {
        Mi = 1.0f + m0_std * philox_normal(hp.seed, (uint32_t)Tp->node, (uint32_t)oij);
        Mj = 1.0f + m0_std * philox_normal(hp.seed, (uint32_t)Tp->node, (uint32_t)oji);
      } else {
        Mi = __ldg(A.m0 + edge_off + oij);
        Mj = __ldg(A.m0 + edge_off + oji);
      }
      float2 m2 = make_float2(0.f, 0.f), v2 = m2;
      if (resume) {
        m2 = make_float2(__ldg(A.x.adam_m_in + edge_off + oij), __ldg(A.x.adam_m_in + edge_off + oji));
        v2 = make_float2(__ldg(A.x.adam_v_in + edge_off + oij), __ldg(A.x.adam_v_in + edge_off + oji));
      }
      const bool mine = CS == 1 || ((p >> 5) % CS) == crank;   // the CTA that owns this pair in the edge phase
      const float Si = resume ? sigmoid_fast(Mi, ieee) : sigmoid_f(Mi), Sj = resume ? sigmoid_fast(Mj, ieee) : sigmoid_f(Mj);   // a resumed state came out of the edge phase: same sigmoid as there, so that a split run equals the straight one bit for bit
      if (mine) {
        MM[p] = make_float2(Mi, Mj);
        mm[p] = m2;
        vv[p] = v2;
        SS[p] = make_float2(Si, Sj);
        // (i, j) and the pair's slots in rows i and j of `a` (kNone: the row is beyond n2), two 16-bit indices per word
        PX[p] = make_uint2((uint32_t)i | ((uint32_t)j << 16),
                           (uint32_t)(i < n2 ? (IdxT)pij : kNone) | ((uint32_t)(j < n2 ? (IdxT)pji : kNone) << 16));
      }
      const float a0 = hp.mode ? 1.0f : 0.5f * (Si + Sj);  // explain.py:665-678 ; gradient baseline: the adjacency itself
      if (i < n2) a[pij] = a0;
      if (j < n2) a[pji] = a0;
      if (mine && hp.out_iter == 0 && !hp.mode) {
        A.out_mask[edge_off + oij] = a0;
        A.out_mask[edge_off + oji] = a0;
        if (A.x.mask_param_out != nullptr) { A.x.mask_param_out[edge_off + oij] = Mi; A.x.mask_param_out[edge_off + oji] = Mj; }
        if (A.x.adam_m_out != nullptr) { A.x.adam_m_out[edge_off + oij] = m2.x; A.x.adam_m_out[edge_off + oji] = m2.y; }
        if (A.x.adam_v_out != nullptr) { A.x.adam_v_out[edge_off + oij] = v2.x; A.x.adam_v_out[edge_off + oji] = v2.y; }
      }
    }
    }
    __syncthreads();
    // rows with more than kLongRow edges (hubs): explicit list (ascending row id), aggregated by whole
    // warps and dealt across warps; everything else goes through the lane-group path
    if (warp == 0) {
      const IdxT* const irp = reinterpret_cast<const IdxT*>(base + sL.irp);
      IdxT* const llist = reinterpret_cast<IdxT*>(base + sL.llist);
      int cnt = 0, cnt1 = 0;
      for (int b0 = 0; b0 < n2; b0 += 32) {
        const int i = b0 + lane;
        const bool lg = i < n2 && ((int)irp[i + 1] - (int)irp[i] > kLongRow);
        const uint32_t bal = __ballot_sync(0xffffffffu, lg);
        if (lg) llist[cnt + __popc(bal & ((1u << lane) - 1u))] = (IdxT)i;
        cnt += __popc(bal);
        cnt1 += __popc(__ballot_sync(0xffffffffu, lg && i < n1));
      }
      if (lane == 0) { s_long[0] = cnt; s_long[1] = cnt1; }
    }
    __syncthreads();
    {  // per row: how many leading columns are < n1 (rows are partitioned by the level of the neighbour)
      const IdxT* const irp = reinterpret_cast<const IdxT*>(base + sL.irp);
      const IdxT* const icol = reinterpret_cast<const IdxT*>(base + sL.icol);
      IdxT* const cnt1 = reinterpret_cast<IdxT*>(base + sL.cnt1);
      for (int i = tid; i < n2; i += nthreads) {
        const int r0 = irp[i], r1 = irp[i + 1];
        int c = 0;
        while (r0 + c < r1 && (int)icol[r0 + c] < n1) ++c;
        cnt1[i] = (IdxT)c;
      }
    }
    __syncthreads();
    if (warp == 0) {   // rows whose gradient-carrying prefix is long (hub-adjacent rows)
      const IdxT* const cnt1 = reinterpret_cast<const IdxT*>(base + sL.cnt1);
      IdxT* const llistB = reinterpret_cast<IdxT*>(base + sL.llistB);
      int cnt = 0;
      for (int b0 = 0; b0 < n2; b0 += 32) {
        const int i = b0 + lane;
        const bool lg = i < n2 && (int)cnt1[i] > kLongRow;
        const uint32_t bal = __ballot_sync(0xffffffffu, lg);
        if (lg) llistB[cnt + __popc(bal & ((1u << lane) - 1u))] = (IdxT)i;
        cnt += __popc(bal);
      }
      if (lane == 0) s_long[2] = cnt;
    }
    __syncthreads();
    const int nlongB1 = s_long[2];
    const int nlongF1 = s_long[0];  // long rows among [0,n2)
    const int nlongF2 = s_long[1];  // long rows among [0,n1) (a prefix of the list)

    // lane groups: GW lanes per row
    Grp G;
    {
      int gw = kNarrow ? H4 : (D4 > H4 ? D4 : H4);
      gw = gw > (EMB / 4) ? gw : (EMB / 4);
      G.GW = gw; G.epi = 32 / gw; G.lane = lane; G.grp = lane / gw; G.q = lane - G.grp * gw; G.gbase = G.grp * gw;
    }
    const int epi = G.epi, q = G.q;

    // ------------------------------------------------------------------ epochs
    // phase timers (tools/phase_timers.py): kept in shared memory, so that they take no registers in the epoch loop
    if (A.dbg != nullptr && tid == 0) {
      for (int k = 0; k < 6; ++k) s_clk[k] = 0;
      s_clk[6] = clock64();
    }
#define GX_MARK(k) if (A.dbg != nullptr && tid == 0) { const long long c_ = clock64(); s_clk[k] += c_ - s_clk[6]; s_clk[6] = c_; }
    for (int it = 1; it <= hp.iters; ++it) {
      // ---- F1: rows [0,n2): U = A_m X ; Y1 = (U . sF) W1 + b1 ; row normalise            (models.py:70-78)
      {
        const IdxT* const irp = reinterpret_cast<const IdxT*>(base + sL.irp);
        const IdxT* const icol = reinterpret_cast<const IdxT*>(base + sL.icol);
        const IdxT* const llist = reinterpret_cast<const IdxT*>(base + sL.llist);
        const float* const a = base + sL.a; const float* const X = base + sL.X; float* const U = base + sL.U;
        float* const zs = base + sL.zs + warp * 128; const float* const bs = base + sL.bs;
        const float* const sF = base + sL.sF; const float* const W1s = base + sL.W1s;
        float* const Yh1 = base + sL.Yh1; float* const q1 = base + sL.q1;
        const int ntask = nlongF1 + (n2 + epi - 1) / epi;
        for (int t = cwarp; t < ntask; t += cnwarps) {
          float4 z;
          const int i = row_task_gather<IdxT, false, (NT >= 512 ? 4 : GX_SHORT_DEPTH)>(t, nlongF1, llist, n2, G, D4, irp, icol, a, X, dp, (const IdxT*)nullptr, zs, z);
          const bool act = i >= 0;
          if (act && q < D4) {
            peer.st4(U + i * dp + 4 * q, z);
            const float4 s4 = ld4(sF + 4 * q);   // x * sigmoid(feat_mask) (explain.py:707), linear in x
            st4(zs + lane * 4, make_float4(z.x * s4.x, z.y * s4.y, z.z * s4.z, z.w * s4.w));
          }
          __syncwarp();
          float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
          if (act && q < H4) y = group_dense<kF4>(zs + G.gbase * 4, D4, W1s, HS, q, ld4(bs + 4 * q));
          const float ss = group_sum<kGW>(y.x * y.x + y.y * y.y + y.z * y.z + y.w * y.w, G);
          const float qn = fmaxf(sqrtf(ss), 1e-12f);  // F.normalize(p=2, dim=2), eps 1e-12
          const float rq = 1.0f / qn;   // one division per row; the row is scaled by (and the backward reuses) the reciprocal
          if (act && q < H4) peer.st4(Yh1 + i * HS + 4 * q, make_float4(y.x * rq, y.y * rq, y.z * rq, y.w * rq));
          if (act && q == 0) peer.st1(q1 + i, rq);
          __syncwarp();
        }
      }
      phase_sync<CS>();
      GX_MARK(0)
      // ---- F2: rows [0,n1): Y2 = (A_m relu(Yh1)) W2 + b2 ; row normalise
      {
        const IdxT* const irp = reinterpret_cast<const IdxT*>(base + sL.irp);
        const IdxT* const icol = reinterpret_cast<const IdxT*>(base + sL.icol);
        const IdxT* const llist = reinterpret_cast<const IdxT*>(base + sL.llist);
        const float* const a = base + sL.a; const float* const Yh1 = base + sL.Yh1;
        float* const zs = base + sL.zs + warp * 128; const float* const bs = base + sL.bs;
        const float* const W2s = base + sL.W2s; float* const Yh2 = base + sL.Yh2; float* const q2 = base + sL.q2;
        const int ntask = nlongF2 + (n1 + epi - 1) / epi;
        for (int t = cwarp; t < ntask; t += cnwarps) {
          float4 z;
          const int i = row_task_gather<IdxT, true, (NT >= 512 ? 4 : GX_SHORT_DEPTH)>(t, nlongF2, llist, n1, G, H4, irp, icol, a, Yh1, HS, (const IdxT*)nullptr, zs, z);
          const bool act = i >= 0;
          if (act && q < H4) st4(zs + lane * 4, z);
          __syncwarp();
          float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
          if (act && q < H4) y = group_dense(zs + G.gbase * 4, H4, W2s, HS, q, ld4(bs + HID + 4 * q));
          const float ss = group_sum<kGW>(y.x * y.x + y.y * y.y + y.z * y.z + y.w * y.w, G);
          const float qn = fmaxf(sqrtf(ss), 1e-12f);
          const float rq = 1.0f / qn;
          if (act && q < H4) peer.st4(Yh2 + i * HS + 4 * q, make_float4(y.x * rq, y.y * rq, y.z * rq, y.w * rq));
          if (act && q == 0) peer.st1(q2 + i, rq);
          __syncwarp();
        }
      }
      phase_sync<CS>();
      GX_MARK(1)
      // ---- S: row r (= level-order id 0): layer 3, readout, softmax, -log p[gt], layer-3 backward
      if (warp == 0) {
        const IdxT* const irp = reinterpret_cast<const IdxT*>(base + sL.irp);
        const IdxT* const icol = reinterpret_cast<const IdxT*>(base + sL.icol);
        const float* const a = base + sL.a; const float* const Yh1 = base + sL.Yh1; const float* const Yh2 = base + sL.Yh2;
        float* const zs = base + sL.zs; const float* const bs = base + sL.bs; const float* const W3s = base + sL.W3s;
        float* const logit = base + sL.logit; float* const dE = base + sL.dE; float* const dZ3 = base + sL.dZ3;
        float* const tr = kTrace ? s_tr + (NT / 32) * CS * 4 : nullptr;
        float* const trp = (kTrace && A.x.trace_pred != nullptr && crank == 0) ? A.x.trace_pred + ((int64_t)task_id * A.x.epochs + (it - 1)) * C : nullptr;
        if (C * (PD + 1) <= GX_WP_SMEM_MAX)   // pred_model.weight (C, 2h+e) + bias staged in shared memory
          readout_phase<IdxT, HID, EMB, true, kTrace>(lane, C, gt, irp, icol, a, Yh1, Yh2, zs, bs, W3s, base + sL.Wp, base + sL.Wp + C * PD, logit, dE, dZ3, tr, trp);
        else
          readout_phase<IdxT, HID, EMB, false, kTrace>(lane, C, gt, irp, icol, a, Yh1, Yh2, zs, bs, W3s, m.Wp, m.bp, logit, dE, dZ3, tr, trp);
        if (kTrace) {   // feat_size_loss = coeff * mean(sigmoid(feat_mask)) with the mask this epoch's forward used (explain.py:763-766)
          const float* const sF = base + sL.sF;
          float fs = 0.f;
          for (int f = lane; f < d; f += 32) fs += sF[f];
          fs = warp_sum(fs);
          if (lane == 0) tr[2] = hp.c_feat_size * fs / (float)d;
        }
      }
      __syncthreads();
      GX_MARK(2)
      // ---- B2: rows {r} U N(r): dYh2 = dEmb2 (row r) + a[r,j] dZ3 (j in N(r)), relu', normalise', dZ2 = dY2 W2^T
      {
        const IdxT* const irp = reinterpret_cast<const IdxT*>(base + sL.irp);
        const IdxT* const icol = reinterpret_cast<const IdxT*>(base + sL.icol);
        const float* const a = base + sL.a; const float* const dE = base + sL.dE; const float* const dZ3 = base + sL.dZ3;
        const float* const Yh2 = base + sL.Yh2; const float* const q2 = base + sL.q2; const float* const W2t = base + sL.W2t;
        float* const dZ2 = base + sL.dZ2; float* const zs = base + sL.zs + warp * 128;
        const int r0 = irp[0];
        const int items = 1 + (int)irp[1] - r0;
        const int ntask = (items + epi - 1) / epi;
        for (int t = warp; t < ntask; t += nwarps) {
          const int item = t * epi + G.grp;
          const bool act = G.grp < epi && item < items;
          int j = 0;
          float coef = 1.f;
          const float* dsrc = dE + HS;
          if (act && item > 0) {
            const int e = r0 + item - 1;
            j = icol[e];
            coef = a[e];
            dsrc = dZ3;
          }
          float4 yh = make_float4(0.f, 0.f, 0.f, 0.f), dy = yh;
          if (act && q < H4) {
            yh = ld4(Yh2 + j * HS + 4 * q);
            const float4 g4 = ld4(dsrc + 4 * q);
            dy.x = yh.x > 0.f ? coef * g4.x : 0.f;   // relu backward: grad where input > 0
            dy.y = yh.y > 0.f ? coef * g4.y : 0.f;
            dy.z = yh.z > 0.f ? coef * g4.z : 0.f;
            dy.w = yh.w > 0.f ? coef * g4.w : 0.f;
          }
          const float sdot = group_sum<kGW>(yh.x * dy.x + yh.y * dy.y + yh.z * dy.z + yh.w * dy.w, G);
          if (act && q < H4) {
            const float rq = q2[j];   // 1 / max(|Y2[j]|, eps)
            st4(zs + lane * 4, make_float4((dy.x - yh.x * sdot) * rq, (dy.y - yh.y * sdot) * rq,
                                           (dy.z - yh.z * sdot) * rq, (dy.w - yh.w * sdot) * rq));
          }
          __syncwarp();
          if (act && q < H4)
            st4(dZ2 + j * HS + 4 * q, group_dense(zs + G.gbase * 4, H4, W2t, HS, q, make_float4(0.f, 0.f, 0.f, 0.f)));
          __syncwarp();
        }
      }
      __syncthreads();
      GX_MARK(3)
      // ---- B1: rows [0,n2): dH1 = A_m^T dZ2 (only columns < n1 carry gradient), relu', normalise',
      //          dZ1 = dY1 W1^T, dL/dsF partial, dZ1 (.) sF kept for the edge dots
      {
        const IdxT* const irp = reinterpret_cast<const IdxT*>(base + sL.irp);
        const IdxT* const icol = reinterpret_cast<const IdxT*>(base + sL.icol);
        const float* const a = base + sL.a; const float* const dZ2 = base + sL.dZ2; const float* const dE = base + sL.dE;
        const float* const Yh1 = base + sL.Yh1; const float* const q1 = base + sL.q1; const float* const W1t = base + sL.W1t;
        const float* const U = base + sL.U; const float* const sF = base + sL.sF;
        const IdxT* const cnt1 = reinterpret_cast<const IdxT*>(base + sL.cnt1);
        const IdxT* const llistB = reinterpret_cast<const IdxT*>(base + sL.llistB);
        float* const dZ1s = base + sL.U;  // row i of U is consumed (dL/dsF) right before dZ1[i] (.) sF overwrites it
        float* const gFp = base + sL.gFp; float* const zs = base + sL.zs + warp * 128;
        float4 gacc = make_float4(0.f, 0.f, 0.f, 0.f);
        const int ntask = nlongB1 + (n2 + epi - 1) / epi;
        for (int t = cwarp; t < ntask; t += cnwarps) {
          float4 dh;
          const int i = row_task_gather<IdxT, false, (NT >= 512 ? 1 : GX_SHORT_DEPTH)>(t, nlongB1, llistB, n2, G, H4, irp, icol, a, dZ2, HS, cnt1, zs, dh);
          const bool act = i >= 0;
          float4 yh = make_float4(0.f, 0.f, 0.f, 0.f), dy = yh;
          if (act && q < H4) {
            yh = ld4(Yh1 + i * HS + 4 * q);
            if (i == 0) { const float4 e4 = ld4(dE + 4 * q); dh.x += e4.x; dh.y += e4.y; dh.z += e4.z; dh.w += e4.w; }
            dy.x = yh.x > 0.f ? dh.x : 0.f; dy.y = yh.y > 0.f ? dh.y : 0.f;
            dy.z = yh.z > 0.f ? dh.z : 0.f; dy.w = yh.w > 0.f ? dh.w : 0.f;
          }
          const float sdot = group_sum<kGW>(yh.x * dy.x + yh.y * dy.y + yh.z * dy.z + yh.w * dy.w, G);
          if (act && q < H4) {
            const float rq = q1[i];   // 1 / max(|Y1[i]|, eps)
            st4(zs + lane * 4, make_float4((dy.x - yh.x * sdot) * rq, (dy.y - yh.y * sdot) * rq,
                                           (dy.z - yh.z * sdot) * rq, (dy.w - yh.w * sdot) * rq));
          }
          __syncwarp();
          if (act && q < D4) {
            const float4 o = group_dense(zs + G.gbase * 4, H4, W1t, dp, q, make_float4(0.f, 0.f, 0.f, 0.f));
            const float4 u = ld4(U + i * dp + 4 * q);
            const float4 s4 = ld4(sF + 4 * q);
            gacc.x = fmaf(o.x, u.x, gacc.x); gacc.y = fmaf(o.y, u.y, gacc.y);
            gacc.z = fmaf(o.z, u.z, gacc.z); gacc.w = fmaf(o.w, u.w, gacc.w);
            peer.st4(dZ1s + i * dp + 4 * q, make_float4(o.x * s4.x, o.y * s4.y, o.z * s4.z, o.w * s4.w));
          }
          __syncwarp();
        }
        // per-warp dL/dsF partial: sum the groups' accumulators (fixed order => deterministic)
        st4(zs + lane * 4, gacc);
        __syncwarp();
        if (G.grp == 0 && q < D4) {
          float4 tsum = gacc;
          for (int g2 = 1; g2 < epi; ++g2) {
            const float4 o = ld4(zs + (g2 * G.GW + q) * 4);
            tsum.x += o.x; tsum.y += o.y; tsum.z += o.z; tsum.w += o.w;
          }
          peer.st4(gFp + cwarp * dp + 4 * q, tsum);
        }
        __syncwarp();
      }
      phase_sync<CS>();
      GX_MARK(4)
      if (A.dbg != nullptr && it == 1 && qi == 0 && crank == 0) {   // debug: [header 16 floats][whole task slab]
        if (tid == 0) {
          A.dbg[0] = (float)sL.total_words; A.dbg[1] = (float)sL.X; A.dbg[2] = (float)sL.U; A.dbg[3] = (float)sL.Yh1;
          A.dbg[4] = (float)sL.q1; A.dbg[5] = (float)sL.Yh2; A.dbg[6] = (float)sL.q2; A.dbg[7] = (float)sL.dZ2;
          A.dbg[8] = (float)sL.U; A.dbg[9] = (float)sL.gFp; A.dbg[10] = (float)sL.dE; A.dbg[11] = (float)sL.dZ3;
          A.dbg[12] = (float)sL.logit; A.dbg[13] = (float)sL.a; A.dbg[14] = (float)dp; A.dbg[15] = (float)nwarps;
        }
        for (int w = tid; w < sL.total_words; w += nthreads) A.dbg[16 + w] = base[w];
      }
      // ---- P: per undirected edge: dA_ij, dA_ji, symmetrise, regularisers, Adam, next mask value
      {
        float* const gFp = base + sL.gFp;
        float* const sF = base + sL.sF;
        float* const Fm = base + sL.F; float* const mF = base + sL.mF; float* const vF = base + sL.vF;
        const float* const yv = base + sL.y;
        const float* const dZ1s = base + sL.U;
        float* const X = base + sL.X;
        float* const dZ2 = base + sL.dZ2;
        float* const Yh1 = base + sL.Yh1;
        float* const dZ3 = base + sL.dZ3;
        float* const Yh2 = base + sL.Yh2;
        float2* const MM = reinterpret_cast<float2*>(A.pws + (int64_t)cid * A.pws_stride_words); float2* const mm = MM + np; float2* const vv = mm + np; float2* const SS = vv + np;
        const uint2* const PX = reinterpret_cast<const uint2*>(SS + np);
        float* const a = base + sL.a;
        // the pairs' indices come from the L2-resident slab one round ahead of their use: the dots below wait for no L2 round trip
        const int p0 = cwarp * 32 + lane, pstride = nthreads * CS;
        uint2 pxn = p0 < np ? PX[p0] : make_uint2(0u, 0u);
        const float2 tab = __ldg(hp.adam_tab + (it - 1));
        const float step = tab.x, bc2s = tab.y, bc2s_inv = 1.0f / tab.y;
        const bool last = (it == hp.out_iter);   // the mask built after this update is the one the reference returns
        const float nn = (float)n * (float)n;      // (formed here rather than once per task: nothing has to stay live across the epoch)
        const float ent_over_nn = hp.c_ent / nn;
        const float lap_over_nn = hp.c_lap / nn;
        // feature mask: dL/dF = sF(1-sF) (sum_i dZ1[i] U[i] + feat_size/d) ; Adam (explain.py:766, train_utils.py:10)
        // (done by the LAST warps of the CTA: the first ones carry the most pair work below, and a warp whose first lanes run this
        //  serial update would hold back its 32 pairs)
        const int fthreads = min(nthreads, gx_round_up(d, 32));
        for (int f = tid - (nthreads - fthreads); f >= 0 && f < d && !hp.mode; f += fthreads) {
          float gsum = 0.f;
          for (int w = 0; w < cnwarps; ++w) gsum += gFp[w * dp + f];
          const float s = sF[f];
          const float g = s * (1.f - s) * (gsum + hp.c_feat_size / (float)d);
          float mf = mF[f], vf = vF[f], Fv = Fm[f];
          mf = mf + (g - mf) * hp.one_minus_b1;
          vf = vf * hp.b2 + hp.one_minus_b2 * g * g;
          Fv = Fv - step * (mf / (sqrtf(vf) / bc2s + hp.eps));
          mF[f] = mf; vF[f] = vf; Fm[f] = Fv;
          const float sn = sigmoid_f(Fv);
          sF[f] = sn;
          if (last && crank == 0) {
            if (A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = sn;
            if (A.x.feat_state_out != nullptr) {
              float* fo = A.x.feat_state_out + (int64_t)task_id * 3 * d;
              fo[f] = Fv; fo[d + f] = mf; fo[2 * d + f] = vf;
            }
          }
        }
        float trS = 0.f, trH = 0.f, trL = 0.f, trD = 0.f;   // trace: this thread's share of sum S, sum H(S), sum a (y_i-y_j)^2, sum 2a'
        if (hp.mode) {
          // gradient baseline (explain.py:125-133): mask_ij = sigmoid(|dL/dA_ij| + |dL/dA_ji|) on the edges, no regulariser, no update
          for (int p = p0; p < np; p += pstride) {
            const uint2 px = pxn;
            if (p + pstride < np) pxn = PX[p + pstride];
            const int i = px.x & 0xffffu, j = px.x >> 16;
            float gij = 0.f, gji = 0.f;
            if (i < n2) gij += dot_v4<kF4>(dZ1s + i * dp, X + j * dp, D4);
            if (j < n2) gji += dot_v4<kF4>(dZ1s + j * dp, X + i * dp, D4);
            if (i < n1) gij += dot_relu_v4(dZ2 + i * HS, Yh1 + j * HS, H4);
            if (j < n1) gji += dot_relu_v4(dZ2 + j * HS, Yh1 + i * HS, H4);
            if (i == 0) gij += dot_relu_v4(dZ3, Yh2 + j * HS, H4);
            const float an = sigmoid_f(fabsf(gij) + fabsf(gji));
            A.out_mask[edge_off + A.plan.pair_oij[pair_off + p]] = an;
            A.out_mask[edge_off + A.plan.pair_oji[pair_off + p]] = an;
          }
        } else
        for (int p = p0; p < np; p += pstride) {
          // optimiser state of the pair (L2-resident slab): issued first so that the L2 round trip overlaps the dots below
          float2 Mv = MM[p];
          const float2 Sv = SS[p];
          float2 m2 = mm[p], v2 = vv[p];
          const uint2 px = pxn;
          if (p + pstride < np) pxn = PX[p + pstride];
          const int i = px.x & 0xffffu, j = px.x >> 16;
          const float yd = yv[i] - yv[j];
          float Gd = lap_over_nn * yd * yd;  // d/dA_ij + d/dA_ji of y^T (D - A) y / n^2 (explain.py:780-793)
          if (kTrace) {
            trS += Sv.x + Sv.y; trH += bern_entropy(Sv.x) + bern_entropy(Sv.y);
            trL += 0.5f * (Sv.x + Sv.y) * yd * yd;
          }
          if (i < n2) Gd += dot_v4<kF4>(dZ1s + i * dp, X + j * dp, D4);
          if (j < n2) Gd += dot_v4<kF4>(dZ1s + j * dp, X + i * dp, D4);
          if (i < n1) Gd += dot_relu_v4(dZ2 + i * HS, Yh1 + j * HS, H4);
          if (j < n1) Gd += dot_relu_v4(dZ2 + j * HS, Yh1 + i * HS, H4);
          if (i == 0) Gd += dot_relu_v4(dZ3, Yh2 + j * HS, H4);
          Gd *= 0.5f;  // sym_mask = (S + S^T)/2 (explain.py:671)
          // size: coeff*sum(S) ; entropy: mean over n^2 of H(S), dH/dM = -M S(1-S) (explain.py:755-770)
          const float gi = Sv.x * (1.f - Sv.x) * (Gd + hp.c_size - ent_over_nn * Mv.x);
          const float gj = Sv.y * (1.f - Sv.y) * (Gd + hp.c_size - ent_over_nn * Mv.y);
          m2.x = m2.x + (gi - m2.x) * hp.one_minus_b1;
          m2.y = m2.y + (gj - m2.y) * hp.one_minus_b1;
          v2.x = v2.x * hp.b2 + hp.one_minus_b2 * gi * gi;
          v2.y = v2.y * hp.b2 + hp.one_minus_b2 * gj * gj;
          Mv.x = Mv.x - adam_delta_fast(m2.x, v2.x, step, bc2s, bc2s_inv, hp.eps, ieee);
          Mv.y = Mv.y - adam_delta_fast(m2.y, v2.y, step, bc2s, bc2s_inv, hp.eps, ieee);
          const float2 Sn = make_float2(sigmoid_fast(Mv.x, ieee), sigmoid_fast(Mv.y, ieee));
          MM[p] = Mv; mm[p] = m2; vv[p] = v2; SS[p] = Sn;
          const float an = 0.5f * (Sn.x + Sn.y);
          if (kTrace) trD += 2.0f * an;
          const IdxT pa = (IdxT)(px.y & 0xffffu), pb = (IdxT)(px.y >> 16);
          if (pa != kNone) peer.st1(a + pa, an);
          if (pb != kNone) peer.st1(a + pb, an);
          if (last) {
            const int64_t oij = edge_off + A.plan.pair_oij[pair_off + p], oji = edge_off + A.plan.pair_oji[pair_off + p];
            A.out_mask[oij] = an;
            A.out_mask[oji] = an;
            if (A.x.mask_param_out != nullptr) { A.x.mask_param_out[oij] = Mv.x; A.x.mask_param_out[oji] = Mv.y; }
            if (A.x.adam_m_out != nullptr) { A.x.adam_m_out[oij] = m2.x; A.x.adam_m_out[oji] = m2.y; }
            if (A.x.adam_v_out != nullptr) { A.x.adam_v_out[oij] = v2.x; A.x.adam_v_out[oji] = v2.y; }
          }
        }
        if (kTrace) {
          trS = warp_sum(trS); trH = warp_sum(trH); trL = warp_sum(trL); trD = warp_sum(trD);
          if (lane == 0) { peer.st1(s_tr + cwarp * 4 + 0, trS); peer.st1(s_tr + cwarp * 4 + 1, trH); peer.st1(s_tr + cwarp * 4 + 2, trL); peer.st1(s_tr + cwarp * 4 + 3, trD); }
        }
      }
      phase_sync<CS>();
      if (kTrace && tid == 0 && crank == 0) {   // raw terms of epoch it-1 over the INNER pairs; trace_finalize_kernel adds the outer pairs and assembles the columns
        float sS = 0.f, sH = 0.f, sLp = 0.f, sD = 0.f;
        for (int w = 0; w < cnwarps; ++w) { sS += s_tr[w * 4]; sH += s_tr[w * 4 + 1]; sLp += s_tr[w * 4 + 2]; sD += s_tr[w * 4 + 3]; }
        float* row = A.x.trace + ((int64_t)task_id * A.x.epochs + (it - 1)) * GX_TRACE_COLS;
        const float* const tr = s_tr + (NT / 32) * CS * 4;
        row[0] = sS; row[1] = tr[0]; row[2] = sH; row[3] = sLp; row[4] = sD; row[5] = tr[2]; row[6] = 0.f; row[7] = tr[1];
      }
      GX_MARK(5)
    }
    if (A.dbg != nullptr && tid == 0 && qi == 0 && crank == 0) {
      float* o = A.dbg + (1 << 19);
      for (int k = 0; k < 6; ++k) o[k] = (float)s_clk[k];
      o[6] = (float)n; o[7] = (float)n1; o[8] = (float)n2; o[9] = (float)np; o[10] = (float)e1; o[11] = (float)nthreads;
      o[12] = kNarrow ? 1.f : 0.f;   // which instantiation ran (tests/test_gpu_node_narrow.py)
    }
    if (A.dbg != nullptr && tid == 0 && crank == 0) {
      unsigned long long t_end_ns; unsigned smid;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_end_ns));
      asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
      unsigned long long* tl64 = reinterpret_cast<unsigned long long*>(A.dbg + (1 << 19) + 64);
      tl64[3 * task_id + 0] = (unsigned long long)s_clk[7]; tl64[3 * task_id + 1] = t_end_ns; tl64[3 * task_id + 2] = ((unsigned long long)smid << 32) | (unsigned)nthreads;
    }
    phase_sync<CS>();
  }
}


// Pairs between two outermost nodes (both endpoints outside every row the forward computes): their
// masked-adjacency value never enters the GCN, so dL/dM is regulariser-only and the whole Adam
// trajectory is a private scalar recurrence -- one thread per pair, state in registers, no barriers.
// kTrace: one CTA per task additionally sums, per epoch, the pairs' shares of the size / entropy / Laplacian terms and of
// the mask density into x.tr_outer (double atomics in shared memory: the order of the adds is not fixed, the sums agree to ~1e-16).
template <bool kTrace>
__global__ void __launch_bounds__(256)
outer_pairs_kernel(const GxHparamsDev hp, const GxGraphDev g, const GxPlanArrays plan, int count,
                   const float* __restrict__ m0, float* __restrict__ out_mask, const GxExtra x) {
  extern __shared__ double s_acc[];   // kTrace: [iters][4]
  const bool ieee = (hp.flags & GX_HP_IEEE_EDGE) != 0;
  const bool resume = hp.init == GX_INIT_STATE && !hp.mode;
  for (int t = blockIdx.x; t < count; t += gridDim.x) {
    const GxTask* __restrict__ Tp = plan.tasks + t;
    const int np = Tp->npairs, np_in = Tp->npairs_in, n = Tp->n;
    const int64_t edge_off = Tp->edge_off, pair_off = Tp->pair_off;
    const int32_t* __restrict__ lo2gid = plan.lo2gid + Tp->node_off;
    const float nn = (float)n * (float)n;
    const float ent_over_nn = hp.c_ent / nn, lap_over_nn = hp.c_lap / nn;
    const float m0_std = sqrtf(2.0f / (float)n);
    if (kTrace) {
      for (int k = threadIdx.x; k < hp.iters * 4; k += blockDim.x) s_acc[k] = 0.0;
      __syncthreads();
    }
    // blockIdx.y slices the pairs of a task (large tasks, few of them: configs[4] has 2.2 M outer pairs per task and one task per SM)
    for (int p = np_in + blockIdx.y * blockDim.x + threadIdx.x; p < np; p += gridDim.y * blockDim.x) {
      const int i = plan.pair_i[pair_off + p], j = plan.pair_j[pair_off + p];
      const int64_t oij = edge_off + plan.pair_oij[pair_off + p], oji = edge_off + plan.pair_oji[pair_off + p];
      if (hp.mode) {   // gradient baseline: no gradient reaches an edge outside the receptive field -> sigmoid(0)
        out_mask[oij] = 0.5f;
        out_mask[oji] = 0.5f;
        continue;
      }
      float Mi, Mj;
      if (hp.init == GX_INIT_PHILOX) {
        Mi = 1.0f + m0_std * philox_normal(hp.seed, (uint32_t)Tp->node, (uint32_t)(oij - edge_off));
        Mj = 1.0f + m0_std * philox_normal(hp.seed, (uint32_t)Tp->node, (uint32_t)(oji - edge_off));
      } else {
        Mi = __ldg(m0 + oij);
        Mj = __ldg(m0 + oji);
      }
      float mi = 0.f, mj = 0.f, vi = 0.f, vj = 0.f;
      if (resume) { mi = __ldg(x.adam_m_in + oij); mj = __ldg(x.adam_m_in + oji); vi = __ldg(x.adam_v_in + oij); vj = __ldg(x.adam_v_in + oji); }
      const float yd = (float)__ldg(g.pred_label + lo2gid[i]) - (float)__ldg(g.pred_label + lo2gid[j]);
      const float Gd = 0.5f * (lap_over_nn * yd * yd);
      float Si = resume ? sigmoid_fast(Mi, ieee) : sigmoid_f(Mi), Sj = resume ? sigmoid_fast(Mj, ieee) : sigmoid_f(Mj);
      auto emit = [&]() {
        const float an = 0.5f * (Si + Sj);
        out_mask[oij] = an;
        out_mask[oji] = an;
        if (x.mask_param_out != nullptr) { x.mask_param_out[oij] = Mi; x.mask_param_out[oji] = Mj; }
        if (x.adam_m_out != nullptr) { x.adam_m_out[oij] = mi; x.adam_m_out[oji] = mj; }
        if (x.adam_v_out != nullptr) { x.adam_v_out[oij] = vi; x.adam_v_out[oji] = vj; }
      };
      if (hp.out_iter == 0) emit();
      for (int it = 1; it <= hp.iters; ++it) {
        const float2 tab = __ldg(hp.adam_tab + (it - 1));
        if (kTrace) {
          atomicAdd(&s_acc[(it - 1) * 4 + 0], (double)(Si + Sj));
          atomicAdd(&s_acc[(it - 1) * 4 + 1], (double)(bern_entropy(Si) + bern_entropy(Sj)));
          atomicAdd(&s_acc[(it - 1) * 4 + 2], (double)(0.5f * (Si + Sj) * yd * yd));
        }
        const float gi = Si * (1.f - Si) * (Gd + hp.c_size - ent_over_nn * Mi);
        const float gj = Sj * (1.f - Sj) * (Gd + hp.c_size - ent_over_nn * Mj);
        if (hp.opt == GX_OPT_ADAM) {
          mi = mi + (gi - mi) * hp.one_minus_b1;
          mj = mj + (gj - mj) * hp.one_minus_b1;
          vi = vi * hp.b2 + hp.one_minus_b2 * gi * gi;
          vj = vj * hp.b2 + hp.one_minus_b2 * gj * gj;
          const float bc2s_inv = 1.0f / tab.y;
          Mi = Mi - adam_delta_fast(mi, vi, tab.x, tab.y, bc2s_inv, hp.eps, ieee);
          Mj = Mj - adam_delta_fast(mj, vj, tab.x, tab.y, bc2s_inv, hp.eps, ieee);
        } else {
          opt_step_other(hp.opt, Mi, gi, mi, vi, tab.x);
          opt_step_other(hp.opt, Mj, gj, mj, vj, tab.x);
        }
        Si = sigmoid_fast(Mi, ieee);
        Sj = sigmoid_fast(Mj, ieee);
        if (kTrace) atomicAdd(&s_acc[(it - 1) * 4 + 3], (double)(Si + Sj));   // 2 a' = S_i + S_j after the step (mask_density, explain.py:148)
        if (it == hp.out_iter) emit();
      }
    }
    if (kTrace) {
      __syncthreads();
      for (int k = threadIdx.x; k < hp.iters * 4; k += blockDim.x) x.tr_outer[(int64_t)t * x.epochs * 4 + k] = s_acc[k];
      __syncthreads();
    }
  }
}

template <typename IdxT, int HID, int EMB, int NT, bool kTrace, int CS, bool kNarrow>
cudaError_t launch_one_t(const GxExplainLaunch& cfg, const ExplainArgs& args, cudaStream_t s) {
  auto kern = explain_node_kernel<IdxT, HID, EMB, NT, kTrace, CS, kNarrow>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, cfg.smem_bytes);
  if (e != cudaSuccess) return e;
  // every launch class asks for the largest shared-memory carveout: CTAs of different classes (= different kernels / footprints) can then
  // share an SM; with per-kernel carveouts a CTA waits for an SM that is completely idle
  e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (e != cudaSuccess) return e;
  if (CS == 1) {
    kern<<<cfg.grid, cfg.threads, cfg.smem_bytes, s>>>(args);
    return cudaGetLastError();
  }
  // cluster launch class: cfg.grid counts CTAs (a multiple of CS); one task per cluster
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3((unsigned)cfg.grid, 1, 1);
  lc.blockDim = dim3((unsigned)cfg.threads, 1, 1);
  lc.dynamicSmemBytes = (size_t)cfg.smem_bytes;
  lc.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = CS; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  lc.attrs = at; lc.numAttrs = 1;
  return cudaLaunchKernelEx(&lc, kern, args);
}
template <typename IdxT, int HID, int EMB, int NT, int CS, bool kNarrow = false>
cudaError_t launch_one(const GxExplainLaunch& cfg, const ExplainArgs& args, cudaStream_t s) {
  if (args.x.trace != nullptr) return launch_one_t<IdxT, HID, EMB, NT, true, CS, kNarrow>(cfg, args, s);
  return launch_one_t<IdxT, HID, EMB, NT, false, CS, kNarrow>(cfg, args, s);
}

template <int HID, int EMB>
cudaError_t launch_dims(const GxExplainLaunch& cfg, const ExplainArgs& args, cudaStream_t s) {
  if (cfg.smem_bytes <= 0) return cudaErrorInvalidValue;  // tasks that do not fit shared memory belong to explain_stream.cu
  if (cfg.cluster == 4) return launch_one<uint16_t, HID, EMB, 512, 4>(cfg, args, s);
  if (cfg.cluster == 2) return launch_one<uint16_t, HID, EMB, 512, 2>(cfg, args, s);
  if (cfg.cluster != 1) return cudaErrorInvalidValue;
  // inputs no wider than the hidden width take the instantiation with the lane-group shape fixed at compile time;
  // GNNX_NODE_GENERIC=1 (GX_HP_NODE_GENERIC) keeps every task on the run-time-shape code, for tests and A/B runs
  const bool narrow = HID == EMB && 4 * ((args.m.d + 3) / 4) <= HID && (args.hp.flags & GX_HP_NODE_GENERIC) == 0;
  if (cfg.threads <= 256)
    return narrow ? launch_one<uint16_t, HID, EMB, 256, 1, true>(cfg, args, s) : launch_one<uint16_t, HID, EMB, 256, 1>(cfg, args, s);
  return narrow ? launch_one<uint16_t, HID, EMB, 512, 1, true>(cfg, args, s) : launch_one<uint16_t, HID, EMB, 512, 1>(cfg, args, s);
}

}  // namespace

int gx_explain_max_smem() { return 227 * 1024; }

cudaError_t gx_launch_outer_pairs(const GxHparamsDev& hp, const GxGraphDev& g, const GxPlanArrays& plan, int count,
                                  const float* m0, float* out_mask, const GxExtra& x, cudaStream_t s) {
  const int grid = count < GX_GRID_CAP ? count : GX_GRID_CAP;
  if (x.trace != nullptr) {   // (the per-task trace sums are accumulated by ONE CTA per task: no slicing)
    const size_t smem = (size_t)(hp.iters > 0 ? hp.iters : 1) * 4 * sizeof(double);
    if (smem > 48 * 1024) return cudaErrorInvalidValue;   // > 1536 epochs with a trace: refused by gx_explain_nodes_ex
    outer_pairs_kernel<true><<<grid, 256, smem, s>>>(hp, g, plan, count, m0, out_mask, x);
  } else {
    const int slices = std::max(1, std::min(32, GX_GRID_CAP / grid));   // fill the machine when the batch has few (large) tasks
    outer_pairs_kernel<false><<<dim3(grid, slices), 256, 0, s>>>(hp, g, plan, count, m0, out_mask, x);
  }
  return cudaGetLastError();
}

cudaError_t gx_launch_explain(const GxExplainLaunch& cfg, const GxGraphDev& g, const GxModelDev& m,
                              const GxHparamsDev& hp, const GxPlanArrays& plan, const float* m0,
                              float* out_mask, float* out_feat, cudaStream_t s) {
  const ExplainArgs args = explain_args(cfg, g, m, hp, plan, m0, out_mask, out_feat);
  if (m.hid == 20 && m.emb == 20) return launch_dims<20, 20>(cfg, args, s);
  if (m.hid == 32 && m.emb == 32) return launch_dims<32, 32>(cfg, args, s);   // any width <= 32, zero-padded by gx_set_model
  return cudaErrorInvalidValue;
}
