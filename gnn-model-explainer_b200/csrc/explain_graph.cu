// explain_graph.cu -- graph-classification mode of the explainer (SURVEY.md section 8 row f1).
//
// Replaces, for the default hyper-parameters, Explainer.explain(node_idx=0, graph_idx=g, graph_mode=True)
// (explainer/explain.py:80-85,137-146,209-211; loss :740-808 with lap_loss = 0 :787-788) on a
// GcnEncoderGraph (models.py:269-316: three GraphConv layers, per-layer max over ALL rows of the padded
// graph, concat, Linear).  One persistent CTA per explained graph, all epochs in one launch.
//
// Differences from the node-mode kernel (explain_node.cu), same primitives (explain_common.cuh):
//   * no receptive-field pruning: every row with at least one edge is computed at every layer, layer 3
//     included; rows WITHOUT an edge (padding, isolated atoms) all have the same embedding
//     relu(normalize(b_l)) whatever the mask is -- they are represented by one constant that joins the
//     max-pool and never receives gradient that could reach M or F;
//   * readout = column max over the rows (first arg-max, like torch.max) of the three layers, Linear,
//     softmax, -log p[graph label]; dEmb is routed to the arg-max rows;
//   * all three layers contribute SDDMM terms to every edge; no Laplacian term; the 1/n^2 of the entropy
//     regulariser and the std of M0 use the PADDED size (the reference's dense tensors are max_nodes^2).
#include "explain_common.cuh"

namespace {

// ---------------------------------------------------------------------------------------------
// Plan: rows with edges relabelled 0..na-1 (ascending), their CSR, the undirected pair list.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int lower_bound_i32(const int32_t* a, int lo, int hi, int key) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(128)
graph_plan_kernel(const GxGraphBatchDev gb, int count, GxPlanArrays P) {
  extern __shared__ int sm_map[];  // [max_nodes] full id -> level-order id (or -1), then [max_nodes+1] scratch
  const int tid = threadIdx.x, nf = gb.max_nodes;
  int* const map = sm_map;
  int* const pcnt = sm_map + nf;
  for (int t = blockIdx.x; t < count; t += gridDim.x) {
    const GxTask* T = P.tasks + t;
    const int g = T->node;
    const int32_t* rp = gb.rowptr + (int64_t)g * nf;
    const int base_e = rp[0];
    int32_t* lo2gid = P.lo2gid + T->node_off;
    int32_t* irp = P.irowptr + T->rp_off;
    int32_t* icol = P.icol + T->edge_off;
    // serial prefix over <= max_nodes rows (tiny): active rows and their row pointers
    if (tid == 0) {
      int na = 0, e = 0;
      for (int i = 0; i < nf; ++i) {
        const int deg = rp[i + 1] - rp[i];
        if (deg > 0) { map[i] = na; lo2gid[na] = i; irp[na] = e; e += deg; ++na; } else map[i] = -1;
      }
      irp[na] = e;
    }
    __syncthreads();
    const int na = T->n;
    for (int i = tid; i < na; i += blockDim.x) {
      const int fi = lo2gid[i];
      int cnt = 0;
      for (int e = rp[fi]; e < rp[fi + 1]; ++e) {
        const int j = map[gb.col[e]];
        icol[irp[i] + (e - rp[fi])] = j;
        cnt += j > i ? 1 : 0;
      }
      pcnt[i] = cnt;
    }
    __syncthreads();
    if (tid == 0) {
      int acc = 0;
      for (int i = 0; i < na; ++i) { const int c = pcnt[i]; pcnt[i] = acc; acc += c; }
    }
    __syncthreads();
    for (int i = tid; i < na; i += blockDim.x) {
      const int fi = lo2gid[i];
      int64_t p = T->pair_off + pcnt[i];
      for (int k = irp[i]; k < irp[i + 1]; ++k) {
        const int j = icol[k];
        if (j <= i) continue;
        const int kji = lower_bound_i32(icol, irp[j], irp[j + 1], i);
        P.pair_i[p] = i; P.pair_j[p] = j;
        P.pair_pij[p] = k; P.pair_pji[p] = kji;
        P.pair_oij[p] = rp[fi] - base_e + (k - irp[i]);                    // canonical slot = position in the graph's CSR
        P.pair_oji[p] = rp[lo2gid[j]] - base_e + (kji - irp[j]);
        ++p;
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------
struct GraphArgs {
  const int32_t* order;
  int32_t ntasks;
  int32_t* counter;
  float* pws;
  int64_t pws_stride_words;
  GxGraphBatchDev gb;
  GxModelDev m;
  GxHparamsDev hp;
  GxPlanArrays plan;
  const float* m0;
  float* out_mask;
  float* out_feat;
  GxExtra x;
  const int32_t* grad_label;   // hp.mode == 1: the loss label of every task (-1: the arg-max of the logits this forward produces)
};

template <int HID, int EMB, int NT, bool kTrace>
__global__ void __launch_bounds__(NT, 1024 / NT) explain_graph_kernel(const GraphArgs A) {
  extern __shared__ __align__(16) float base[];
  __shared__ int s_task;
  __shared__ float s_tr[kTrace ? (NT / 32) * 4 + 4 : 1];   // trace: per-warp partial sums of the edge phase + (pred loss, p[gt], feat-size term)
  __shared__ GxLayoutG sL;
  typedef uint16_t IdxT;
  constexpr IdxT kNone = 0xFFFFu;
  constexpr int HS = HID, H4 = HID / 4, E4 = EMB / 4, PD = 2 * HID + EMB;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nthreads = blockDim.x, nwarps = nthreads >> 5;
  const GxModelDev& m = A.m;
  const GxHparamsDev& hp = A.hp;
  const int d = m.d, C = m.C;
  const bool ieee = (hp.flags & GX_HP_IEEE_EDGE) != 0;

  for (;;) {
    if (tid == 0) s_task = atomicAdd(A.counter, 1);
    __syncthreads();
    const int qi = s_task;
    __syncthreads();
    if (qi >= A.ntasks) break;
    const int task_id = A.order[qi];
    const GxTask* __restrict__ Tp = A.plan.tasks + task_id;
    const int na = Tp->n, e_d = Tp->e_d, np = Tp->npairs, g = Tp->node;
    // gradient baseline: the loss is taken at the label the caller gives (the graph's predicted label, explain.py:102,129),
    // otherwise at label[graph] (explain.py:750-753)
    const int gt = hp.mode ? __ldg(A.grad_label + task_id) : Tp->gt_label;
    const bool has_const = (Tp->flags & 1) != 0;
    const int64_t node_off = Tp->node_off, rp_off = Tp->rp_off, edge_off = Tp->edge_off, pair_off = Tp->pair_off;
    if (tid == 0) sL = gx_make_layout_graph(na, e_d, np, d, HID, EMB, C, nwarps);
    __syncthreads();
    const int dp = sL.dp, D4 = dp / 4;
    const float nn = (float)Tp->n_norm * (float)Tp->n_norm;
    const float ent_over_nn = hp.c_ent / nn;
    float* const X = base + sL.X; float* const U = base + sL.U;
    float* const Yh1 = base + sL.Yh1; float* const Yh2 = base + sL.Yh2; float* const Yh3 = base + sL.Yh3;
    float* const q1 = base + sL.q; float* const q2 = q1 + na; float* const q3 = q2 + na;
    float* const dZ2 = base + sL.dZ2; float* const dZ3 = base + sL.dZ3; float* const a = base + sL.a;
    float* const W1s = base + sL.W1s; float* const W1t = base + sL.W1t; float* const W2s = base + sL.W2s;
    float* const W2t = base + sL.W2t; float* const W3s = base + sL.W3s; float* const W3t = base + sL.W3t;
    float* const bs = base + sL.bs; float* const cst = base + sL.cst; float* const emb = base + sL.emb; float* const dE = base + sL.dE;
    float* const sF = base + sL.sF; float* const Fm = base + sL.F; float* const mF = base + sL.mF; float* const vF = base + sL.vF;
    float* const gFp = base + sL.gFp; float* const zs = base + sL.zs + warp * 128; float* const logit = base + sL.logit;
    int* const arg = reinterpret_cast<int*>(base + sL.arg);
    IdxT* const icol = reinterpret_cast<IdxT*>(base + sL.icol); IdxT* const irp = reinterpret_cast<IdxT*>(base + sL.irp);
    IdxT* const pi = reinterpret_cast<IdxT*>(base + sL.pi); IdxT* const pj = reinterpret_cast<IdxT*>(base + sL.pj);
    IdxT* const ppij = reinterpret_cast<IdxT*>(base + sL.ppij); IdxT* const ppji = reinterpret_cast<IdxT*>(base + sL.ppji);
    float2* const MM = reinterpret_cast<float2*>(A.pws + (int64_t)blockIdx.x * A.pws_stride_words);
    float2* const mm = MM + np; float2* const vv = mm + np; float2* const SS = vv + np;
    const bool wp_smem = C * (PD + 1) <= GX_WP_SMEM_MAX;
    const float* const Wpp = wp_smem ? base + sL.Wp : m.Wp;
    const float* const bpp = wp_smem ? base + sL.Wp + C * PD : m.bp;
    const int32_t* __restrict__ lo2gid = A.plan.lo2gid + node_off;

    // ------------------------------------------------------------------ load
    for (int idx = tid; idx < na * dp; idx += nthreads) {
      const int i = idx / dp, f = idx - i * dp;
      X[idx] = f < d ? __ldg(A.gb.feat + ((int64_t)g * A.gb.max_nodes + lo2gid[i]) * d + f) : 0.f;
    }
    for (int idx = tid; idx < dp * HS; idx += nthreads) { const int f = idx / HS, c = idx - f * HS; W1s[idx] = f < d ? __ldg(m.W[0] + f * HID + c) : 0.f; }
    for (int idx = tid; idx < HID * dp; idx += nthreads) { const int c = idx / dp, f = idx - c * dp; W1t[idx] = f < d ? __ldg(m.Wt[0] + c * d + f) : 0.f; }
    for (int idx = tid; idx < HID * HID; idx += nthreads) { W2s[idx] = __ldg(m.W[1] + idx); W2t[idx] = __ldg(m.Wt[1] + idx); }
    for (int idx = tid; idx < HID * EMB; idx += nthreads) { W3s[idx] = __ldg(m.W[2] + idx); W3t[idx] = __ldg(m.Wt[2] + idx); }
    for (int idx = tid; idx < HID; idx += nthreads) { bs[idx] = __ldg(m.b[0] + idx); bs[HID + idx] = __ldg(m.b[1] + idx); }
    for (int idx = tid; idx < EMB; idx += nthreads) bs[2 * HID + idx] = __ldg(m.b[2] + idx);
    if (wp_smem) {
      float* const Wps = base + sL.Wp;
      for (int idx = tid; idx < C * PD; idx += nthreads) Wps[idx] = __ldg(m.Wp + idx);
      for (int idx = tid; idx < C; idx += nthreads) Wps[C * PD + idx] = __ldg(m.bp + idx);
    }
    for (int e = tid; e < e_d; e += nthreads) icol[e] = (IdxT)A.plan.icol[edge_off + e];
    for (int i = tid; i <= na; i += nthreads) irp[i] = (IdxT)A.plan.irowptr[rp_off + i];
    const bool resume = hp.init == GX_INIT_STATE;   // optimiser state supplied by the caller (gx_explain_io)
    for (int f = tid; f < dp; f += nthreads) {
      sF[f] = hp.mode ? 1.0f : 0.5f;   // sigmoid(0) (explain.py:633-643); gradient baseline: unmasked features
      Fm[f] = 0.f; mF[f] = 0.f; vF[f] = 0.f;
      if (resume && A.x.feat_state_in != nullptr && f < d) {
        const float* fs = A.x.feat_state_in + (int64_t)task_id * 3 * d;
        Fm[f] = fs[f]; mF[f] = fs[d + f]; vF[f] = fs[2 * d + f];
        sF[f] = sigmoid_f(fs[f]);
      }
      if (hp.out_iter == 0 && f < d) {
        if (A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = sF[f];
        if (A.x.feat_state_out != nullptr) {
          float* fo = A.x.feat_state_out + (int64_t)task_id * 3 * d;
          fo[f] = Fm[f]; fo[d + f] = mF[f]; fo[2 * d + f] = vF[f];
        }
      }
    }
    const float m0_std = sqrtf(2.0f / (float)Tp->n_norm);
    for (int p = tid; p < np; p += nthreads) {
      const int i = A.plan.pair_i[pair_off + p], j = A.plan.pair_j[pair_off + p];
      const int pij = A.plan.pair_pij[pair_off + p], pji = A.plan.pair_pji[pair_off + p];
      const int oij = A.plan.pair_oij[pair_off + p], oji = A.plan.pair_oji[pair_off + p];
      pi[p] = (IdxT)i; pj[p] = (IdxT)j; ppij[p] = (IdxT)pij; ppji[p] = (IdxT)pji;
      if (hp.mode) { a[pij] = 1.0f; a[pji] = 1.0f; continue; }   // gradient baseline: the adjacency itself, no mask parameters
      float Mi, Mj;
      if (hp.init != GX_INIT_PHILOX) { Mi = __ldg(A.m0 + edge_off + oij); Mj = __ldg(A.m0 + edge_off + oji); }
      else {
        Mi = 1.0f + m0_std * philox_normal(hp.seed, (uint32_t)g, (uint32_t)oij);
        Mj = 1.0f + m0_std * philox_normal(hp.seed, (uint32_t)g, (uint32_t)oji);
      }
      float2 m2 = make_float2(0.f, 0.f), v2 = m2;
      if (resume) {
        m2 = make_float2(__ldg(A.x.adam_m_in + edge_off + oij), __ldg(A.x.adam_m_in + edge_off + oji));
        v2 = make_float2(__ldg(A.x.adam_v_in + edge_off + oij), __ldg(A.x.adam_v_in + edge_off + oji));
      }
      MM[p] = make_float2(Mi, Mj); mm[p] = m2; vv[p] = v2;
      // a resumed state came out of the edge phase: same sigmoid as there, so that a split run equals the straight one bit for bit
      const float Si = resume ? sigmoid_fast(Mi, ieee) : sigmoid_f(Mi), Sj = resume ? sigmoid_fast(Mj, ieee) : sigmoid_f(Mj);
      SS[p] = make_float2(Si, Sj);
      const float a0 = 0.5f * (Si + Sj);
      a[pij] = a0; a[pji] = a0;
      if (hp.out_iter == 0) {
        A.out_mask[edge_off + oij] = a0; A.out_mask[edge_off + oji] = a0;
        if (A.x.mask_param_out != nullptr) { A.x.mask_param_out[edge_off + oij] = Mi; A.x.mask_param_out[edge_off + oji] = Mj; }
        if (A.x.adam_m_out != nullptr) { A.x.adam_m_out[edge_off + oij] = m2.x; A.x.adam_m_out[edge_off + oji] = m2.y; }
        if (A.x.adam_v_out != nullptr) { A.x.adam_v_out[edge_off + oij] = v2.x; A.x.adam_v_out[edge_off + oji] = v2.y; }
      }
    }
    __syncthreads();
    // embedding of a row without edges: Y = 0 W + b -> normalize(b_l) (-> ReLU for l < 3), independent of the masks
    if (warp == 0) {
      for (int l = 0; l < 3; ++l) {
        const int w = l < 2 ? HID : EMB;
        const float bv = lane < w ? bs[l * HID + lane] : 0.f;
        const float qn = fmaxf(sqrtf(warp_sum(bv * bv)), 1e-12f);
        const float v = bv / qn;
        if (lane < w) cst[l * HID + lane] = l < 2 ? fmaxf(v, 0.f) : v;
      }
    }
    __syncthreads();

    Grp G;
    {
      int gw = D4 > H4 ? D4 : H4;
      gw = gw > E4 ? gw : E4;
      G.GW = gw; G.epi = 32 / gw; G.lane = lane; G.grp = lane / gw; G.q = lane - G.grp * gw; G.gbase = G.grp * gw;
    }
    const int epi = G.epi, q = G.q;
    const int ntask = (na + epi - 1) / epi;

    for (int it = 1; it <= hp.iters; ++it) {
      // ---- forward: three layers over all rows with edges (models.py:269-305)
#pragma unroll 1
      for (int l = 0; l < 3; ++l) {
        const float* src = l == 0 ? X : (l == 1 ? Yh1 : Yh2);
        const int sstride = l == 0 ? dp : HS, W4 = l == 0 ? D4 : H4, O4 = l == 2 ? E4 : H4, ldw = l == 2 ? EMB : HS;
        const float* Wd = l == 0 ? W1s : (l == 1 ? W2s : W3s);
        float* Yo = l == 0 ? Yh1 : (l == 1 ? Yh2 : Yh3);
        float* qo = l == 0 ? q1 : (l == 1 ? q2 : q3);
#pragma unroll 1
        for (int t = warp; t < ntask; t += nwarps) {
          const int i = t * epi + G.grp;
          const bool act = G.grp < epi && i < na;
          float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
          if (act && q < W4) {
            const int r0 = irp[i], r1 = irp[i + 1];
            for (int e = r0; e < r1; ++e) {
              float4 v = ld4(src + (int)icol[e] * sstride + 4 * q);
              if (l > 0) v = relu4(v);
              fma4(z, a[e], v);
            }
            if (l == 0) {
              st4(U + i * dp + 4 * q, z);
              const float4 s4 = ld4(sF + 4 * q);
              z = make_float4(z.x * s4.x, z.y * s4.y, z.z * s4.z, z.w * s4.w);
            }
            st4(zs + lane * 4, z);
          }
          __syncwarp();
          float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
          if (act && q < O4) y = group_dense(zs + G.gbase * 4, W4, Wd, ldw, q, ld4(bs + l * HID + 4 * q));
          const float ss = group_sum(y.x * y.x + y.y * y.y + y.z * y.z + y.w * y.w, G);
          const float qn = fmaxf(sqrtf(ss), 1e-12f);
          const float rq = 1.0f / qn;
          if (act && q < O4) st4(Yo + i * HS + 4 * q, make_float4(y.x * rq, y.y * rq, y.z * rq, y.w * rq));
          if (act && q == 0) qo[i] = qn;
          __syncwarp();
        }
        __syncthreads();
      }
      // ---- readout (one warp): per-layer max over rows (+ the edge-less constant), Linear, softmax,
      //      dL/dlogits = p - onehot(label), dEmb = Wp^T g                     (models.py:283-314, explain.py:711,750-753)
      if (warp == 0) {
        for (int k = lane; k < PD; k += 32) {
          const int l = k < HID ? 0 : (k < 2 * HID ? 1 : 2);
          const int c = k - l * HID;
          const float* Y = l == 0 ? Yh1 : (l == 1 ? Yh2 : Yh3);
          float best = has_const ? cst[k] : -INFINITY;
          int bi = -1;
          for (int i = 0; i < na; ++i) {
            float v = Y[i * HS + c];
            if (l < 2) v = fmaxf(v, 0.f);
            if (v > best) { best = v; bi = i; }   // strict: first maximal row wins, like torch.max
          }
          emb[k] = best; arg[k] = bi;
        }
        __syncwarp();
        for (int c = 0; c < C; ++c) {
          float t = 0.f;
          for (int k = lane; k < PD; k += 32) t = fmaf(emb[k], Wpp[c * PD + k], t);
          t = warp_sum(t);
          if (lane == 0) logit[c] = t + bpp[c];
        }
        __syncwarp();
        float mx = -INFINITY;
        for (int c = lane; c < C; c += 32) mx = fmaxf(mx, logit[c]);
        mx = warp_max(mx);
        float se = 0.f;
        for (int c = lane; c < C; c += 32) se += expf(logit[c] - mx);
        se = warp_sum(se);
        __syncwarp();
        int lbl = gt;
        if (lbl < 0) {   // gradient baseline without a label: the model's own prediction, first maximum (np.argmax)
          lbl = 0;
          for (int c = 1; c < C; ++c) lbl = logit[c] > logit[lbl] ? c : lbl;
          __syncwarp();   // every lane has read the logits before they are overwritten below
        }
        if (kTrace) {
          float* const tr = s_tr + (NT / 32) * 4;
          if (lane == 0) { const float lg = logit[gt]; tr[0] = -((lg - mx) - logf(se)); tr[1] = expf(lg - mx) / se; }
          if (A.x.trace_pred != nullptr) {
            float* trp = A.x.trace_pred + ((int64_t)task_id * A.x.epochs + (it - 1)) * C;
            for (int c = lane; c < C; c += 32) trp[c] = expf(logit[c] - mx) / se;
          }
          float fs = 0.f;   // feat_size_loss = coeff * mean(sigmoid(feat_mask)) (explain.py:763-766)
          for (int f = lane; f < d; f += 32) fs += sF[f];
          fs = warp_sum(fs);
          if (lane == 0) tr[2] = hp.c_feat_size * fs / (float)d;
          __syncwarp();
        }
        for (int c = lane; c < C; c += 32) logit[c] = expf(logit[c] - mx) / se - (c == lbl ? 1.f : 0.f);
        __syncwarp();
        for (int k = lane; k < PD; k += 32) {
          float t = 0.f;
          for (int c = 0; c < C; ++c) t = fmaf(logit[c], Wpp[c * PD + k], t);
          dE[k] = t;
        }
      }
      __syncthreads();
      // ---- backward: layers 3, 2, 1 over all rows with edges
      float4 gacc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
      for (int l = 2; l >= 0; --l) {
        const float* Yb = l == 0 ? Yh1 : (l == 1 ? Yh2 : Yh3);
        const float* qb = l == 0 ? q1 : (l == 1 ? q2 : q3);
        const float* gsrc = l == 1 ? dZ3 : dZ2;                                  // upstream dZ_{l+2} (unused for l == 2)
        const float* Wd = l == 0 ? W1t : (l == 1 ? W2t : W3t);
        const int B4 = l == 2 ? E4 : H4, O4 = l == 0 ? D4 : H4, ldw = l == 0 ? dp : HID;
        float* Zo = l == 0 ? U : (l == 1 ? dZ2 : dZ3);
        const int ostride = l == 0 ? dp : HS;
#pragma unroll 1
        for (int t = warp; t < ntask; t += nwarps) {
          const int i = t * epi + G.grp;
          const bool act = G.grp < epi && i < na;
          float4 z = make_float4(0.f, 0.f, 0.f, 0.f), yh = z;
          if (act && q < B4) {
            if (l < 2) {                       // dH_l = A_m^T dZ_{l+1}  (A_m symmetric)
              const int r0 = irp[i], r1 = irp[i + 1];
              for (int e = r0; e < r1; ++e) fma4(z, a[e], ld4(gsrc + (int)icol[e] * HS + 4 * q));
            }
            const int k0 = l * HID + 4 * q;    // dEmb routed to the arg-max rows
            if (arg[k0] == i) z.x += dE[k0];
            if (arg[k0 + 1] == i) z.y += dE[k0 + 1];
            if (arg[k0 + 2] == i) z.z += dE[k0 + 2];
            if (arg[k0 + 3] == i) z.w += dE[k0 + 3];
            yh = ld4(Yb + i * HS + 4 * q);
            if (l < 2) {                       // relu backward (no ReLU after the last layer)
              z.x = yh.x > 0.f ? z.x : 0.f; z.y = yh.y > 0.f ? z.y : 0.f;
              z.z = yh.z > 0.f ? z.z : 0.f; z.w = yh.w > 0.f ? z.w : 0.f;
            }
          }
          const float sdot = group_sum(yh.x * z.x + yh.y * z.y + yh.z * z.z + yh.w * z.w, G);
          if (act && q < B4) {
            const float rq = 1.0f / qb[i];
            st4(zs + lane * 4, make_float4((z.x - yh.x * sdot) * rq, (z.y - yh.y * sdot) * rq,
                                           (z.z - yh.z * sdot) * rq, (z.w - yh.w * sdot) * rq));
          }
          __syncwarp();
          if (act && q < O4) {
            float4 o = group_dense(zs + G.gbase * 4, B4, Wd, ldw, q, make_float4(0.f, 0.f, 0.f, 0.f));
            if (l == 0) {
              const float4 u = ld4(U + i * dp + 4 * q);
              const float4 s4 = ld4(sF + 4 * q);
              gacc.x = fmaf(o.x, u.x, gacc.x); gacc.y = fmaf(o.y, u.y, gacc.y);
              gacc.z = fmaf(o.z, u.z, gacc.z); gacc.w = fmaf(o.w, u.w, gacc.w);
              o = make_float4(o.x * s4.x, o.y * s4.y, o.z * s4.z, o.w * s4.w);
            }
            st4(Zo + i * ostride + 4 * q, o);
          }
          __syncwarp();
        }
        if (l == 0) {
          st4(zs + lane * 4, gacc);
          __syncwarp();
          if (G.grp == 0 && q < D4) {
            float4 tsum = gacc;
            for (int g2 = 1; g2 < epi; ++g2) {
              const float4 o = ld4(zs + (g2 * G.GW + q) * 4);
              tsum.x += o.x; tsum.y += o.y; tsum.z += o.z; tsum.w += o.w;
            }
            st4(gFp + warp * dp + 4 * q, tsum);
          }
          __syncwarp();
        }
        __syncthreads();
      }
      // ---- edge phase: every edge sees all three layers; no Laplacian term in graph mode (explain.py:787-788)
      if (hp.mode) {
        // gradient baseline (explain.py:128-133): mask_ij = sigmoid(|dL/dA_ij| + |dL/dA_ji|) on both slots, no regulariser, no update
        for (int p = tid; p < np; p += nthreads) {
          const int i = pi[p], j = pj[p];
          const float gij = dot_v4(U + i * dp, X + j * dp, D4) + dot_relu_v4(dZ2 + i * HS, Yh1 + j * HS, H4)
                          + dot_relu_v4(dZ3 + i * HS, Yh2 + j * HS, H4);
          const float gji = dot_v4(U + j * dp, X + i * dp, D4) + dot_relu_v4(dZ2 + j * HS, Yh1 + i * HS, H4)
                          + dot_relu_v4(dZ3 + j * HS, Yh2 + i * HS, H4);
          const float an = sigmoid_f(fabsf(gij) + fabsf(gji));
          A.out_mask[edge_off + A.plan.pair_oij[pair_off + p]] = an;
          A.out_mask[edge_off + A.plan.pair_oji[pair_off + p]] = an;
        }
      } else {
        const float2 tab = __ldg(hp.adam_tab + (it - 1));
        const float step = tab.x, bc2s = tab.y, bc2s_inv = 1.0f / tab.y;
        const bool last = (it == hp.out_iter);   // the mask built after this update is the one the reference returns
        for (int f = tid; f < d; f += nthreads) {
          float gsum = 0.f;
          for (int w = 0; w < nwarps; ++w) gsum += gFp[w * dp + f];
          const float s = sF[f];
          const float gg = s * (1.f - s) * (gsum + hp.c_feat_size / (float)d);
          float mf = mF[f], vf = vF[f], Fv = Fm[f];
          mf = mf + (gg - mf) * hp.one_minus_b1;
          vf = vf * hp.b2 + hp.one_minus_b2 * gg * gg;
          Fv = Fv - step * (mf / (sqrtf(vf) / bc2s + hp.eps));
          mF[f] = mf; vF[f] = vf; Fm[f] = Fv;
          const float sn = sigmoid_f(Fv);
          sF[f] = sn;
          if (last) {
            if (A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = sn;
            if (A.x.feat_state_out != nullptr) {
              float* fo = A.x.feat_state_out + (int64_t)task_id * 3 * d;
              fo[f] = Fv; fo[d + f] = mf; fo[2 * d + f] = vf;
            }
          }
        }
        float trS = 0.f, trH = 0.f, trD = 0.f;   // trace: this thread's share of sum S, sum H(S), sum 2a' (no Laplacian term in graph mode)
        for (int p = tid; p < np; p += nthreads) {
          const int i = pi[p], j = pj[p];
          float Gd = dot_v4(U + i * dp, X + j * dp, D4) + dot_v4(U + j * dp, X + i * dp, D4);
          Gd += dot_relu_v4(dZ2 + i * HS, Yh1 + j * HS, H4) + dot_relu_v4(dZ2 + j * HS, Yh1 + i * HS, H4);
          Gd += dot_relu_v4(dZ3 + i * HS, Yh2 + j * HS, H4) + dot_relu_v4(dZ3 + j * HS, Yh2 + i * HS, H4);
          Gd *= 0.5f;
          float2 Mv = MM[p];
          const float2 Sv = SS[p];
          if (kTrace) { trS += Sv.x + Sv.y; trH += bern_entropy(Sv.x) + bern_entropy(Sv.y); }
          const float gi = Sv.x * (1.f - Sv.x) * (Gd + hp.c_size - ent_over_nn * Mv.x);
          const float gj = Sv.y * (1.f - Sv.y) * (Gd + hp.c_size - ent_over_nn * Mv.y);
          float2 m2 = mm[p], v2 = vv[p];
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
          a[ppij[p]] = an; a[ppji[p]] = an;
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
          trS = warp_sum(trS); trH = warp_sum(trH); trD = warp_sum(trD);
          if (lane == 0) { s_tr[warp * 4 + 0] = trS; s_tr[warp * 4 + 1] = trH; s_tr[warp * 4 + 2] = 0.f; s_tr[warp * 4 + 3] = trD; }
        }
      }
      __syncthreads();
      if (kTrace && tid == 0) {   // raw terms of epoch it-1 (trace_finalize_kernel assembles the columns)
        float sS = 0.f, sH = 0.f, sD = 0.f;
        for (int w = 0; w < nwarps; ++w) { sS += s_tr[w * 4]; sH += s_tr[w * 4 + 1]; sD += s_tr[w * 4 + 3]; }
        float* row = A.x.trace + ((int64_t)task_id * A.x.epochs + (it - 1)) * GX_TRACE_COLS;
        const float* const tr = s_tr + (NT / 32) * 4;
        row[0] = sS; row[1] = tr[0]; row[2] = sH; row[3] = 0.f; row[4] = sD; row[5] = tr[2]; row[6] = 0.f; row[7] = tr[1];
      }
    }
    __syncthreads();
  }
  (void)kNone;
}

}  // namespace

cudaError_t gx_launch_graph_plan(const GxGraphBatchDev& gb, int count, GxPlanArrays plan, cudaStream_t s) {
  const int grid = count < GX_GRID_CAP ? count : GX_GRID_CAP;
  const size_t smem = (size_t)(2 * gb.max_nodes + 2) * sizeof(int);
  graph_plan_kernel<<<grid, 128, smem, s>>>(gb, count, plan);
  return cudaGetLastError();
}

cudaError_t gx_launch_explain_graphs(const GxExplainLaunch& cfg, const GxGraphBatchDev& gb, const GxModelDev& m,
                                     const GxHparamsDev& hp, const GxPlanArrays& plan, const float* m0, float* out_mask,
                                     float* out_feat, const int32_t* grad_label, cudaStream_t s) {
  GraphArgs args;
  fill_queue_args(args, cfg, m, hp, plan, m0, out_mask, out_feat);
  args.gb = gb; args.x = cfg.x; args.grad_label = grad_label;
  const bool tr = cfg.x.trace != nullptr;
  auto launch = [&](auto kern) -> cudaError_t {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, cfg.smem_bytes);
    if (e != cudaSuccess) return e;
    // every launch class asks for the largest shared-memory carveout: CTAs of different classes (= different kernels / footprints) can then
    // share an SM; with per-kernel carveouts a CTA waits for an SM that is completely idle
    e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return e;
    kern<<<cfg.grid, cfg.threads, cfg.smem_bytes, s>>>(args);
    return cudaGetLastError();
  };
  if (m.hid == 20 && m.emb == 20) return tr ? launch(explain_graph_kernel<20, 20, 128, true>) : launch(explain_graph_kernel<20, 20, 128, false>);
  if (m.hid == 32 && m.emb == 32)   // widths <= 32, zero-padded
    return tr ? launch(explain_graph_kernel<32, 32, 128, true>) : launch(explain_graph_kernel<32, 32, 128, false>);
  return cudaErrorInvalidValue;
}
