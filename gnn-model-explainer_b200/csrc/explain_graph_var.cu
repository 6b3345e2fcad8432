// explain_graph_var.cu -- graph-classification mode for the model and optimiser VARIANTS: the graph-mode counterpart of explain_var.cu.
//
// Replaces Explainer.explain(node_idx=0, graph_idx=g, graph_mode=True) (explain.py:80-85,137-146,209-211; loss :740-808 with
// lap_loss = 0) on a GcnEncoderGraph (models.py:269-316) with num_gc_layers = 2 / 3 / 4, --bn, hidden / output widths up to 128,
// and the optimisers of utils/train_utils.py:7-23 (Adam, SGD momentum 0.95, RMSprop, Adagrad; step / cos schedulers).  The tuned
// graph kernel (explain_graph.cu) keeps the default model with Adam.
//
// Semantics (as in explain_graph.cu, generalised to L layers):
//   * layer l = normalize((A_m H_{l-1}) W_l + b_l); every layer but the last applies ReLU and, with --bn, a fresh BatchNorm1d(max_nodes)
//     in train mode (a per-row standardisation over the feature axis);
//   * no receptive-field pruning: every row with at least one edge is computed at every layer; rows WITHOUT an edge (padding,
//     isolated nodes) all hold one per-layer constant, bn(relu(normalize(b_l))) / normalize(b_L), independent of the masks -- it joins
//     every max-pool and never carries gradient to M or F;
//   * readout = per-layer column max over the padded rows (the constant first, then the rows in ascending order; the first maximum
//     takes the gradient), concatenation, Linear, softmax, -log p[graph label];
//   * every edge gets SDDMM terms from all L layers; the 1/n^2 of the entropy term and the std of M0 use the PADDED size.
// Layout and parallelisation as explain_var.cu: one persistent CTA per graph, the graph's state in a per-CTA global slab that stays
// in L2 (GxGraphVarLayout), one warp per row with lane = feature, one thread per undirected edge in the edge phase.
// Phases per epoch (one __syncthreads each): F1 .. FL | pool | S | BL .. B1 | P.
#include "explain_var_common.cuh"

namespace {

struct GraphVarArgs {
  const int32_t* order;
  int32_t ntasks;
  int32_t* counter;
  float* gws;
  int64_t gws_stride_words;
  float* pws;
  int64_t pws_stride_words;
  GxGraphBatchDev gb;
  GxModelDev m;
  GxHparamsDev hp;
  GxPlanArrays plan;
  const float* m0;
  float* out_mask;
  float* out_feat;
};

// shared memory: explain_var.cu's carve-up + the edge-less rows' constant embedding and the arg-max row of every pooled feature
struct GraphVarSmem { VarSmem S; int cst, arg, total; };
__host__ __device__ inline GraphVarSmem graph_var_smem(int d, int L, int hid, int emb, int C, int nwarps) {
  GraphVarSmem G;
  G.S = var_smem(d, L, hid, emb, C, nwarps);
  const int PD = hid * (L - 1) + emb;
  G.cst = G.S.total;
  G.arg = G.cst + gx_round_up(PD, 4);
  G.total = G.arg + gx_round_up(PD, 4);
  return G;
}

template <bool kBn, int KW>
__global__ void __launch_bounds__(kVarThreads, KW == 1 && !kBn ? 2 : 1) explain_graph_var_kernel(const GraphVarArgs A) {
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
  const GraphVarSmem GS = graph_var_smem(d, L, hid, embw, C, nwarps);
  const VarSmem& S = GS.S;
  float* const sF = sm + S.sF; float* const Fm = sm + S.F; float* const mF = sm + S.mF; float* const vF = sm + S.vF;
  float* const zs = sm + S.zs + warp * S.zlen;
  float* const gFp = sm + S.gFp;
  float* const emb = sm + S.emb; float* const dEmb = sm + S.dEmb; float* const logit = sm + S.logit;
  float* const cst = sm + GS.cst;
  int* const arg = reinterpret_cast<int*>(sm + GS.arg);
  const bool wp_smem = C * (PD + 1) <= GX_WP_SMEM_MAX;
  const float* const Wpp = wp_smem ? sm + S.Wp : m.Wp;
  const float* const bpp = wp_smem ? sm + S.Wp + C * PD : m.bp;
  auto win_of = [&](int l) { return l == 0 ? d : hid; };            // l = 0 .. L-1
  auto wout_of = [&](int l) { return l == L - 1 ? embw : hid; };

  const float* Wl[GX_MAX_LAYERS];   // conv weights: shared memory when they fit, else global (L2 resident)
  var_stage_model(m, S, sm, Wl, tid, NT);
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
  float* const slab = A.gws + (int64_t)blockIdx.x * A.gws_stride_words;
  float2* const MM = reinterpret_cast<float2*>(A.pws + (int64_t)blockIdx.x * A.pws_stride_words);

  for (;;) {
    __syncthreads();
    if (tid == 0) s_task = atomicAdd(A.counter, 1);
    __syncthreads();
    const int qi = s_task;
    if (qi >= A.ntasks) break;
    const int task_id = A.order[qi];
    const GxTask* __restrict__ Tp = A.plan.tasks + task_id;
    const int na = Tp->n, e_d = Tp->e_d, np = Tp->npairs, gt = Tp->gt_label, g = Tp->node;
    const bool has_const = (Tp->flags & 1) != 0;
    const int64_t node_off = Tp->node_off, rp_off = Tp->rp_off, edge_off = Tp->edge_off, pair_off = Tp->pair_off;
    const GxGraphVarLayout Lo = gx_make_graph_var_layout(na, e_d, d, L, VW);
    const float* const feat = A.gb.feat + (int64_t)g * A.gb.max_nodes * d;   // this graph's padded feature rows
    const int32_t* __restrict__ lo2gid = A.plan.lo2gid + node_off;
    const int32_t* __restrict__ irp = A.plan.irowptr + rp_off;
    const int32_t* __restrict__ icol = A.plan.icol + edge_off;
    const int32_t* __restrict__ pi = A.plan.pair_i + pair_off; const int32_t* __restrict__ pj = A.plan.pair_j + pair_off;
    const int32_t* __restrict__ ppij = A.plan.pair_pij + pair_off; const int32_t* __restrict__ ppji = A.plan.pair_pji + pair_off;
    const int32_t* __restrict__ poij = A.plan.pair_oij + pair_off; const int32_t* __restrict__ poji = A.plan.pair_oji + pair_off;
    float* const a = slab + Lo.a; float* const U = slab + Lo.U; float* const dZ1 = slab + Lo.dZ1;
    auto Yh = [&](int l) { return slab + Lo.Yh + (int64_t)(l - 1) * na * VW; };     // l = 1..L: normalised pre-activation
    auto Hh = [&](int l) { return slab + Lo.H + (int64_t)(l - 1) * na * VW; };      // l = 1..L: what the next layer / the max-pool sees
    auto dZ = [&](int l) { return slab + Lo.dZ + (int64_t)(l - 2) * na * VW; };     // l = 2..L: dL/d(A_m H_{l-1}) (width hid)
    auto qn = [&](int l) { return slab + Lo.q + (int64_t)(l - 1) * na; };
    auto istd = [&](int l) { return slab + Lo.istd + (int64_t)(l - 1) * na; };
    float2* const mm = MM + np; float2* const vv = mm + np; float2* const SS = vv + np;
    const float nn = (float)Tp->n_norm * (float)Tp->n_norm;
    const float ent_over_nn = hp.c_ent / nn;

    for (int f = tid; f < dp; f += NT) {
      sF[f] = 0.5f; Fm[f] = 0.f; mF[f] = 0.f; vF[f] = 0.f;   // feat_mask = 0 (explain.py:633-643)
      if (hp.out_iter == 0 && f < d && A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = 0.5f;
    }
    {
      const float m0_std = sqrtf(2.0f / (float)Tp->n_norm);   // gain('relu') * sqrt(2/(n+n)), n = the padded size
      for (int p = tid; p < np; p += NT) {
        const int oij = poij[p], oji = poji[p];
        const float Mi = var_init_param(hp, A.m0, edge_off + oij, (uint32_t)g, (uint32_t)oij, m0_std);
        const float Mj = var_init_param(hp, A.m0, edge_off + oji, (uint32_t)g, (uint32_t)oji, m0_std);
        MM[p] = make_float2(Mi, Mj);
        mm[p] = make_float2(0.f, 0.f);
        vv[p] = make_float2(0.f, 0.f);
        const float Si = sigmoid_f(Mi), Sj = sigmoid_f(Mj);
        SS[p] = make_float2(Si, Sj);
        const float a0 = 0.5f * (Si + Sj);  // explain.py:665-678
        a[ppij[p]] = a0; a[ppji[p]] = a0;
        if (hp.out_iter == 0) { A.out_mask[edge_off + oij] = a0; A.out_mask[edge_off + oji] = a0; }
      }
    }
    __syncthreads();

    for (int it = 1; it <= hp.iters; ++it) {
      // ---------------------------------------------------------------- forward, layer by layer, every row with an edge
      for (int l = 1; l <= L; ++l) {
        const int win = win_of(l - 1), wout = wout_of(l - 1);
        const float* const Ws = Wl[l - 1]; const float* const bsm = sm + S.b[l - 1];
        for (int i = warp; i < na; i += nwarps) {
          const int r0 = irp[i], r1 = irp[i + 1];
          if (l == 1) var_gather_feat(r0, r1, icol, a, feat, lo2gid, d, sF, U + (int64_t)i * dp, zs, lane);
          else var_gather_hidden<KW>(r0, r1, icol, a, Hh(l - 1), win, zs, lane);
          __syncwarp();
          float y[KW];
          var_dense<KW>(zs, win, Ws, wout, bsm, y, lane);
          __syncwarp();
          float yh[KW], h[KW], is = 1.f;
          const float q = var_activate<kBn, KW>(y, wout, l < L, yh, h, &is, lane);
          if (kBn && l < L && lane == 0) istd(l)[i] = is;
#pragma unroll
          for (int k = 0; k < KW; ++k) {
            Yh(l)[(int64_t)i * VW + lane + 32 * k] = yh[k];
            Hh(l)[(int64_t)i * VW + lane + 32 * k] = lane + 32 * k < wout ? h[k] : 0.f;
          }
          if (lane == 0) qn(l)[i] = q;
        }
        __syncthreads();
      }
      // ---------------------------------------------------------------- max-pool of every layer (models.py:283,291,300)
      for (int k = tid; k < PD; k += NT) {
        const int l = k < hid * (L - 1) ? k / hid + 1 : L;
        const int c = k - hid * (l - 1);
        const float* const H = Hh(l);
        float best = has_const ? cst[k] : -INFINITY;
        int bi = -1;
        for (int i = 0; i < na; ++i) {
          const float v = H[(int64_t)i * VW + c];
          if (v > best) { best = v; bi = i; }   // strict: the first maximal row wins, like torch.max
        }
        emb[k] = best; arg[k] = bi;
      }
      __syncthreads();
      // ---------------------------------------------------------------- S: Linear, softmax, dEmb   (models.py:305-314, explain.py:711)
      if (warp == 0) var_readout_tail(emb, Wpp, bpp, C, PD, gt, logit, dEmb, lane);
      for (int idx = tid; idx < nwarps * dp; idx += NT) gFp[idx] = 0.f;
      __syncthreads();
      // ---------------------------------------------------------------- backward, layer by layer
      for (int l = L; l >= 1; --l) {
        const int win = win_of(l - 1), wout = wout_of(l - 1);
        const float* const Ws = Wl[l - 1];
        const int koff = hid * (l - 1);
        for (int i = warp; i < na; i += nwarps) {
          // dL/dH_l[i] = (A_m^T dZ_{l+1})[i] + the share of the pooled features whose arg-max is row i
          float g[KW], yh[KW];
#pragma unroll
          for (int k = 0; k < KW; ++k) g[k] = 0.f;
          if (l < L) var_gather_back<KW>(irp[i], irp[i + 1], icol, a, dZ(l + 1), wout, na, g, lane);
#pragma unroll
          for (int k = 0; k < KW; ++k) {
            const int c = lane + 32 * k;
            if (c < wout && arg[koff + c] == i) g[k] += dEmb[koff + c];
            yh[k] = Yh(l)[(int64_t)i * VW + c];
          }
          if (l < L) var_hidden_backward<kBn, KW>(g, yh, Hh(l) + (int64_t)i * VW, kBn ? istd(l)[i] : 1.f, wout, lane);
          const float sdot = var_norm_dot<KW>(g, yh, wout, lane);
          const float qi = qn(l)[i];
          __syncwarp();
          var_norm_backward<KW>(g, yh, sdot, qi, wout, zs, lane);   // dY: backward of y / max(|y|, eps)
          __syncwarp();
          if (l == 1) var_first_layer_dz(zs, Ws, d, wout, U + (int64_t)i * dp, sF, gFp + warp * dp, dZ1 + (int64_t)i * dp, lane);
          else var_hidden_dz<KW>(zs, Ws, win, wout, dZ(l) + (int64_t)i * VW, lane);
          __syncwarp();
        }
        __syncthreads();
      }
      // ---------------------------------------------------------------- P: edge gradients, regularisers, optimiser step, next mask
      {
        const float2 tab = __ldg(hp.adam_tab + (it - 1));
        const float step = tab.x, bc2s = tab.y, bc2s_inv = 1.0f / tab.y;
        const bool last = (it == hp.out_iter);   // the mask built after this update is the one the reference returns
        for (int f = tid; f < d; f += NT) {
          float gsum = 0.f;
          for (int w = 0; w < nwarps; ++w) gsum += gFp[w * dp + f];
          const float s = sF[f];
          const float gg = s * (1.f - s) * (gsum + hp.c_feat_size / (float)d);
          float mf = mF[f], vf = vF[f], Fv = Fm[f];
          var_feat_update(hp, gg, Fv, mf, vf, step, bc2s);
          mF[f] = mf; vF[f] = vf; Fm[f] = Fv;
          const float sn = sigmoid_f(Fv);
          sF[f] = sn;   // (the edge dots below use dZ1 (.) sF stored in the backward, not this value)
          if (last && A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = sn;
        }
        for (int p = tid; p < np; p += NT) {
          const int i = pi[p], j = pj[p];
          float Gd = 0.f;   // no Laplacian term in graph mode (explain.py:787-788)
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
          a[ppij[p]] = an; a[ppji[p]] = an;
          if (last) { A.out_mask[edge_off + poij[p]] = an; A.out_mask[edge_off + poji[p]] = an; }
        }
      }
      __syncthreads();
    }
  }
}

// calls f(kernel) with the instantiation for the model
template <typename F>
cudaError_t with_graph_var_kernel(const GxModelDev& m, F&& f) {
  const int kw = var_kw(m.hid, m.emb);
  if (m.bn) {
    if (kw == 1) return f(explain_graph_var_kernel<true, 1>);
    if (kw == 2) return f(explain_graph_var_kernel<true, 2>);
    return f(explain_graph_var_kernel<true, 4>);
  }
  if (kw == 1) return f(explain_graph_var_kernel<false, 1>);
  if (kw == 2) return f(explain_graph_var_kernel<false, 2>);
  return f(explain_graph_var_kernel<false, 4>);
}

}  // namespace

int gx_graph_var_smem_bytes(int d, int L, int hid, int emb, int C) { return graph_var_smem(d, L, hid, emb, C, kVarThreads / 32).total * 4; }

// co-resident CTAs per SM of the model's instantiation (sizes the persistent grid); 0 on error
int gx_graph_var_ctas_per_sm(const GxModelDev& m) {
  const int bytes = gx_graph_var_smem_bytes(m.d, m.L, m.hid, m.emb, m.C);
  int n = 0;
  const cudaError_t e = with_graph_var_kernel(m, [&](auto kern) -> cudaError_t {
    cudaError_t r = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (r != cudaSuccess) return r;
    r = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (r != cudaSuccess) return r;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, kVarThreads, bytes);
  });
  return e == cudaSuccess ? n : 0;
}

cudaError_t gx_launch_explain_graph_var(const GxExplainLaunch& cfg, const GxGraphBatchDev& gb, const GxModelDev& m,
                                        const GxHparamsDev& hp, const GxPlanArrays& plan, const float* m0, float* out_mask,
                                        float* out_feat, cudaStream_t s) {
  GraphVarArgs args;
  fill_queue_args(args, cfg, m, hp, plan, m0, out_mask, out_feat);
  args.gb = gb; args.gws = cfg.gws; args.gws_stride_words = cfg.gws_stride_words;
  const int bytes = gx_graph_var_smem_bytes(m.d, m.L, m.hid, m.emb, m.C);
  return with_graph_var_kernel(m, [&](auto kern) -> cudaError_t {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return e;
    kern<<<cfg.grid, kVarThreads, bytes, s>>>(args);
    return cudaGetLastError();
  });
}
