// explain_var.cu -- K2v: the mask-optimisation kernel for the model VARIANTS of the reference (SURVEY 8 row f3):
//   num_gc_layers = 2 / 3 / 4 (explainer_main.py:57-66, explain.py:64: n_hops = num_gc_layers; models.py:193-220,230-267) and
//   --bn (models.py:222-228: a FRESH BatchNorm1d(n) in train mode on the (1, n, h) activations = per-node standardisation over
//   the feature axis, eps 1e-5, biased variance, applied after the ReLU of every hidden layer; the readout concatenates the
//   standardised activations, models.py:241-260).
// It computes exactly what oracle/kernel_spec.py specifies (parameters on the directed edges, layer l only on the rows within
// L - l hops of the explained node, inner / outer pair split), for hidden / output widths up to 128 (the tuned kernels stop at 32) and d <= 128.  These options are rare, so the
// kernel is written for clarity, not speed: one persistent CTA per task, state in a per-CTA global slab (L2 resident for the
// reference's graph sizes), one warp per row with lane = feature, one thread per undirected edge in the edge phase.
// Phases per epoch (one __syncthreads each): F1 .. FL | S | BL .. B1 | P.  The default model (3 layers, no bn) never comes here.
#include "explain_var_common.cuh"

namespace {

template <bool kBn, int KW>
__global__ void __launch_bounds__(kVarThreads) explain_var_kernel(const ExplainArgs A) {
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
  const VarSmem S = var_smem(d, L, hid, embw, C, nwarps);
  float* const sF = sm + S.sF; float* const Fm = sm + S.F; float* const mF = sm + S.mF; float* const vF = sm + S.vF;
  float* const zs = sm + S.zs + warp * S.zlen;
  float* const gFp = sm + S.gFp;
  float* const emb = sm + S.emb; float* const dEmb = sm + S.dEmb; float* const logit = sm + S.logit;
  const bool wp_smem = C * (PD + 1) <= GX_WP_SMEM_MAX;
  const float* const Wpp = wp_smem ? sm + S.Wp : m.Wp;
  const float* const bpp = wp_smem ? sm + S.Wp + C * PD : m.bp;
  auto win_of = [&](int l) { return l == 0 ? d : hid; };            // l = 0 .. L-1
  auto wout_of = [&](int l) { return l == L - 1 ? embw : hid; };

  const float* Wl[GX_MAX_LAYERS];   // conv weights: shared memory when they fit, else global (L2 resident)
  var_stage_model(m, S, sm, Wl, tid, NT);
  float* const slab = A.gws + (int64_t)blockIdx.x * A.gws_stride_words;
  float2* const MM0 = reinterpret_cast<float2*>(A.pws + (int64_t)blockIdx.x * A.pws_stride_words);

  for (;;) {
    __syncthreads();
    if (tid == 0) s_task = atomicAdd(A.counter, 1);
    __syncthreads();
    const int qi = s_task;
    if (qi >= A.ntasks) break;
    const int task_id = A.order[qi];
    const GxTask* __restrict__ Tp = A.plan.tasks + task_id;
    const int n = Tp->n, n2 = Tp->n2, e1 = Tp->e1, np = Tp->npairs_in;
    const int gt = Tp->gt_label;
    const int64_t node_off = Tp->node_off, rp_off = Tp->rp_off, edge_off = Tp->edge_off, pair_off = Tp->pair_off;
    int R[GX_MAX_LAYERS + 1];   // R[l] = rows of layer l (1-based): nodes within L - l hops; R[0] = n
    R[0] = n;
    for (int l = 1; l <= L; ++l) R[l] = Tp->cum[L - l] < n ? Tp->cum[L - l] : n;
    const GxVarLayout Lo = gx_make_var_layout(n, n2, e1, np, d, L, VW);
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
    float2* const MM = MM0; float2* const mm = MM + np; float2* const vv = mm + np; float2* const SS = vv + np;
    const float nn = (float)n * (float)n;
    const float ent_over_nn = hp.c_ent / nn;
    const float lap_over_nn = hp.c_lap / nn;

    for (int f = tid; f < dp; f += NT) {
      sF[f] = 0.5f; Fm[f] = 0.f; mF[f] = 0.f; vF[f] = 0.f;   // feat_mask = 0 (explain.py:633-643)
      if (hp.out_iter == 0 && f < d && A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = 0.5f;
    }
    {
      const float m0_std = sqrtf(2.0f / (float)n);  // gain('relu') * sqrt(2/(n+n)) (explain.py:647-651)
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
        if (i < n2) a[ppij[p]] = a0;
        if (j < n2) a[ppji[p]] = a0;
        const float yd = (float)__ldg(A.g.pred_label + lo2gid[i]) - (float)__ldg(A.g.pred_label + lo2gid[j]);
        lapg[p] = lap_over_nn * yd * yd;   // d/dA_ij + d/dA_ji of y^T (D - A) y / n^2 (explain.py:780-793)
        if (hp.out_iter == 0) { A.out_mask[edge_off + oij] = a0; A.out_mask[edge_off + oji] = a0; }
      }
    }
    __syncthreads();

    for (int it = 1; it <= hp.iters; ++it) {
      // ---------------------------------------------------------------- forward, layer by layer        (models.py:58-80,230-267)
      for (int l = 1; l <= L; ++l) {
        const int win = win_of(l - 1), wout = wout_of(l - 1);
        const float* const Ws = Wl[l - 1]; const float* const bsm = sm + S.b[l - 1];
        for (int i = warp; i < R[l]; i += nwarps) {
          const int r0 = irp[i], r1 = irp[i + 1];
          if (l == 1) var_gather_feat(r0, r1, icol, a, A.g.feat, lo2gid, d, sF, U + (int64_t)i * dp, zs, lane);
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
      // ---------------------------------------------------------------- S: readout of row r = level-order id 0, softmax, dEmb
      if (warp == 0) {
        for (int l = 1; l <= L; ++l)
          for (int c = lane; c < wout_of(l - 1); c += 32) emb[hid * (l - 1) + c] = Hh(l)[c];
        __syncwarp();
        var_readout_tail(emb, Wpp, bpp, C, PD, gt, logit, dEmb, lane);
      }
      for (int idx = tid; idx < nwarps * dp; idx += NT) gFp[idx] = 0.f;
      __syncthreads();
      // ---------------------------------------------------------------- backward, layer by layer
      for (int l = L; l >= 1; --l) {
        const int win = win_of(l - 1), wout = wout_of(l - 1);
        const float* const Ws = Wl[l - 1];
        for (int i = warp; i < R[l]; i += nwarps) {
          // dL/dH_l[i] = (A_m^T dZ_{l+1})[i] over the neighbours that are rows of layer l+1 (a prefix of row i) + the readout's share
          float g[KW], yh[KW];
#pragma unroll
          for (int k = 0; k < KW; ++k) g[k] = 0.f;
          if (l < L) var_gather_back<KW>(irp[i], irp[i + 1], icol, a, dZ(l + 1), wout, R[l + 1], g, lane);   // columns are partitioned by level
#pragma unroll
          for (int k = 0; k < KW; ++k) {
            if (i == 0 && lane + 32 * k < wout) g[k] += dEmb[hid * (l - 1) + lane + 32 * k];
            yh[k] = Yh(l)[(int64_t)i * VW + lane + 32 * k];
          }
          if (l < L) var_hidden_backward<kBn, KW>(g, yh, Hh(l) + (int64_t)i * VW, kBn ? istd(l)[i] : 1.f, wout, lane);
          const float sdot = var_norm_dot<KW>(g, yh, wout, lane);
          const float qi = qn(l)[i];
          __syncwarp();
          var_norm_backward<KW>(g, yh, sdot, qi, wout, zs, lane);   // dY: backward of y / max(|y|, eps)
          __syncwarp();
          // dZ[f] = sum_c dY[c] W[f][c]
          if (l == 1) var_first_layer_dz(zs, Ws, d, wout, U + (int64_t)i * dp, sF, gFp + warp * dp, dZ1 + (int64_t)i * dp, lane);
          else var_hidden_dz<KW>(zs, Ws, win, wout, dZ(l) + (int64_t)i * VW, lane);
          __syncwarp();
        }
        __syncthreads();
      }
      // ---------------------------------------------------------------- P: edge gradients, regularisers, Adam, next mask
      {
        const float2 tab = __ldg(hp.adam_tab + (it - 1));
        const float step = tab.x, bc2s = tab.y, bc2s_inv = 1.0f / tab.y;
        const bool last = (it == hp.out_iter);
        for (int f = tid; f < d; f += NT) {
          float gsum = 0.f;
          for (int w = 0; w < nwarps; ++w) gsum += gFp[w * dp + f];
          const float s = sF[f];
          const float g = s * (1.f - s) * (gsum + hp.c_feat_size / (float)d);
          float mf = mF[f], vf = vF[f], Fv = Fm[f];
          var_feat_update(hp, g, Fv, mf, vf, step, bc2s);
          mF[f] = mf; vF[f] = vf; Fm[f] = Fv;
          const float sn = sigmoid_f(Fv);
          sF[f] = sn;   // (the edge dots below use dZ1 (.) sF stored in the backward, not this value)
          if (last && A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = sn;
        }
        for (int p = tid; p < np; p += NT) {
          const int i = pi[p], j = pj[p];   // i < j in level order
          float Gd = lapg[p];
          if (i < R[1]) {
            float t = 0.f;
            const float* xr = A.g.feat + (int64_t)lo2gid[j] * d;
            for (int f = 0; f < d; ++f) t = fmaf(dZ1[(int64_t)i * dp + f], __ldg(xr + f), t);
            Gd += t;
          }
          if (j < R[1]) {
            float t = 0.f;
            const float* xr = A.g.feat + (int64_t)lo2gid[i] * d;
            for (int f = 0; f < d; ++f) t = fmaf(dZ1[(int64_t)j * dp + f], __ldg(xr + f), t);
            Gd += t;
          }
          for (int l = 2; l <= L; ++l) {
            const float* const dZl = dZ(l); const float* const Hp = Hh(l - 1);
            if (i < R[l]) { float t = 0.f; for (int f = 0; f < hid; ++f) t = fmaf(dZl[(int64_t)i * VW + f], Hp[(int64_t)j * VW + f], t); Gd += t; }
            if (j < R[l]) { float t = 0.f; for (int f = 0; f < hid; ++f) t = fmaf(dZl[(int64_t)j * VW + f], Hp[(int64_t)i * VW + f], t); Gd += t; }
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
          if (i < n2) a[ppij[p]] = an;
          if (j < n2) a[ppji[p]] = an;
          if (last) { A.out_mask[edge_off + poij[p]] = an; A.out_mask[edge_off + poji[p]] = an; }
        }
      }
      __syncthreads();
    }
  }
}

}  // namespace

int gx_var_smem_bytes(int d, int L, int hid, int emb, int C) { return var_smem(d, L, hid, emb, C, kVarThreads / 32).total * 4; }
int gx_var_row_stride(int hid, int emb) { return 32 * var_kw(hid, emb); }

cudaError_t gx_launch_explain_var(const GxExplainLaunch& cfg, const GxGraphDev& g, const GxModelDev& m,
                                  const GxHparamsDev& hp, const GxPlanArrays& plan, const float* m0,
                                  float* out_mask, float* out_feat, cudaStream_t s) {
  const ExplainArgs args = explain_args(cfg, g, m, hp, plan, m0, out_mask, out_feat);
  const int bytes = gx_var_smem_bytes(m.d, m.L, m.hid, m.emb, m.C);
  const int kw = var_kw(m.hid, m.emb);
  auto go = [&](auto kern) -> cudaError_t {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return e;
    // every launch class asks for the largest shared-memory carveout: CTAs of different classes (= different kernels / footprints) can then
    // share an SM; with per-kernel carveouts a CTA waits for an SM that is completely idle
    e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return e;
    kern<<<cfg.grid, kVarThreads, bytes, s>>>(args);
    return cudaGetLastError();
  };
  if (m.bn) {
    if (kw == 1) return go(explain_var_kernel<true, 1>);
    if (kw == 2) return go(explain_var_kernel<true, 2>);
    return go(explain_var_kernel<true, 4>);
  }
  if (kw == 1) return go(explain_var_kernel<false, 1>);
  if (kw == 2) return go(explain_var_kernel<false, 2>);
  return go(explain_var_kernel<false, 4>);
}
