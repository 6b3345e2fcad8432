// explain_var_common.cuh -- the per-row and per-parameter steps shared by the two model-variant kernels: explain_var.cu (node tasks)
// and explain_graph_var.cu (graph classification).  Both are written for clarity, not speed: one warp per row with lane = feature,
// KW chunks of 32 lanes for widths up to 128 (chunk k holds features 32k + lane), the TRUE widths (no zero padding: a padded column
// would enter the bn statistics), state in a per-CTA global slab.
#pragma once
#include "explain_common.cuh"

namespace {

constexpr int kVarThreads = 256;
constexpr int kVarWeightWords = 36 * 1024;   // conv weights are staged in shared memory up to this many floats (144 KB), read through L2 beyond

// KW = 32-lane chunks of a hidden-width row: 1 for widths <= 32, 2 <= 64, 4 <= 128
__host__ __device__ inline int var_kw(int hid, int emb) { const int w = hid > emb ? hid : emb; return w <= 32 ? 1 : (w <= 64 ? 2 : 4); }

// Shared-memory carve-up (words) of the model-variant kernels: conv weights (when they fit) and biases, pred_model, the feature-mask
// state, per-warp scratch rows and partial dL/dsF, the readout vectors.
struct VarSmem { int W[GX_MAX_LAYERS], b[GX_MAX_LAYERS], Wp, sF, F, mF, vF, zs, zlen, gFp, emb, dEmb, logit, w_in_smem, total; };
__host__ __device__ inline VarSmem var_smem(int d, int L, int hid, int emb, int C, int nwarps) {
  VarSmem S;
  const int dp = gx_round_up(d, 4);
  int o = 0;
  auto take = [&](int words) { int r = o; o += gx_round_up(words, 4); return r; };
  int wwords = 0;
  for (int l = 0; l < L; ++l) wwords += (l == 0 ? d : hid) * (l == L - 1 ? emb : hid);
  S.w_in_smem = wwords <= kVarWeightWords;
  for (int l = 0; l < L; ++l) {
    const int win = l == 0 ? d : hid, wout = l == L - 1 ? emb : hid;
    S.W[l] = take(S.w_in_smem ? win * wout : 0);
    S.b[l] = take(wout);
  }
  const int PD = hid * (L - 1) + emb;
  S.Wp = take(C * (PD + 1) <= GX_WP_SMEM_MAX ? C * (PD + 1) : 0);
  S.sF = take(dp); S.F = take(dp); S.mF = take(dp); S.vF = take(dp);
  S.zlen = dp > 32 * var_kw(hid, emb) ? dp : 32 * var_kw(hid, emb);   // per-warp scratch row: a feature row or a hidden row
  S.zs = take(nwarps * S.zlen);
  S.gFp = take(nwarps * dp);
  S.emb = take(PD); S.dEmb = take(PD); S.logit = take(C < 32 ? 32 : C);
  S.total = o;
  return S;
}

// Stages conv biases (always), conv weights (when S.w_in_smem) and pred_model (when small) in shared memory; Wl[l] = where layer l's
// weights are read from.
__device__ __forceinline__ void var_stage_model(const GxModelDev& m, const VarSmem& S, float* sm, const float** Wl, int tid, int nt) {
  const int L = m.L, PD = m.hid * (L - 1) + m.emb;
  for (int l = 0; l < L; ++l) {
    const int win = l == 0 ? m.d : m.hid, wout = l == L - 1 ? m.emb : m.hid;
    const int cnt = win * wout;
    if (S.w_in_smem)
      for (int idx = tid; idx < cnt; idx += nt) sm[S.W[l] + idx] = __ldg(m.W[l] + idx);
    Wl[l] = S.w_in_smem ? sm + S.W[l] : m.W[l];
    for (int idx = tid; idx < wout; idx += nt) sm[S.b[l] + idx] = __ldg(m.b[l] + idx);
  }
  if (m.C * (PD + 1) <= GX_WP_SMEM_MAX) {
    for (int idx = tid; idx < m.C * PD; idx += nt) sm[S.Wp + idx] = __ldg(m.Wp + idx);
    for (int idx = tid; idx < m.C; idx += nt) sm[S.Wp + m.C * PD + idx] = __ldg(m.bp + idx);
  }
}

// Initial mask parameter of one directed edge slot: the caller's M0 or N(1, m0_std^2) from Philox keyed by (seed, key, slot) --
// key = explained node (node mode) or graph id (graph mode), slot = the canonical edge slot; the tuned kernels draw the same numbers.
__device__ __forceinline__ float var_init_param(const GxHparamsDev& hp, const float* m0, int64_t m0_idx, uint32_t key, uint32_t slot, float m0_std) {
  if (hp.init == GX_INIT_PHILOX) return 1.0f + m0_std * philox_normal(hp.seed, key, slot);
  return __ldg(m0 + m0_idx);
}

// ---------------------------------------------------------------------------------------------------------------------------- forward
// zs[f] = (A_m X)[row] (.) sF for f < d, and Urow = (A_m X)[row] (unmasked, for dL/dsF).  feat rows are addressed feat + gid * d.
__device__ __forceinline__ void var_gather_feat(int r0, int r1, const int32_t* __restrict__ icol, const float* a, const float* feat,
                                                const int32_t* __restrict__ lo2gid, int d, const float* sF, float* Urow, float* zs, int lane) {
  for (int f0 = 0; f0 < d; f0 += 32) {
    const int f = f0 + lane;
    float z = 0.f;
    if (f < d)
      for (int e = r0; e < r1; ++e) z = fmaf(a[e], __ldg(feat + (int64_t)lo2gid[icol[e]] * d + f), z);
    if (f < d) { Urow[f] = z; zs[f] = z * sF[f]; }   // x * sigmoid(feat_mask) (explain.py:707), linear in x
  }
}
// zs[f] = (A_m H)[row] for f < win; H rows have stride 32 * KW
template <int KW>
__device__ __forceinline__ void var_gather_hidden(int r0, int r1, const int32_t* __restrict__ icol, const float* a, const float* Hp, int win,
                                                  float* zs, int lane) {
#pragma unroll
  for (int k = 0; k < KW; ++k) {
    const int f = lane + 32 * k;
    float z = 0.f;
    if (f < win)
      for (int e = r0; e < r1; ++e) z = fmaf(a[e], Hp[(int64_t)icol[e] * (32 * KW) + f], z);
    if (f < win) zs[f] = z;
  }
}
// y = b + zs W (W row-major (win, wout)); lane + 32k < wout
template <int KW>
__device__ __forceinline__ void var_dense(const float* zs, int win, const float* Ws, int wout, const float* bsm, float (&y)[KW], int lane) {
#pragma unroll
  for (int k = 0; k < KW; ++k) y[k] = lane + 32 * k < wout ? bsm[lane + 32 * k] : 0.f;
  for (int f = 0; f < win; ++f) {
    const float zf = zs[f];
#pragma unroll
    for (int k = 0; k < KW; ++k)
      if (lane + 32 * k < wout) y[k] = fmaf(zf, Ws[f * wout + lane + 32 * k], y[k]);
  }
}
// yh = y / max(|y|, 1e-12) (F.normalize(p=2), models.py:78); h = yh on the last layer, else relu(yh) and, with --bn, a fresh
// BatchNorm1d(n) in train mode = per-row standardisation over the feature axis, biased variance, eps 1e-5 (models.py:222-228).
// Returns the norm q; *istd_out = the standardisation's 1/std (bn hidden layers only).
template <bool kBn, int KW>
__device__ __forceinline__ float var_activate(const float (&y)[KW], int wout, bool hidden, float (&yh)[KW], float (&h)[KW], float* istd_out, int lane) {
  float ssl = 0.f;
#pragma unroll
  for (int k = 0; k < KW; ++k) ssl += lane + 32 * k < wout ? y[k] * y[k] : 0.f;
  const float ss = warp_sum(ssl);
  const float q = fmaxf(sqrtf(ss), 1e-12f);
#pragma unroll
  for (int k = 0; k < KW; ++k) { yh[k] = lane + 32 * k < wout ? y[k] / q : 0.f; h[k] = yh[k]; }
  if (hidden) {
#pragma unroll
    for (int k = 0; k < KW; ++k) h[k] = fmaxf(yh[k], 0.f);
    if (kBn) {
      float sl = 0.f;
#pragma unroll
      for (int k = 0; k < KW; ++k) sl += lane + 32 * k < wout ? h[k] : 0.f;
      const float mu = warp_sum(sl) / (float)wout;
      float vl = 0.f;
#pragma unroll
      for (int k = 0; k < KW; ++k) { h[k] = lane + 32 * k < wout ? h[k] - mu : 0.f; vl += h[k] * h[k]; }
      const float var = warp_sum(vl) / (float)wout;
      const float is = 1.0f / sqrtf(var + 1e-5f);
#pragma unroll
      for (int k = 0; k < KW; ++k) h[k] *= is;
      *istd_out = is;
    }
  }
  return q;
}

// --------------------------------------------------------------------------------------------------------------------------- backward
// g += (A_m^T dZ_{l+1})[row] over the row's leading columns < bound (A_m symmetric); dZn rows have stride 32 * KW
template <int KW>
__device__ __forceinline__ void var_gather_back(int r0, int r1, const int32_t* __restrict__ icol, const float* a, const float* dZn, int wout, int bound,
                                                float (&g)[KW], int lane) {
  for (int e = r0; e < r1; ++e) {
    const int j = icol[e];
    if (j >= bound) break;
    const float ae = a[e];
#pragma unroll
    for (int k = 0; k < KW; ++k)
      if (lane + 32 * k < wout) g[k] = fmaf(ae, dZn[(int64_t)j * (32 * KW) + lane + 32 * k], g[k]);
  }
}
// g = dL/dH of a hidden row -> dL/dYh: backward of the standardisation, (g - mean(g) - Hb mean(g Hb)) * istd, then of the ReLU
template <bool kBn, int KW>
__device__ __forceinline__ void var_hidden_backward(float (&g)[KW], const float (&yh)[KW], const float* Hrow, float is, int wout, int lane) {
  if (kBn) {
    float hb[KW], s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < KW; ++k) {
      hb[k] = Hrow[lane + 32 * k];
      if (lane + 32 * k < wout) { s1 += g[k]; s2 += g[k] * hb[k]; }
    }
    const float m1 = warp_sum(s1) / (float)wout, m2 = warp_sum(s2) / (float)wout;
#pragma unroll
    for (int k = 0; k < KW; ++k) g[k] = lane + 32 * k < wout ? (g[k] - m1 - hb[k] * m2) * is : 0.f;
  }
#pragma unroll
  for (int k = 0; k < KW; ++k) g[k] = yh[k] > 0.f ? g[k] : 0.f;
}
// <yh, g> over the row: the backward of y / max(|y|, eps) is dY = (g - yh <yh, g>) / q
template <int KW>
__device__ __forceinline__ float var_norm_dot(const float (&g)[KW], const float (&yh)[KW], int wout, int lane) {
  float sl = 0.f;
#pragma unroll
  for (int k = 0; k < KW; ++k) sl += lane + 32 * k < wout ? yh[k] * g[k] : 0.f;
  return warp_sum(sl);
}
template <int KW>
__device__ __forceinline__ void var_norm_backward(const float (&g)[KW], const float (&yh)[KW], float sdot, float q, int wout, float* zs, int lane) {
#pragma unroll
  for (int k = 0; k < KW; ++k)
    if (lane + 32 * k < wout) zs[lane + 32 * k] = (g[k] - yh[k] * sdot) / q;
}
// layer 1: dZ[f] = sum_c dY[c] W[f][c] for f < d; gFp[f] += dZ[f] U[f] (dL/dsF partial), dZ1row = dZ (.) sF (kept masked for the edge dots)
__device__ __forceinline__ void var_first_layer_dz(const float* zs, const float* Ws, int d, int wout, const float* Urow, const float* sF,
                                                   float* gFp, float* dZ1row, int lane) {
  for (int f0 = 0; f0 < d; f0 += 32) {
    const int f = f0 + lane;
    float t = 0.f;
    if (f < d)
      for (int c = 0; c < wout; ++c) t = fmaf(zs[c], Ws[f * wout + c], t);
    if (f < d) {
      gFp[f] = fmaf(t, Urow[f], gFp[f]);
      dZ1row[f] = t * sF[f];
    }
  }
}
// layers >= 2: dZrow[f] = sum_c dY[c] W[f][c] for f < win (0 in the padding lanes)
template <int KW>
__device__ __forceinline__ void var_hidden_dz(const float* zs, const float* Ws, int win, int wout, float* dZrow, int lane) {
#pragma unroll
  for (int k = 0; k < KW; ++k) {
    const int f = lane + 32 * k;
    float t = 0.f;
    if (f < win)
      for (int c = 0; c < wout; ++c) t = fmaf(zs[c], Ws[f * wout + c], t);
    dZrow[f] = f < win ? t : 0.f;
  }
}

// ---------------------------------------------------------------------------------------------------------------------- optimisers
// One step of the optimiser on a feature-mask entry (IEEE arithmetic) and on an edge-mask parameter (the edge phase's arithmetic,
// explain_common.cuh).  (step, bc2s) = this epoch's row of the per-step table: Adam (lr_t / (1-b1^t), sqrt(1-b2^t)), other optimisers (lr_t, 1).
__device__ __forceinline__ void var_feat_update(const GxHparamsDev& hp, float g, float& P, float& m, float& v, float step, float bc2s) {
  if (hp.opt == GX_OPT_ADAM) {
    m = m + (g - m) * hp.one_minus_b1;
    v = v * hp.b2 + hp.one_minus_b2 * g * g;
    P = P - step * (m / (sqrtf(v) / bc2s + hp.eps));
  } else {
    opt_step_other(hp.opt, P, g, m, v, step);
  }
}
__device__ __forceinline__ void var_edge_update(const GxHparamsDev& hp, float g, float& P, float& m, float& v, float step, float bc2s, float bc2s_inv,
                                                bool ieee) {
  if (hp.opt == GX_OPT_ADAM) {
    m = m + (g - m) * hp.one_minus_b1;
    v = v * hp.b2 + hp.one_minus_b2 * g * g;
    P = P - adam_delta_fast(m, v, step, bc2s, bc2s_inv, hp.eps, ieee);
  } else {
    opt_step_other(hp.opt, P, g, m, v, step);
  }
}

// Readout tail shared by both modes (one warp): logits = Wp emb + bp, softmax, dL/dlogits = p - onehot(gt) (explain.py:750-753),
// dEmb = Wp^T dL/dlogits.
__device__ __forceinline__ void var_readout_tail(const float* emb, const float* Wpp, const float* bpp, int C, int PD, int gt, float* logit,
                                                 float* dEmb, int lane) {
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
  for (int c = lane; c < C; c += 32) logit[c] = expf(logit[c] - mx) / se - (c == gt ? 1.f : 0.f);
  __syncwarp();
  for (int k = lane; k < PD; k += 32) {
    float t = 0.f;
    for (int c = 0; c < C; ++c) t = fmaf(logit[c], Wpp[c * PD + k], t);
    dEmb[k] = t;
  }
}

}  // namespace
