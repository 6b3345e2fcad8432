// explain_var_common.cuh -- the per-row and per-parameter steps and the launch code shared by the model-variant kernel
// (explain_var.cu, node and graph mode) and the unconstrained kernel (explain_dense.cu).  Both are written for clarity, not speed:
// one persistent CTA per task, one warp per row with lane = feature, KW chunks of 32 lanes for widths up to 128, or 256 on the
// variant kernel's row-block path (chunk k holds features 32k + lane), the TRUE widths (no zero padding: a padded column would enter
// the bn statistics), state in a per-CTA global slab.
#pragma once
#include <type_traits>

#include "explain_common.cuh"

namespace {

constexpr int kVarThreads = 256;
constexpr int kVarWeightWords = 36 * 1024;   // conv weights are staged in shared memory up to this many floats (144 KB), read through L2 beyond

// KW = 32-lane chunks of a hidden-width row: 1 for widths <= 32, 2 <= 64, 4 <= 128
__host__ __device__ inline int var_kw(int hid, int emb) { const int w = hid > emb ? hid : emb; return w <= 32 ? 1 : (w <= 64 ? 2 : 4); }
// the same with 8 for widths 129 .. 256 (explain_var.cu's row-block path: its per-warp scratch rows stay var_kw wide, the dY rows are
// written to the slab in place)
inline int var_row_kw(int hid, int emb) { return (hid > emb ? hid : emb) > 128 ? 8 : var_kw(hid, emb); }

// Shared-memory carve-up (words) of the model-variant kernels: conv weights (when they fit) and biases, pred_model, the feature-mask
// state, per-warp scratch rows and partial dL/dsF, the readout vectors.  Attention models (att != 0) also stage the (in, in)
// attention weights when they fit the weight budget together with the conv weights (var_att_in_smem): the last var_att_words words
// before S.total, layer by layer; else they are read through L2 and the conv weights are staged as for any other model.
// Models with an MLP prediction head (hd.k > 0) also hold the head's activations hx (its widths back to back) and two gradient
// vectors hg of its largest width; pred_model's slot Wp holds the whole head block when it fits.  Head-less models: zero words.
struct VarSmem { int W[GX_MAX_LAYERS], b[GX_MAX_LAYERS], Wp, sF, F, mF, vF, zs, zlen, gFp, emb, dEmb, logit, hx, hg, w_in_smem, total; };
__host__ __device__ inline int var_att_words(int d, int L, int hid) {
  int w = 0;
  for (int l = 0; l < L; ++l) w += gx_round_up((l == 0 ? d : hid) * (l == 0 ? d : hid), 4);
  return w;
}
__host__ __device__ inline int var_conv_words(int d, int L, int hid, int emb) {
  int w = 0;
  for (int l = 0; l < L; ++l) w += (l == 0 ? d : hid) * (l == L - 1 ? emb : hid);
  return w;
}
__host__ __device__ inline bool var_att_in_smem(int d, int L, int hid, int emb) {
  return var_conv_words(d, L, hid, emb) + var_att_words(d, L, hid) <= kVarWeightWords;
}
__host__ __device__ inline VarSmem var_smem(int d, int L, int hid, int emb, int C, int nwarps, int att = 0, const GxHeadDev& hd = GxHeadDev{}) {
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
  const int hw = gx_head_words(hd, PD, C);
  S.Wp = take(hw <= GX_WP_SMEM_MAX ? hw : 0);
  S.sF = take(dp); S.F = take(dp); S.mF = take(dp); S.vF = take(dp);
  S.zlen = dp > 32 * var_kw(hid, emb) ? dp : 32 * var_kw(hid, emb);   // per-warp scratch row: a feature row or a hidden row
  S.zs = take(nwarps * S.zlen);
  S.gFp = take(nwarps * dp);
  S.emb = take(PD); S.dEmb = take(PD); S.logit = take(C < 32 ? 32 : C);
  S.hx = take(gx_head_act_words(hd)); S.hg = take(2 * gx_head_max_width(hd));
  if (att && var_att_in_smem(d, L, hid, emb)) take(var_att_words(d, L, hid));
  S.total = o;
  return S;
}

// Wide inputs (d > 128, explain_var.cu kWide) keep the feature-mask state and layer 1's products in the task slab and read W1 through
// L2, so that nothing here grows with d: no feature-mask arrays or dL/dsF partials, hidden-width scratch rows, and only the layers
// >= 2 are staged (S.W[0] takes zero words).
__host__ __device__ inline VarSmem var_smem_wide(int d, int L, int hid, int emb, int C, int nwarps, const GxHeadDev& hd = GxHeadDev{}) {
  VarSmem S;
  int o = 0;
  auto take = [&](int words) { int r = o; o += gx_round_up(words, 4); return r; };
  int wwords = 0;
  for (int l = 1; l < L; ++l) wwords += hid * (l == L - 1 ? emb : hid);
  S.w_in_smem = wwords <= kVarWeightWords;
  for (int l = 0; l < L; ++l) {
    const int wout = l == L - 1 ? emb : hid;
    S.W[l] = take(S.w_in_smem && l > 0 ? hid * wout : 0);
    S.b[l] = take(wout);
  }
  const int PD = hid * (L - 1) + emb;
  const int hw = gx_head_words(hd, PD, C);
  S.Wp = take(hw <= GX_WP_SMEM_MAX ? hw : 0);
  S.sF = S.F = S.mF = S.vF = o;
  S.zlen = 32 * var_kw(hid, emb);
  S.zs = take(nwarps * S.zlen);
  S.gFp = o;
  S.emb = take(PD); S.dEmb = take(PD); S.logit = take(C < 32 ? 32 : C);
  S.hx = take(gx_head_act_words(hd)); S.hg = take(2 * gx_head_max_width(hd));
  S.total = o;
  (void)d;
  return S;
}
template <bool kWide>
__host__ __device__ inline VarSmem var_smem_of(int d, int L, int hid, int emb, int C, int nwarps, int att, const GxHeadDev& hd) {
  if constexpr (kWide) return var_smem_wide(d, L, hid, emb, C, nwarps, hd);
  else return var_smem(d, L, hid, emb, C, nwarps, att, hd);
}

// Stages conv biases (always), conv weights (when S.w_in_smem) and pred_model or the MLP head block (when small) in shared memory;
// Wl[l] = where layer l's weights are read from.
// With kWide, layer 1's weights stay in global memory (var_smem_wide).
template <bool kWide = false>
__device__ __forceinline__ void var_stage_model(const GxModelDev& m, const GxHeadDev& hd, const VarSmem& S, float* sm, const float** Wl, int tid,
                                                int nt) {
  const int L = m.L, PD = m.hid * (L - 1) + m.emb;
  for (int l = 0; l < L; ++l) {
    if constexpr (kWide) {
      if (l == 0) {
        Wl[0] = m.W[0];
        for (int idx = tid; idx < m.hid; idx += nt) sm[S.b[0] + idx] = __ldg(m.b[0] + idx);
        continue;
      }
    }
    const int win = l == 0 ? m.d : m.hid, wout = l == L - 1 ? m.emb : m.hid;
    const int cnt = win * wout;
    if (S.w_in_smem)
      for (int idx = tid; idx < cnt; idx += nt) sm[S.W[l] + idx] = __ldg(m.W[l] + idx);
    Wl[l] = S.w_in_smem ? sm + S.W[l] : m.W[l];
    for (int idx = tid; idx < wout; idx += nt) sm[S.b[l] + idx] = __ldg(m.b[l] + idx);
  }
  const int hw = gx_head_words(hd, PD, m.C);
  if (hw > GX_WP_SMEM_MAX) return;
  if (hd.k > 0) {
    for (int idx = tid; idx < hw; idx += nt) sm[S.Wp + idx] = __ldg(hd.W + idx);
  } else {
    for (int idx = tid; idx < m.C * PD; idx += nt) sm[S.Wp + idx] = __ldg(m.Wp + idx);
    for (int idx = tid; idx < m.C; idx += nt) sm[S.Wp + m.C * PD + idx] = __ldg(m.bp + idx);
  }
}
// Attention models: stages the attention weights when var_att_in_smem; Wal[l] = where layer l's are read from.
__device__ __forceinline__ void var_stage_att(const GxModelDev& m, const VarSmem& S, float* sm, const float** Wal, int tid, int nt) {
  const bool in_smem = var_att_in_smem(m.d, m.L, m.hid, m.emb);
  int o = S.total - var_att_words(m.d, m.L, m.hid);
  for (int l = 0; l < m.L; ++l) {
    const int win = l == 0 ? m.d : m.hid;
    if (in_smem)
      for (int idx = tid; idx < win * win; idx += nt) sm[o + idx] = __ldg(gx_att_weight(m, l) + idx);
    Wal[l] = in_smem ? sm + o : gx_att_weight(m, l);
    o += gx_round_up(win * win, 4);
  }
}

// Initial mask parameter of one directed edge slot: the caller's M0 or N(1, m0_std^2) from Philox keyed by (seed, key, slot) --
// key = explained node (node mode) or graph id (graph mode), slot = the canonical edge slot; the tuned kernels draw the same numbers.
__device__ __forceinline__ float var_init_param(const GxHparamsDev& hp, const float* m0, int64_t m0_idx, uint32_t key, uint32_t slot, float m0_std) {
  if (hp.init == GX_INIT_PHILOX) return 1.0f + m0_std * philox_normal(hp.seed, key, slot);
  return __ldg(m0 + m0_idx);
}

// Takes the persistent CTA's next task from the work queue (A.order, A.ntasks, A.counter) into task_id; false when the queue is drained.
// Every thread calls.
template <typename Args>
__device__ __forceinline__ bool var_next_task(const Args& A, int& s_task, int tid, int& task_id) {
  __syncthreads();
  if (tid == 0) s_task = atomicAdd(A.counter, 1);
  __syncthreads();
  const int qi = s_task;
  if (qi >= A.ntasks) return false;
  task_id = A.order[qi];
  return true;
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
// Layer l's per-row arrays, as the kernels' slab accessors give them: Yh(l) normalised pre-activations (row stride 32 * KW), H(l) outputs
// (row stride ldh), qn(l) norms, istd(l) the bn standardisation's 1/std.  The addresses are formed where they are used.
// Row i of layer l (1 .. L) from its pre-activation y: var_activate, then the stores (H is 0 in the padding lanes).  (The wide path's
// layer 1; var_row_forward below is the same steps after y = b + zs W.)
template <bool kBn, int KW, typename YhF, typename HF, typename QF, typename IF>
__device__ __forceinline__ void var_row_epilogue(const float (&y)[KW], int wout, int l, int L, int i, YhF Yh, HF H, int64_t ldh, QF qn, IF istd,
                                                 int lane) {
  float yh[KW], h[KW], is = 1.f;
  const float q = var_activate<kBn, KW>(y, wout, l < L, yh, h, &is, lane);
  if (kBn && l < L && lane == 0) istd(l)[i] = is;
#pragma unroll
  for (int k = 0; k < KW; ++k) {
    Yh(l)[(int64_t)i * (32 * KW) + lane + 32 * k] = yh[k];
    H(l)[(int64_t)i * ldh + lane + 32 * k] = lane + 32 * k < wout ? h[k] : 0.f;
  }
  if (lane == 0) qn(l)[i] = q;
}
// Row i of layer l (1 .. L) after its aggregate is in zs: y = b + zs W, var_activate, then the stores (H is 0 in the padding lanes).
template <bool kBn, int KW, typename YhF, typename HF, typename QF, typename IF>
__device__ __forceinline__ void var_row_forward(const float* zs, int win, const float* Ws, int wout, const float* bsm, int l, int L, int i,
                                                YhF Yh, HF H, int64_t ldh, QF qn, IF istd, int lane) {
  __syncwarp();
  float y[KW];
  var_dense<KW>(zs, win, Ws, wout, bsm, y, lane);
  __syncwarp();
  float yh[KW], h[KW], is = 1.f;
  const float q = var_activate<kBn, KW>(y, wout, l < L, yh, h, &is, lane);
  if (kBn && l < L && lane == 0) istd(l)[i] = is;
#pragma unroll
  for (int k = 0; k < KW; ++k) {
    Yh(l)[(int64_t)i * (32 * KW) + lane + 32 * k] = yh[k];
    H(l)[(int64_t)i * ldh + lane + 32 * k] = lane + 32 * k < wout ? h[k] : 0.f;
  }
  if (lane == 0) qn(l)[i] = q;
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
// Row i of layer l, g = dL/dH -> zs = dL/dY: the bn and ReLU backward on hidden layers, then the backward of y / max(|y|, eps).
// H, qn, istd as in var_row_forward.
template <bool kBn, int KW, typename HF, typename QF, typename IF>
__device__ __forceinline__ void var_row_backward(float (&g)[KW], const float (&yh)[KW], int l, int L, int i, HF H, int64_t ldh, QF qn, IF istd,
                                                 int wout, float* zs, int lane) {
  if (l < L) var_hidden_backward<kBn, KW>(g, yh, H(l) + (int64_t)i * ldh, kBn ? istd(l)[i] : 1.f, wout, lane);
  const float sdot = var_norm_dot<KW>(g, yh, wout, lane);
  const float q = qn(l)[i];
  __syncwarp();
  var_norm_backward<KW>(g, yh, sdot, q, wout, zs, lane);
  __syncwarp();
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

// Readout tail shared by both modes and kernels (every thread calls; emb must be complete; the caller synchronises before reading
// logit or dEmb).  pred_model = Linear 0 .. k of the head (k = 0: Wp / bp; else the head block blk, models.py:193-207):
//   forward  x_0 = emb, x_j = relu(W_j x_{j-1} + b_j) into hx, logits = W_k x_k + b_k;  softmax, dL/dlogits = p - onehot(gt)
//            (explain.py:750-753) into logit;
//   backward g = W_j^T g, through each ReLU (0 where x_j <= 0, as torch) down to dEmb = W_0^T g.
// Each output of a forward product is one warp's lane-strided dot and warp sum, each entry of a backward product one thread's chain over
// the outputs in ascending order, whichever warp or thread takes it: a head-less model computes what one warp computed before.
__device__ __forceinline__ void var_readout_tail(const float* emb, const GxHeadDev& hd, const float* blk, const float* Wpp, const float* bpp,
                                                 int C, int PD, int gt, float* hx, float* hg, float* logit, float* dEmb, int tid, int nt) {
  const int lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
  const int k = hd.k, mw = gx_head_max_width(hd);
  auto lin = [&](int j, const float*& W, const float*& b) {   // Linear j's weight (out, in) and bias
    if (k == 0) { W = Wpp; b = bpp; return; }
    W = blk + gx_head_off(hd, PD, C, j);
    b = W + gx_head_out(hd, C, j) * gx_head_in(hd, PD, j);
  };
  auto act = [&](int j) { int o = 0; for (int i = 0; i < j; ++i) o += hd.w[i]; return hx + o; };   // hidden layer j's output x_{j+1}
  for (int j = 0; j <= k; ++j) {
    const int in = gx_head_in(hd, PD, j), out = gx_head_out(hd, C, j);
    const float *W, *b;
    lin(j, W, b);
    const float* const x = j == 0 ? emb : act(j - 1);
    float* const y = j == k ? logit : act(j);
    for (int o = warp; o < out; o += nwarps) {
      float t = 0.f;
      for (int i = lane; i < in; i += 32) t = fmaf(x[i], W[o * in + i], t);
      t = warp_sum(t);
      if (lane == 0) y[o] = j == k ? t + b[o] : fmaxf(t + b[o], 0.f);
    }
    __syncthreads();
  }
  if (warp == 0) {
    float mx = -INFINITY;
    for (int c = lane; c < C; c += 32) mx = fmaxf(mx, logit[c]);
    mx = warp_max(mx);
    float se = 0.f;
    for (int c = lane; c < C; c += 32) se += expf(logit[c] - mx);
    se = warp_sum(se);
    __syncwarp();
    for (int c = lane; c < C; c += 32) logit[c] = expf(logit[c] - mx) / se - (c == gt ? 1.f : 0.f);
  }
  __syncthreads();
  for (int j = k; j >= 0; --j) {
    const int in = gx_head_in(hd, PD, j), out = gx_head_out(hd, C, j);
    const float *W, *b;
    lin(j, W, b);
    const float* const g = j == k ? logit : hg + (j & 1) * mw;
    float* const dx = j == 0 ? dEmb : hg + ((j - 1) & 1) * mw;
    const float* const xin = j == 0 ? nullptr : act(j - 1);
    for (int i = tid; i < in; i += nt) {
      float t = 0.f;
      for (int o = 0; o < out; ++o) t = fmaf(g[o], W[o * in + i], t);
      dx[i] = xin != nullptr && !(xin[i] > 0.f) ? 0.f : t;
    }
    if (j > 0) __syncthreads();
  }
}

// Graph mode's readout input (models.py:283,291,300): pooled feature k = column c of layer l is the max over rows 0 .. n-1 of
// Hl(l)[i * ld + c], starting from best0[k] (nullptr: -inf) and arg0; arg[k] = the first maximal row, like torch.max.  Every thread calls.
template <typename Hl>
__device__ __forceinline__ void var_max_pool(int L, int hid, int PD, int n, Hl Hl_of, int64_t ld, const float* best0, int arg0,
                                             float* emb, int* arg, int tid, int nt) {
  for (int k = tid; k < PD; k += nt) {
    const int l = k < hid * (L - 1) ? k / hid + 1 : L;
    const int c = k - hid * (l - 1);
    const float* const H = Hl_of(l);
    float best = best0 != nullptr ? best0[k] : -INFINITY;
    int bi = arg0;
    for (int i = 0; i < n; ++i) {
      const float v = H[(int64_t)i * ld + c];
      if (v > best) { best = v; bi = i; }   // strict: the first maximal row wins
    }
    emb[k] = best; arg[k] = bi;
  }
}

// ------------------------------------------------------------------------------------------------------------------------- launch
// Calls f(std::integral_constant<bool, kBn>, std::integral_constant<int, KW>) with the model's instantiation, widths up to 128 (wider
// rows have no instantiation here: explain_var.cu dispatches its row-block path itself).
template <typename F>
cudaError_t var_dispatch(const GxModelDev& m, F&& f) {
  using B = std::integral_constant<bool, true>;
  using N = std::integral_constant<bool, false>;
  const int kw = var_row_kw(m.hid, m.emb);
  if (kw > 4) return cudaErrorInvalidValue;
  if (m.bn) {
    if (kw == 1) return f(B(), std::integral_constant<int, 1>());
    if (kw == 2) return f(B(), std::integral_constant<int, 2>());
    return f(B(), std::integral_constant<int, 4>());
  }
  if (kw == 1) return f(N(), std::integral_constant<int, 1>());
  if (kw == 2) return f(N(), std::integral_constant<int, 2>());
  return f(N(), std::integral_constant<int, 4>());
}

// Lets kern use `bytes` of dynamic shared memory with the largest carveout: CTAs of different launch classes (= different kernels /
// footprints) can then share an SM; with per-kernel carveouts a CTA waits for an SM that is completely idle
template <typename Args>
cudaError_t var_set_smem(void (*kern)(Args), int bytes) {
  const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}
template <typename Args>
cudaError_t var_launch(void (*kern)(Args), const Args& args, int grid, int bytes, cudaStream_t s) {
  const cudaError_t e = var_set_smem(kern, bytes);
  if (e != cudaSuccess) return e;
  kern<<<grid, kVarThreads, bytes, s>>>(args);
  return cudaGetLastError();
}
// co-resident CTAs of kern per SM (sizes the persistent grid); 0 on error
template <typename Args>
int var_ctas_per_sm(void (*kern)(Args), int bytes) {
  int n = 0;
  cudaError_t e = var_set_smem(kern, bytes);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, kVarThreads, bytes);
  return e == cudaSuccess ? n : 0;
}

}  // namespace
