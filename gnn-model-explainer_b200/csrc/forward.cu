// forward.cu -- the GCN forward of the reference model on the WHOLE graph (models.py:58-80 GraphConv.forward, :230-267 gcn_forward,
// :363-376 GcnEncoderNode.forward): what produces the `pred` the Explainer is constructed with (explainer_main.py:186-193 reads it
// from the checkpoint; `Explainer(pred=None)` computes it here).  Unmasked adjacency, no feature mask, every model gx_set_model accepts
// (num_layers 2 .. 7, widths up to 256, --bn).  One launch per layer (a layer reads every row of the previous one), a warp per node with
// lane = feature (1, 2, 4 or 8 chunks of 32 lanes) -- the same row
// arithmetic as explain_var.cu: Y = (sum_{j in N(i)} H_{l-1}[j]) W_l + b_l, row L2-normalise, ReLU (+ per-node standardisation
// with --bn) on hidden layers; logits = pred_model(concat of the layer outputs).  Attention models (--method att, models.py:62-68) first
// project P = H_{l-1} Wa_l (att_project_kernel) and weight every edge, self loops included, by s_ij = P_i . P_j.
#include <algorithm>

#include "explain_common.cuh"

namespace {

constexpr int kFwdThreads = 256;

// P = Hin Wa for all N nodes (attention models): a warp per node, Hin rows of stride ldin, P rows of stride ldp = round_up(win, 4)
__global__ void __launch_bounds__(kFwdThreads) att_project_kernel(int64_t N, const float* __restrict__ Hin, int ldin, const float* __restrict__ Wa, int win,
                                                                  float* __restrict__ P) {
  extern __shared__ float zs_all[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = kFwdThreads / 32;
  const int ldp = gx_round_up(win, 4);
  float* const zs = zs_all + warp * ldp;
  for (int64_t i = (int64_t)blockIdx.x * nwarps + warp; i < N; i += (int64_t)gridDim.x * nwarps) {
    for (int f = lane; f < win; f += 32) zs[f] = Hin[i * ldin + f];
    __syncwarp();
    for (int c = lane; c < win; c += 32) {
      float p = 0.f;
      for (int f = 0; f < win; ++f) p = fmaf(zs[f], __ldg(Wa + f * win + c), p);
      P[i * ldp + c] = p;
    }
    __syncwarp();
  }
}

// s_ij = P_i . P_j (every lane gets it); P rows of stride round_up(win, 4)
__device__ __forceinline__ float att_score(const float* __restrict__ P, int64_t i, int64_t j, int win, int lane) {
  const int ldp = gx_round_up(win, 4);
  float sp = 0.f;
  for (int f = lane; f < win; f += 32) sp = fmaf(P[i * ldp + f], P[j * ldp + f], sp);
  return warp_sum(sp);
}

// one GCN layer for all N nodes, KW chunks of 32 lanes per row (lane + 32 k = feature, as explain_var.cu).  Hin: [N][32 KW] (layer > 1)
// or the feature matrix [N][d] (layer 1); Hout: [N][32 KW] what the next layer / the readout sees (relu / standardised on hidden
// layers, the normalised output on the last).  kAtt: edge weights s_ij from P.
template <bool kFirst, bool kAtt, int KW>
__global__ void __launch_bounds__(kFwdThreads) gcn_layer_kernel(GxGraphDev g, const float* __restrict__ Hin, const float* __restrict__ W, const float* __restrict__ b,
                                                                int win, int wout, int last, int bn, const float* __restrict__ P, float* __restrict__ Hout) {
  extern __shared__ float zs_all[];
  constexpr int LD = 32 * KW;   // row stride of the hidden-width arrays
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = kFwdThreads / 32;
  const int dp = gx_round_up(win, 4);
  float* const zs = zs_all + warp * dp;
  for (int64_t i = (int64_t)blockIdx.x * nwarps + warp; i < g.N; i += (int64_t)gridDim.x * nwarps) {
    const int r0 = g.rowptr[i], r1 = g.rowptr[i + 1];
    float y[KW];
#pragma unroll
    for (int k = 0; k < KW; ++k) y[k] = lane + 32 * k < wout ? __ldg(b + lane + 32 * k) : 0.f;
    if (kAtt || kFirst || KW > 1) {   // zs = the row's aggregate, then y += zs W
      for (int f0 = 0; f0 < win; f0 += 32) {
        const int f = f0 + lane;
        float z = 0.f;
        if constexpr (kAtt) {   // (A (.) s) Hin[i]: every lane takes part in every edge's score
          for (int e = r0; e < r1; ++e) {
            const int64_t j = g.col[e];
            const float se = att_score(P, i, j, win, lane);
            if (f < win) z = fmaf(se, Hin[j * (kFirst ? win : LD) + f], z);
          }
        } else if (f < win) {
          for (int e = r0; e < r1; ++e) z += __ldg(Hin + (int64_t)g.col[e] * (kFirst ? win : LD) + f);   // raw adjacency, self loops included (models.py:70: torch.matmul(adj, x))
        }
        if (f < win) zs[f] = z;
      }
      __syncwarp();
#pragma unroll
      for (int k = 0; k < KW; ++k)
        if (lane + 32 * k < wout)
          for (int f = 0; f < win; ++f) y[k] = fmaf(zs[f], __ldg(W + f * wout + lane + 32 * k), y[k]);
      __syncwarp();
    } else {   // one chunk: the aggregate stays in the lanes
      float z = 0.f;
      if (lane < win)
        for (int e = r0; e < r1; ++e) z += Hin[(int64_t)g.col[e] * 32 + lane];
      for (int f = 0; f < win; ++f) {
        const float zf = __shfl_sync(0xffffffffu, z, f);
        if (lane < wout) y[0] = fmaf(zf, __ldg(W + f * wout + lane), y[0]);
      }
    }
    float ssl = 0.f;
#pragma unroll
    for (int k = 0; k < KW; ++k) ssl += lane + 32 * k < wout ? y[k] * y[k] : 0.f;
    const float ss = warp_sum(ssl);
    const float q = fmaxf(sqrtf(ss), 1e-12f);   // F.normalize(p=2, dim=2), eps 1e-12 (models.py:78)
    float h[KW];
#pragma unroll
    for (int k = 0; k < KW; ++k) h[k] = lane + 32 * k < wout ? y[k] / q : 0.f;
    if (!last) {
#pragma unroll
      for (int k = 0; k < KW; ++k) h[k] = fmaxf(h[k], 0.f);
      if (bn) {   // fresh BatchNorm1d(n) in train mode: per node over the feature axis (models.py:222-228)
        float sl = 0.f;
#pragma unroll
        for (int k = 0; k < KW; ++k) sl += lane + 32 * k < wout ? h[k] : 0.f;
        const float mu = warp_sum(sl) / (float)wout;
        float vl = 0.f;
#pragma unroll
        for (int k = 0; k < KW; ++k) { h[k] = lane + 32 * k < wout ? h[k] - mu : 0.f; vl += h[k] * h[k]; }
        const float var = warp_sum(vl) / (float)wout;
#pragma unroll
        for (int k = 0; k < KW; ++k) h[k] = h[k] / sqrtf(var + 1e-5f);
      }
    }
#pragma unroll
    for (int k = 0; k < KW; ++k) Hout[i * LD + lane + 32 * k] = lane + 32 * k < wout ? h[k] : 0.f;
  }
}

// logits[i][c] = bp[c] + sum_k emb_i[k] Wp[c][k], emb_i = [H_1[i] | ... | H_L[i]] (models.py:260,375); H rows of stride 32 KW
template <int KW>
__global__ void __launch_bounds__(kFwdThreads) readout_kernel(int64_t N, int L, int hid, int emb, int C, const float* __restrict__ H, const float* __restrict__ Wp,
                                                              const float* __restrict__ bp, float* __restrict__ pred, float* __restrict__ emb_out) {
  constexpr int LD = 32 * KW;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = kFwdThreads / 32;
  const int PD = hid * (L - 1) + emb;
  for (int64_t i = (int64_t)blockIdx.x * nwarps + warp; i < N; i += (int64_t)gridDim.x * nwarps) {
    for (int c = 0; c < C; ++c) {
      float t = 0.f;
      for (int l = 0; l < L; ++l) {
        const int w = l == L - 1 ? emb : hid;
#pragma unroll
        for (int k = 0; k < KW; ++k)
          if (lane + 32 * k < w) t = fmaf(H[((int64_t)l * N + i) * LD + lane + 32 * k], __ldg(Wp + c * PD + hid * l + lane + 32 * k), t);
      }
      t = warp_sum(t);
      if (lane == 0) pred[i * C + c] = t + __ldg(bp + c);
    }
    if (emb_out != nullptr)
      for (int l = 0; l < L; ++l) {
        const int w = l == L - 1 ? emb : hid;
        for (int c = lane; c < w; c += 32) emb_out[i * PD + hid * l + c] = H[((int64_t)l * N + i) * LD + c];
      }
  }
}

// MLP prediction head (models.py:193-207) on every row: x_0 = emb_i, x_j = relu(W_j x_{j-1} + b_j), pred_i = W_k x_k + b_k, a warp per row
// with the products of the explainer kernels' readout tail (each output a lane-strided dot and a warp sum), x_j in two per-warp vectors
// of the head's largest width.
__global__ void __launch_bounds__(kFwdThreads) head_kernel(int64_t N, int PD, int C, GxHeadDev hd, const float* __restrict__ emb,
                                                           float* __restrict__ pred) {
  extern __shared__ float xs_all[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = kFwdThreads / 32;
  const int mw = gx_head_max_width(hd);
  float* const xs = xs_all + warp * 2 * mw;
  for (int64_t i = (int64_t)blockIdx.x * nwarps + warp; i < N; i += (int64_t)gridDim.x * nwarps) {
    for (int j = 0; j <= hd.k; ++j) {
      const int in = gx_head_in(hd, PD, j), out = gx_head_out(hd, C, j);
      const float* const W = hd.W + gx_head_off(hd, PD, C, j);
      const float* const b = W + out * in;
      const float* const x = j == 0 ? emb + i * PD : xs + ((j - 1) & 1) * mw;
      for (int o = 0; o < out; ++o) {
        float t = 0.f;
        for (int f = lane; f < in; f += 32) t = fmaf(x[f], __ldg(W + o * in + f), t);
        t = warp_sum(t);
        if (lane == 0) {
          if (j == hd.k) pred[i * C + o] = t + __ldg(b + o);
          else xs[(j & 1) * mw + o] = fmaxf(t + __ldg(b + o), 0.f);
        }
      }
      __syncwarp();
    }
  }
}

template <int KW>
cudaError_t model_forward(const GxGraphDev& g, const GxModelDev& m, const GxHeadDev& hd, float* H, float* pred, float* emb_out, float* P,
                          cudaStream_t s) {
  constexpr int LD = 32 * KW;
  const int nwarps = kFwdThreads / 32;
  const int grid = (int)std::min<int64_t>((g.N + nwarps - 1) / nwarps, GX_GRID_CAP);
  for (int l = 0; l < m.L; ++l) {
    const int win = l == 0 ? m.d : m.hid, wout = l == m.L - 1 ? m.emb : m.hid;
    const float* Hin = l == 0 ? g.feat : H + (int64_t)(l - 1) * g.N * LD;
    float* Hout = H + (int64_t)l * g.N * LD;
    const size_t smem = (size_t)nwarps * gx_round_up(win, 4) * sizeof(float);
    if (m.att) {
      att_project_kernel<<<grid, kFwdThreads, smem, s>>>(g.N, Hin, l == 0 ? win : LD, gx_att_weight(m, l), win, P);
      if (l == 0) gcn_layer_kernel<true, true, KW><<<grid, kFwdThreads, smem, s>>>(g, Hin, m.W[l], m.b[l], win, wout, l == m.L - 1, m.bn, P, Hout);
      else gcn_layer_kernel<false, true, KW><<<grid, kFwdThreads, smem, s>>>(g, Hin, m.W[l], m.b[l], win, wout, l == m.L - 1, m.bn, P, Hout);
      continue;
    }
    if (l == 0 && smem > 48 * 1024) {
      const cudaError_t e = cudaFuncSetAttribute(gcn_layer_kernel<true, false, KW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return e;
    }
    if (l == 0) gcn_layer_kernel<true, false, KW><<<grid, kFwdThreads, smem, s>>>(g, Hin, m.W[l], m.b[l], win, wout, l == m.L - 1, m.bn, nullptr, Hout);
    else gcn_layer_kernel<false, false, KW><<<grid, kFwdThreads, smem, s>>>(g, Hin, m.W[l], m.b[l], win, wout, l == m.L - 1, m.bn, nullptr, Hout);
  }
  if (hd.k == 0) {
    readout_kernel<KW><<<grid, kFwdThreads, 0, s>>>(g.N, m.L, m.hid, m.emb, m.C, H, m.Wp, m.bp, pred, emb_out);
    return cudaGetLastError();
  }
  // head models: the concatenated rows into emb_out (no pred_model product: C = 0), then the head
  readout_kernel<KW><<<grid, kFwdThreads, 0, s>>>(g.N, m.L, m.hid, m.emb, 0, H, nullptr, nullptr, nullptr, emb_out);
  head_kernel<<<grid, kFwdThreads, (size_t)nwarps * 2 * gx_head_max_width(hd) * sizeof(float), s>>>(g.N, m.hid * (m.L - 1) + m.emb, m.C, hd,
                                                                                                      emb_out, pred);
  return cudaGetLastError();
}

}  // namespace

// H: workspace [L][N][gx_var_row_stride(hid, emb)] floats (device).  Layer 1 keeps one input row per warp in dynamic shared memory: 128 KB
// at the widest input (d = 4096), beyond the 48 KB a launch gets without opting in.  pred [N][C], emb_out [N][PD] or nullptr (device;
// required with an MLP head, hd.k > 0).  P: attention models' workspace [N][round_up(max(d, hid), 4)] floats (device), else unused.
cudaError_t gx_launch_model_forward(const GxGraphDev& g, const GxModelDev& m, const GxHeadDev& hd, float* H, float* pred, float* emb_out, float* P,
                                    cudaStream_t s) {
  if (hd.k > 0 && emb_out == nullptr) return cudaErrorInvalidValue;
  const int kw = gx_var_row_stride(m.hid, m.emb) / 32;
  if (kw == 1) return model_forward<1>(g, m, hd, H, pred, emb_out, P, s);
  if (kw == 2) return model_forward<2>(g, m, hd, H, pred, emb_out, P, s);
  if (kw == 4) return model_forward<4>(g, m, hd, H, pred, emb_out, P, s);
  return model_forward<8>(g, m, hd, H, pred, emb_out, P, s);
}
