// explain_dense.cu -- Explainer.explain(..., unconstrained=True) (explain.py:97-146,209-211; ExplainModule.forward explain.py:688-692,
// loss :740-808, mask_density :680-683), node mode and graph mode, every model and optimiser of the variant kernels.
//
// With unconstrained=True the forward's adjacency is the DENSE mask a = sym(sigmoid(M)) (.) (1 - I), not multiplied by adj, and the
// features are not masked.  Every off-diagonal entry of M therefore carries gradient and the problem is dense:
//   * forward   Z_l = a H_{l-1}                 (n x n) (n x w_in)
//   * backward  dL/dH_l = a^T dZ_{l+1} = a dZ_{l+1}   (a is symmetric)
//   * pairs     dA = sum_l dZ_l H_{l-1}^T       one (n x K) (K x n) product over the concatenated layers (GxDenseLayout)
// These three products run on the tensor cores with the 3xTF32 split (mma_tf32.cuh, FP32-grade accuracy); the per-row steps (dense
// W, normalise, bn, readout tail) and the optimiser updates are explain_var_common.cuh's.  Node mode computes all n rows at every
// layer and reads out row node_idx_new; graph mode reads out the per-layer max-pool over all max_nodes padded rows (no edge-less
// constant: every row is connected through the mask).  F is moved by feat_size alone.  Diagonal entries follow the regulariser-only
// recurrence; they reach the printed loss only.
// Layout: one persistent CTA per task from the largest-first work queue, the task's state in a per-CTA global slab.
// Phases per epoch (one __syncthreads each): (Z_l | F_l) x L | S | (Z | B_l) x L | G | P.
#include "explain_var_common.cuh"
#include "mma_tf32.cuh"

namespace {

struct DenseArgs {
  const int32_t* order;
  int32_t ntasks;
  int32_t* counter;
  float* gws;
  int64_t gws_stride_words;
  int32_t graph_mode;
  GxGraphDev g;
  GxGraphBatchDev gb;
  GxModelDev m;
  GxHparamsDev hp;
  GxPlanArrays plan;
  GxDenseIo io;
  GxHeadDev hd;   // MLP prediction head (k = 0: none)
};

// shared memory: the variant kernels' carve-up + the arg-max row of every pooled feature (graph mode) + reduction scratch
struct DenseSmem { VarSmem S; int arg, red, total; };
__host__ __device__ inline DenseSmem dense_smem(int d, int L, int hid, int emb, int C, int nwarps, const GxHeadDev& hd) {
  DenseSmem D;
  D.S = var_smem(d, L, hid, emb, C, nwarps, 0, hd);
  const int PD = hid * (L - 1) + emb;
  D.arg = D.S.total;
  D.red = D.arg + gx_round_up(PD, 4);
  D.total = D.red + nwarps * 4 * 2;   // 4 doubles per warp
  return D;
}

// C[i][j] = sum_{k < K} A[i * lda + k] B[k * bk + j * bj] for i < M, j < N, on the tensor cores (3xTF32).  Each warp of the CTA
// takes 16 x 32 output tiles; operands are read from the slab (L2) and zero padded at the edges.
__device__ void dense_mma(const float* __restrict__ A, int64_t lda, const float* __restrict__ B, int64_t bk, int64_t bj,
                          float* __restrict__ Cm, int64_t ldc, int M, int N, int K, int warp, int nwarps, int lane) {
  constexpr int NTL = 4;
  const int g = lane >> 2, t4 = lane & 3;
  const int mt = (M + 15) / 16, nt = (N + 8 * NTL - 1) / (8 * NTL);
  for (int tile = warp; tile < mt * nt; tile += nwarps) {
    const int i0 = (tile / nt) * 16, j0 = (tile % nt) * (8 * NTL);
    const int ra = i0 + g, rb = i0 + g + 8;
    float cb[NTL][4], cs[NTL][4];
#pragma unroll
    for (int s = 0; s < NTL; ++s)
#pragma unroll
      for (int c = 0; c < 4; ++c) { cb[s][c] = 0.f; cs[s][c] = 0.f; }
#pragma unroll 2
    for (int k0 = 0; k0 < K; k0 += 8) {
      const int ka = k0 + t4, kb = k0 + t4 + 4;
      const float av0 = (ra < M && ka < K) ? A[ra * lda + ka] : 0.f;
      const float av1 = (rb < M && ka < K) ? A[rb * lda + ka] : 0.f;
      const float av2 = (ra < M && kb < K) ? A[ra * lda + kb] : 0.f;
      const float av3 = (rb < M && kb < K) ? A[rb * lda + kb] : 0.f;
      uint32_t ahi[4], alo[4];
      tf32_split(av0, ahi[0], alo[0]); tf32_split(av1, ahi[1], alo[1]);
      tf32_split(av2, ahi[2], alo[2]); tf32_split(av3, ahi[3], alo[3]);
#pragma unroll
      for (int s = 0; s < NTL; ++s) {
        const int j = j0 + 8 * s + g;
        const float b0 = (ka < K && j < N) ? B[ka * bk + j * bj] : 0.f;
        const float b1 = (kb < K && j < N) ? B[kb * bk + j * bj] : 0.f;
        uint32_t bh0, bl0, bh1, bl1;
        tf32_split(b0, bh0, bl0); tf32_split(b1, bh1, bl1);
        mma_tf32(cs[s], alo, bh0, bh1);
        mma_tf32(cb[s], ahi, bh0, bh1);
        mma_tf32(cs[s], ahi, bl0, bl1);
      }
    }
#pragma unroll
    for (int s = 0; s < NTL; ++s) {
      const int c0 = j0 + 8 * s + 2 * t4;
      if (ra < M) {
        if (c0 < N) Cm[ra * ldc + c0] = cb[s][0] + cs[s][0];
        if (c0 + 1 < N) Cm[ra * ldc + c0 + 1] = cb[s][1] + cs[s][1];
      }
      if (rb < M) {
        if (c0 < N) Cm[rb * ldc + c0] = cb[s][2] + cs[s][2];
        if (c0 + 1 < N) Cm[rb * ldc + c0 + 1] = cb[s][3] + cs[s][3];
      }
    }
  }
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <bool kBn, int KW>
__global__ void __launch_bounds__(kVarThreads) explain_dense_kernel(const DenseArgs A) {
  extern __shared__ __align__(16) float sm[];
  __shared__ int s_task;
  __shared__ float s_pgt;
  constexpr int NT = kVarThreads, nwarps = NT / 32;
  constexpr int VW = 32 * KW;   // row stride of every hidden-width array
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const GxModelDev& m = A.m;
  const GxHparamsDev& hp = A.hp;
  const GxDenseIo& io = A.io;
  const bool graph = A.graph_mode != 0;
  const int d = m.d, C = m.C, L = m.L, hid = m.hid, embw = m.emb;
  const int dp = gx_round_up(d, 4);
  const int PD = hid * (L - 1) + embw;
  const bool ieee = (hp.flags & GX_HP_IEEE_EDGE) != 0;
  const GxHeadDev& hd = A.hd;
  const DenseSmem DS = dense_smem(d, L, hid, embw, C, nwarps, hd);
  const VarSmem& S = DS.S;
  float* const sF = sm + S.sF; float* const Fm = sm + S.F; float* const mF = sm + S.mF; float* const vF = sm + S.vF;
  float* const zs = sm + S.zs + warp * S.zlen;
  float* const emb = sm + S.emb; float* const dEmb = sm + S.dEmb; float* const logit = sm + S.logit;
  int* const arg = reinterpret_cast<int*>(sm + DS.arg);
  double* const red = reinterpret_cast<double*>(sm + DS.red);
  const bool wp_smem = gx_head_words(hd, PD, C) <= GX_WP_SMEM_MAX;
  const float* const Wpp = wp_smem ? sm + S.Wp : m.Wp;
  const float* const bpp = wp_smem ? sm + S.Wp + C * PD : m.bp;
  auto win_of = [&](int l) { return l == 0 ? d : hid; };            // l = 0 .. L-1
  auto wout_of = [&](int l) { return l == L - 1 ? embw : hid; };
  // sums of v over the CTA (every thread calls; the result is valid in thread 0)
  auto block_sum4 = [&](double (&v)[4]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) { const double w = warp_sum_d(v[k]); if (lane == 0) red[warp * 4 + k] = w; }
    __syncthreads();
    if (tid == 0)
      for (int k = 0; k < 4; ++k) { double t = 0.0; for (int w = 0; w < nwarps; ++w) t += red[w * 4 + k]; v[k] = t; }
    __syncthreads();
  };

  const float* Wl[GX_MAX_LAYERS];   // conv weights: shared memory when they fit, else global (L2 resident)
  var_stage_model(m, hd, S, sm, Wl, tid, NT);
  float* const slab = A.gws + (int64_t)blockIdx.x * A.gws_stride_words;

  for (;;) {
    int task_id;
    if (!var_next_task(A, s_task, tid, task_id)) break;
    const GxTask* __restrict__ Tp = A.plan.tasks + task_id;
    const int n = graph ? A.gb.max_nodes : Tp->n;
    const int r = graph ? 0 : Tp->idx_new;
    const int gt = Tp->gt_label, key = Tp->node;
    const int adj_sum = Tp->e_d + Tp->loops;   // sum(adj) of mask_density (explain.py:680-683): self loops count, their mask entry is 0
    const int64_t nn64 = (int64_t)n * n;
    const GxDenseLayout Lo = gx_make_dense_layout(n, d, L, VW);
    const int KH = Lo.kh, ZW = Lo.zw;
    float* const Mv = slab + Lo.M; float* const mv = slab + Lo.m; float* const vv = slab + Lo.v;
    float* const a = slab + Lo.a; float* const Gp = slab + Lo.G;
    float* const Hc = slab + Lo.Hc; float* const dZc = slab + Lo.dZc; float* const Z = slab + Lo.Z;
    auto off = [&](int l) { return l == 0 ? 0 : Lo.off1 + (l - 1) * VW; };   // column of H_l (and of dZ_{l+1}) in Hc / dZc
    auto Yh = [&](int l) { return slab + Lo.Yh + (int64_t)(l - 1) * n * VW; };
    auto Hl = [&](int l) { return Hc + off(l); };
    auto qn = [&](int l) { return slab + Lo.q + (int64_t)(l - 1) * n; };
    auto istd = [&](int l) { return slab + Lo.istd + (int64_t)(l - 1) * n; };
    // this task's rows: canonical (ascending-id) k-hop set in node mode, the padded graph in graph mode
    const int32_t* __restrict__ nbrs = graph ? nullptr : A.plan.nbrs + Tp->node_off;
    auto xrow = [&](int i) { return graph ? A.gb.feat + ((int64_t)key * n + i) * d : A.g.feat + (int64_t)nbrs[i] * d; };
    auto ylab = [&](int i) { return graph ? 0.f : (float)__ldg(A.g.pred_label + nbrs[i]); };
    // the sub-adjacency slots the result is returned at: rows erp[i] .. erp[i+1], column ecol[e], slot e - ebase
    const int32_t* __restrict__ erp = graph ? A.gb.rowptr + (int64_t)key * n : A.plan.sub_rowptr + Tp->rp_off;
    const int32_t* __restrict__ ecol = graph ? A.gb.col : A.plan.sub_col + Tp->edge_off;
    const int64_t ebase = graph ? erp[0] : 0;
    const int64_t edge_off = Tp->edge_off;
    const float nnf = (float)n * (float)n;
    const float ent_over_nn = hp.c_ent / nnf, lap_over_nn = hp.c_lap / nnf;

    // ---------------------------------------------------------------- init: M0, optimiser state, a, X
    {
      const float m0_std = sqrtf(2.0f / (float)n);   // gain('relu') * sqrt(2/(n+n)) (explain.py:647-651), n = the padded size in graph mode
      const int64_t m0_off = io.m0 != nullptr ? io.dense_off[task_id] : 0;
      for (int64_t idx = tid; idx < nn64; idx += NT) {
        Mv[idx] = var_init_param(hp, io.m0, m0_off + idx, (uint32_t)key, (uint32_t)idx, m0_std);
        mv[idx] = 0.f; vv[idx] = 0.f;
      }
      for (int64_t idx = tid; idx < (int64_t)n * KH; idx += NT) { Hc[idx] = 0.f; dZc[idx] = 0.f; }
      for (int f = tid; f < dp; f += NT) { sF[f] = 0.5f; Fm[f] = 0.f; mF[f] = 0.f; vF[f] = 0.f; }   // feat_mask = 0 (explain.py:633-643)
    }
    __syncthreads();
    for (int64_t idx = tid; idx < nn64; idx += NT) {
      const int i = (int)(idx / n), j = (int)(idx - (int64_t)i * n);
      a[idx] = i == j ? 0.f : 0.5f * (sigmoid_fast(Mv[idx], ieee) + sigmoid_fast(Mv[(int64_t)j * n + i], ieee));   // explain.py:688-692
    }
    for (int i = warp; i < n; i += nwarps) {
      const float* x = xrow(i);
      for (int f = lane; f < d; f += 32) Hc[(int64_t)i * KH + f] = __ldg(x + f);
    }
    __syncthreads();
    // the returned array: masked_adj[0] * sub_adj at the sub-adjacency slots (explain.py:209-211); optionally the whole a.  With a trace,
    // dens = sum of a over those slots (mask_density keeps the constrained _masked_adj, explain.py:680-683)
    auto edges_pass = [&](bool emit) -> double {
      double s = 0.0;
      for (int i = warp; i < n; i += nwarps)
        for (int e = erp[i] + lane; e < erp[i + 1]; e += 32) {
          const float v = a[(int64_t)i * n + ecol[e]];
          s += (double)v;
          if (emit) io.out_mask[edge_off + (e - ebase)] = v;
        }
      if (emit && io.out_dense != nullptr)
        for (int64_t idx = tid; idx < nn64; idx += NT) io.out_dense[io.dense_off[task_id] + idx] = a[idx];
      return s;
    };
    if (hp.out_iter == 0) edges_pass(true);

    for (int it = 1; it <= hp.iters; ++it) {
      // ---------------------------------------------------------------- forward: Z_l = a H_{l-1}, then every row   (models.py:58-80)
      for (int l = 1; l <= L; ++l) {
        const int win = win_of(l - 1), wout = wout_of(l - 1);
        dense_mma(a, n, Hc + off(l - 1), KH, 1, Z, ZW, n, win, n, warp, nwarps, lane);
        __syncthreads();
        const float* const Ws = Wl[l - 1]; const float* const bsm = sm + S.b[l - 1];
        for (int i = warp; i < n; i += nwarps) {
          for (int f = lane; f < win; f += 32) zs[f] = Z[(int64_t)i * ZW + f];
          var_row_forward<kBn, KW>(zs, win, Ws, wout, bsm, l, L, i, Yh, Hl, KH, qn, istd, lane);
        }
        __syncthreads();
      }
      // ---------------------------------------------------------------- S: readout, softmax, dEmb   (explain.py:709-714)
      if (graph) {
        var_max_pool(L, hid, PD, n, Hl, KH, nullptr, 0, emb, arg, tid, NT);   // over all padded rows
      } else if (warp == 0) {
        for (int l = 1; l <= L; ++l)
          for (int c = lane; c < wout_of(l - 1); c += 32) emb[hid * (l - 1) + c] = Hc[(int64_t)r * KH + off(l) + c];
      }
      __syncthreads();
      var_readout_tail(emb, hd, wp_smem ? sm + S.Wp : hd.W, Wpp, bpp, C, PD, gt, sm + S.hx, sm + S.hg, logit, dEmb, tid, NT);
      __syncthreads();
      if (warp == 0) {
        if (lane == 0) s_pgt = logit[gt] + 1.f;
        if (io.trace_pred != nullptr)
          for (int c = lane; c < C; c += 32) io.trace_pred[((int64_t)task_id * io.epochs + (it - 1)) * C + c] = logit[c] + (c == gt ? 1.f : 0.f);
      }
      __syncthreads();
      // ---------------------------------------------------------------- backward: dL/dH_l = a dZ_{l+1} + the readout's share
      for (int l = L; l >= 1; --l) {
        const int win = win_of(l - 1), wout = wout_of(l - 1);
        const int koff = hid * (l - 1);
        if (l < L) {
          dense_mma(a, n, dZc + off(l), KH, 1, Z, ZW, n, wout, n, warp, nwarps, lane);
          __syncthreads();
        }
        const float* const Ws = Wl[l - 1];
        for (int i = warp; i < n; i += nwarps) {
          float g[KW], yh[KW];
#pragma unroll
          for (int k = 0; k < KW; ++k) {
            const int c = lane + 32 * k;
            g[k] = (l < L && c < wout) ? Z[(int64_t)i * ZW + c] : 0.f;
            if (c < wout && (graph ? arg[koff + c] == i : i == r)) g[k] += dEmb[koff + c];
            yh[k] = Yh(l)[(int64_t)i * VW + c];
          }
          var_row_backward<kBn, KW>(g, yh, l, L, i, Hl, KH, qn, istd, wout, zs, lane);
          if (l == 1) {   // dZ_1 = dY W_1^T, width d (the features are not masked: no dL/dsF)
            for (int f = lane; f < d; f += 32) {
              float t = 0.f;
              for (int c = 0; c < wout; ++c) t = fmaf(zs[c], Ws[f * wout + c], t);
              dZc[(int64_t)i * KH + f] = t;
            }
          } else {
            var_hidden_dz<KW>(zs, Ws, win, wout, dZc + (int64_t)i * KH + off(l - 1), lane);
          }
          __syncwarp();
        }
        __syncthreads();
      }
      // ---------------------------------------------------------------- G = sum_l dZ_l H_{l-1}^T (= dL/dA without the Laplacian term)
      dense_mma(dZc, KH, Hc, 1, KH, Gp, n, n, n, Lo.k_pair, warp, nwarps, lane);
      __syncthreads();
      // ---------------------------------------------------------------- P: one thread per unordered pair i <= j, optimiser step, next a
      const float2 tab = __ldg(hp.adam_tab + (it - 1));
      const float step = tab.x, bc2s = tab.y, bc2s_inv = 1.0f / tab.y;
      double tr[4] = {0.0, 0.0, 0.0, 0.0};   // sum sigmoid(M), sum H(sigmoid(M)) over all n^2 entries, sum a_ij (y_i - y_j)^2 over i < j, sum sF
      for (int64_t idx = tid; idx < nn64; idx += NT) {
        const int i = (int)(idx / n), j = (int)(idx - (int64_t)i * n);
        if (j < i) continue;
        if (i == j) {   // diagonal: masked out of the forward, moved by size and entropy only
          float M = Mv[idx], mo = mv[idx], vo = vv[idx];
          const float Sd = sigmoid_fast(M, ieee);
          if (io.trace != nullptr) { tr[0] += (double)Sd; tr[1] += (double)bern_entropy(Sd); }
          var_edge_update(hp, Sd * (1.f - Sd) * (hp.c_size - ent_over_nn * M), M, mo, vo, step, bc2s, bc2s_inv, ieee);
          Mv[idx] = M; mv[idx] = mo; vv[idx] = vo;
          continue;
        }
        const int64_t ji = (int64_t)j * n + i;
        float Mi = Mv[idx], Mj = Mv[ji], mi = mv[idx], mj = mv[ji], vi = vv[idx], vj = vv[ji];
        const float Si = sigmoid_fast(Mi, ieee), Sj = sigmoid_fast(Mj, ieee);
        const float yd = ylab(i) - ylab(j);
        if (io.trace != nullptr) {
          tr[0] += (double)Si + (double)Sj;
          tr[1] += (double)bern_entropy(Si) + (double)bern_entropy(Sj);
          tr[2] += (double)a[idx] * (double)(yd * yd);
        }
        // d/dA_ij + d/dA_ji of y^T (D - A_m) y / n^2 (explain.py:780-793) and of the GCN; sym_mask = (S + S^T)/2 (explain.py:689)
        const float Gd = 0.5f * (lap_over_nn * yd * yd + Gp[idx] + Gp[ji]);
        const float gi = Si * (1.f - Si) * (Gd + hp.c_size - ent_over_nn * Mi);
        const float gj = Sj * (1.f - Sj) * (Gd + hp.c_size - ent_over_nn * Mj);
        var_edge_update(hp, gi, Mi, mi, vi, step, bc2s, bc2s_inv, ieee);
        var_edge_update(hp, gj, Mj, mj, vj, step, bc2s, bc2s_inv, ieee);
        Mv[idx] = Mi; mv[idx] = mi; vv[idx] = vi;
        Mv[ji] = Mj; mv[ji] = mj; vv[ji] = vj;
        const float an = 0.5f * (sigmoid_fast(Mi, ieee) + sigmoid_fast(Mj, ieee));
        a[idx] = an; a[ji] = an;
      }
      for (int f = tid; f < d; f += NT) {   // F: gradient of feat_size = mean sigmoid(F) only (explain.py:763-766)
        const float s = sF[f];
        if (io.trace != nullptr) tr[3] += (double)s;
        float mf = mF[f], vf = vF[f], Fv = Fm[f];
        var_feat_update(hp, s * (1.f - s) * (hp.c_feat_size / (float)d), Fv, mf, vf, step, bc2s);
        mF[f] = mf; vF[f] = vf; Fm[f] = Fv;
        sF[f] = sigmoid_f(Fv);
      }
      __syncthreads();
      const bool emit = it == hp.out_iter;   // the mask built after this update is the one the reference returns
      if (emit || io.trace != nullptr) {
        double dens[4] = {edges_pass(emit), 0.0, 0.0, 0.0};
        if (io.trace != nullptr) {
          block_sum4(tr);
          block_sum4(dens);
          if (tid == 0) {   // the columns print_training prints and the terms of the loss (explain.py:740-808), all n^2 entries
            float* row = io.trace + ((int64_t)task_id * io.epochs + (it - 1)) * GX_TRACE_COLS;
            const double nn = (double)n * (double)n;
            const float pred = -logf(s_pgt);
            const float size = (float)((double)hp.c_size * tr[0]);
            const float ent = (float)((double)hp.c_ent * tr[1] / nn);
            const float lap = (float)((double)hp.c_lap * tr[2] / nn);
            const float feat = (float)((double)hp.c_feat_size * tr[3] / (double)d);
            row[GX_TR_LOSS_EDGES] = pred + size + lap + ent + feat;
            row[GX_TR_PRED] = pred; row[GX_TR_SIZE] = size; row[GX_TR_ENT] = ent; row[GX_TR_LAP] = lap; row[GX_TR_FEAT] = feat;
            row[GX_TR_DENSITY] = adj_sum > 0 ? (float)(dens[0] / (double)adj_sum) : 0.f;
            row[GX_TR_PGT] = s_pgt;
          }
        }
      }
      __syncthreads();
    }
  }
}

}  // namespace

int gx_dense_smem_bytes(int d, int L, int hid, int emb, int C, const GxHeadDev& hd) { return dense_smem(d, L, hid, emb, C, kVarThreads / 32, hd).total * 4; }

// co-resident CTAs per SM of the model's instantiation (sizes the persistent grid); 0 on error
int gx_dense_ctas_per_sm(const GxModelDev& m, const GxHeadDev& hd) {
  const int bytes = gx_dense_smem_bytes(m.d, m.L, m.hid, m.emb, m.C, hd);
  int n = 0;
  var_dispatch(m, [&](auto bn, auto kw) { n = var_ctas_per_sm(explain_dense_kernel<decltype(bn)::value, decltype(kw)::value>, bytes); return cudaSuccess; });
  return n;
}

cudaError_t gx_launch_explain_dense(const GxExplainLaunch& cfg, int graph_mode, const GxGraphDev& g, const GxGraphBatchDev& gb,
                                    const GxModelDev& m, const GxHeadDev& hd, const GxHparamsDev& hp, const GxPlanArrays& plan,
                                    const GxDenseIo& io, cudaStream_t s) {
  DenseArgs args;
  args.order = cfg.order; args.ntasks = cfg.ntasks; args.counter = cfg.counter;
  args.gws = cfg.gws; args.gws_stride_words = cfg.gws_stride_words;
  args.graph_mode = graph_mode; args.g = g; args.gb = gb; args.m = m; args.hp = hp; args.plan = plan; args.io = io; args.hd = hd;
  const int bytes = gx_dense_smem_bytes(m.d, m.L, m.hid, m.emb, m.C, hd);
  return var_dispatch(m, [&](auto bn, auto kw) {
    return var_launch(explain_dense_kernel<decltype(bn)::value, decltype(kw)::value>, args, cfg.grid, bytes, s);
  });
}
