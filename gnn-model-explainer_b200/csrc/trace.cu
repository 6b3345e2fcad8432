// trace.cu -- the per-epoch log of the optimisation (SURVEY 8 row a12: ExplainModule.loss terms and mask_density,
// explainer/explain.py:148-159,680-683,740-808), assembled from what the explainer kernels record while they run.
//
//   trace_finalize_kernel  combines the raw per-epoch terms written by the persistent explainer kernels (inner pairs, the
//                          explained node's own row) with the outer pairs' sums (outer_pairs_kernel<true>) into the columns
//                          GX_TR_* of include/gnnx.h.
//   offedge_kernel         the part of the reference's PRINTED loss that never influences the result: size and entropy are
//                          summed over all n^2 mask entries (explain.py:755-770), and the n^2 - E_d entries outside the
//                          sub-adjacency each follow a private scalar Adam recurrence driven by those two regularisers only.
//   offedge_graph_kernel   the same for padded graphs (graph mode): the max_nodes^2 entries of a graph's mask minus its directed
//                          edges -- padded rows and columns, non-edges, the diagonal -- normalised by max_nodes^2.
#include <algorithm>

#include "explain_common.cuh"

namespace {

__global__ void __launch_bounds__(128)
trace_finalize_kernel(const GxHparamsDev hp, const GxPlanArrays plan, int count, const GxExtra x) {
  const int64_t rows = (int64_t)count * x.epochs;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(r / x.epochs);
    const GxTask* T = plan.tasks + t;
    float* row = x.trace + r * GX_TRACE_COLS;
    if ((int)(r - (int64_t)t * x.epochs) >= hp.iters) {   // (cannot happen: a trace run executes every epoch)
      for (int k = 0; k < GX_TRACE_COLS; ++k) row[k] = 0.f;
      continue;
    }
    double oS = 0.0, oH = 0.0, oL = 0.0, oD = 0.0;
    if (x.tr_outer != nullptr) { const double* o = x.tr_outer + r * 4; oS = o[0]; oH = o[1]; oL = o[2]; oD = o[3]; }
    const double nn = (double)T->n_norm * (double)T->n_norm;
    const float sS = row[0], pred = row[1], sH = row[2], sL = row[3], sD = row[4], feat = row[5], pgt = row[7];
    const float size = (float)((double)hp.c_size * ((double)sS + oS));
    const float ent = (float)((double)hp.c_ent * ((double)sH + oH) / nn);
    const float lap = (float)((double)hp.c_lap * ((double)sL + oL) / nn);
    // mask_density (explain.py:680-683) divides by sum(adj): the self loops count there, the masked diagonal contributes nothing
    const int adj_sum = T->e_d + T->loops;
    const float dens = adj_sum > 0 ? (float)(((double)sD + oD) / (double)adj_sum) : 0.f;
    row[GX_TR_LOSS_EDGES] = pred + size + lap + ent + feat;   // explain.py:808, the sums restricted to the edge entries
    row[GX_TR_PRED] = pred; row[GX_TR_SIZE] = size; row[GX_TR_ENT] = ent; row[GX_TR_LAP] = lap;
    row[GX_TR_FEAT] = feat; row[GX_TR_DENSITY] = dens; row[GX_TR_PGT] = pgt;
  }
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One off-edge entry's trajectory: per epoch e, warp sums of (sigmoid(M_e), H(sigmoid(M_e))) over the active lanes into s_acc[e],
// then the entry's Adam step on size + entropy (no Laplacian: an off-edge entry never reaches the masked adjacency).
// ent_over_nn = c_ent / n^2 with the n of the reference's dense mask.
__device__ __forceinline__ void offedge_trajectory(const GxHparamsDev& hp, bool act, float M, int epochs, float ent_over_nn, bool ieee,
                                                   int lane, double* s_acc) {
  float mo = 0.f, vo = 0.f;
  float S = sigmoid_f(M);
  for (int e = 0; e < epochs; ++e) {
    const double cs = warp_sum_d(act ? (double)S : 0.0);
    const double ch = warp_sum_d(act ? (double)bern_entropy(S) : 0.0);
    if (lane == 0) { atomicAdd(&s_acc[2 * e], cs); atomicAdd(&s_acc[2 * e + 1], ch); }
    const float2 tab = __ldg(hp.adam_tab + e);
    const float gM = S * (1.f - S) * (hp.c_size - ent_over_nn * M);
    mo = mo + (gM - mo) * hp.one_minus_b1;
    vo = vo * hp.b2 + hp.one_minus_b2 * gM * gM;
    M = M - adam_delta_fast(mo, vo, tab.x, tab.y, 1.0f / tab.y, hp.eps, ieee);
    S = sigmoid_fast(M, ieee);
  }
}

// grid = (chunks, tasks of the launch; plan.tasks starts at its first).  out[t][e][0..1] += (sum sigmoid(M_e), sum H(sigmoid(M_e))) over the off-edge entries of task t,
// M_e = the entry after e Adam steps (what epoch e's loss sees).
__global__ void __launch_bounds__(256)
offedge_kernel(const GxHparamsDev hp, const GxPlanArrays plan, int epochs, const int64_t* __restrict__ dense_off,
               const float* __restrict__ m0_dense, double* __restrict__ out) {
  extern __shared__ double s_acc[];   // [epochs][2]
  const bool ieee = (hp.flags & GX_HP_IEEE_EDGE) != 0;
  const int t = blockIdx.y;
  const GxTask* T = plan.tasks + t;
  const int n = T->n;
  const int64_t nn = (int64_t)n * n;
  const int32_t* srp = plan.sub_rowptr + T->rp_off;
  const int32_t* scol = plan.sub_col + T->edge_off;
  const float* M0 = m0_dense + dense_off[t];
  const float ent_over_nn = hp.c_ent / ((float)n * (float)n);
  const int lane = threadIdx.x & 31;
  for (int k = threadIdx.x; k < epochs * 2; k += blockDim.x) s_acc[k] = 0.0;
  __syncthreads();
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < nn; base += (int64_t)gridDim.x * blockDim.x) {
    const int64_t idx = base + threadIdx.x;
    bool act = idx < nn;
    float M = 0.f;
    if (act) {
      const int r = (int)(idx / n), c = (int)(idx - (int64_t)r * n);
      int lo = srp[r], hi = srp[r + 1];
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (scol[mid] < c) lo = mid + 1; else hi = mid; }
      act = !(lo < srp[r + 1] && scol[lo] == c);   // entries of the sub-adjacency belong to the explainer kernels
      M = M0[idx];
    }
    offedge_trajectory(hp, act, M, epochs, ent_over_nn, ieee, lane, s_acc);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < epochs * 2; k += blockDim.x) atomicAdd(out + (int64_t)t * epochs * 2 + k, s_acc[k]);
}

// Graph mode, grid = (chunks, graphs of the launch; plan.tasks, m0_dense and out start at its first): planned graph t (T->node = g) owns the dense max_nodes x max_nodes block at m0_dense + t * nf^2.
// Its directed edges (the batch CSR rows of g, global offsets) belong to the explainer kernels; every other entry is summed.  The
// entropy factor is 1 / max_nodes^2 (T->n_norm, the padded size of the reference's tensors), not 1 / T->n: in a graph plan T->n
// counts only the rows that have an edge.
__global__ void __launch_bounds__(256)
offedge_graph_kernel(const GxHparamsDev hp, const GxPlanArrays plan, const GxGraphBatchDev gb, int epochs,
                     const float* __restrict__ m0_dense, double* __restrict__ out) {
  extern __shared__ double s_acc[];   // [epochs][2]
  const bool ieee = (hp.flags & GX_HP_IEEE_EDGE) != 0;
  const int t = blockIdx.y;
  const GxTask* T = plan.tasks + t;
  const int nf = T->n_norm;
  const int64_t nn = (int64_t)nf * nf;
  const int32_t* rp = gb.rowptr + (int64_t)T->node * gb.max_nodes;
  const float* M0 = m0_dense + (int64_t)t * nn;
  const float ent_over_nn = hp.c_ent / ((float)nf * (float)nf);
  const int lane = threadIdx.x & 31;
  for (int k = threadIdx.x; k < epochs * 2; k += blockDim.x) s_acc[k] = 0.0;
  __syncthreads();
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < nn; base += (int64_t)gridDim.x * blockDim.x) {
    const int64_t idx = base + threadIdx.x;
    bool act = idx < nn;
    float M = 0.f;
    if (act) {
      const int r = (int)(idx / nf), c = (int)(idx - (int64_t)r * nf);
      const int end = rp[r + 1];
      int lo = rp[r], hi = end;
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (gb.col[mid] < c) lo = mid + 1; else hi = mid; }
      act = !(lo < end && gb.col[lo] == c);   // the graph's directed edges belong to the explainer kernels
      M = M0[idx];
    }
    offedge_trajectory(hp, act, M, epochs, ent_over_nn, ieee, lane, s_acc);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < epochs * 2; k += blockDim.x) atomicAdd(out + (int64_t)t * epochs * 2 + k, s_acc[k]);
}

constexpr int kMaxGridY = 65535;   // gridDim.y limit

}  // namespace

cudaError_t gx_launch_trace_finalize(const GxHparamsDev& hp, const GxPlanArrays& plan, int count, const GxExtra& x, cudaStream_t s) {
  const int64_t rows = (int64_t)count * x.epochs;
  const int grid = (int)((rows + 127) / 128 < GX_GRID_CAP ? (rows + 127) / 128 : GX_GRID_CAP);
  trace_finalize_kernel<<<grid > 0 ? grid : 1, 128, 0, s>>>(hp, plan, count, x);
  return cudaGetLastError();
}

cudaError_t gx_launch_offedge(const GxHparamsDev& hp, const GxPlanArrays& plan, int count, int epochs, const int64_t* dense_off,
                              const float* m0_dense, double* out, cudaStream_t s) {
  const size_t smem = (size_t)epochs * 2 * sizeof(double);
  if (smem > 48 * 1024) return cudaErrorInvalidValue;
  // one task per blockIdx.y: batches beyond the grid's y limit go in slices, each seeing the plan from its first task on
  for (int t0 = 0; t0 < count; t0 += kMaxGridY) {
    GxPlanArrays p = plan;
    p.tasks += t0;
    dim3 grid(32, std::min(kMaxGridY, count - t0));
    offedge_kernel<<<grid, 256, smem, s>>>(hp, p, epochs, dense_off + t0, m0_dense, out + (int64_t)t0 * epochs * 2);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t gx_launch_offedge_graphs(const GxHparamsDev& hp, const GxPlanArrays& plan, const GxGraphBatchDev& gb, int count, int epochs,
                                     const float* m0_dense, double* out, cudaStream_t s) {
  const size_t smem = (size_t)epochs * 2 * sizeof(double);
  if (smem > 48 * 1024) return cudaErrorInvalidValue;
  const int64_t nn = (int64_t)gb.max_nodes * gb.max_nodes;
  for (int t0 = 0; t0 < count; t0 += kMaxGridY) {   // as gx_launch_offedge: slices of at most kMaxGridY graphs
    GxPlanArrays p = plan;
    p.tasks += t0;
    dim3 grid(32, std::min(kMaxGridY, count - t0));
    offedge_graph_kernel<<<grid, 256, smem, s>>>(hp, p, gb, epochs, m0_dense + t0 * nn, out + (int64_t)t0 * epochs * 2);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}
