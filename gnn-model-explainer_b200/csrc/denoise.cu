// denoise.cu -- the thresholding step of io_utils.denoise_graph (utils/io_utils.py:193-231), on the packed edge masks, on device.
//
// The consumers of the masks (explain.py:238-288,308: denoise_graph(masked_adj, ..., threshold_num=20)) keep the
// 2*threshold_num largest entries of the dense symmetric mask ("edges are repeated twice in adj"): threshold = the
// min(2k, #positive)-th largest positive value, kept = entries >= threshold.  Here that is a per-task radix select over the
// E_t packed values (4 passes of an 8-bit histogram on the float bits: positive floats order like unsigned integers) and an
// order-preserving compaction -- one CTA per explained node.  It is also the payload policy of the multi-GPU gather for graphs
// whose full masks cannot be gathered (BASELINE configs[4]: 3.4 GB of masks per 132 nodes; the top-k lists are 132 x 40 entries).
// The edges mode (gx_denoise_topk_edges) shares the select and the compaction: it keeps the row < col half of the surviving slots
// and writes them as global (u, v) pairs, so a gathered list needs no plan to be read.
#include "gnnx_internal.cuh"

namespace {

constexpr int DN_THREADS = 256;

// Row of canonical slot e of a task: the last r with rp[r] <= e (rp = the task's n+1 sub_rowptr entries, rp[0] = 0 <= e < rp[n]).
__device__ __forceinline__ int slot_row(const int32_t* __restrict__ rp, int n, int e) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (rp[mid] <= e) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// kEdges = false (gx_denoise_topk): out_idx[t*cap + i] = the i-th kept slot (task-local), every kept slot.
// kEdges = true (gx_denoise_topk_edges): only kept slots with row < col, written as the global pair (nbrs[row], nbrs[col]) at
// out_idx[(t*cap + i)*2 ..]; the kernels write both directions of an edge with the same bits, so the other half adds nothing.
template <bool kEdges>
__global__ void __launch_bounds__(DN_THREADS)
denoise_topk_kernel(const GxPlanArrays plan, int count, const float* __restrict__ edge_mask, int k2, int cap,
                    float* __restrict__ out_thr, int32_t* __restrict__ out_cnt, int32_t* __restrict__ out_idx,
                    float* __restrict__ out_vals) {
  __shared__ int s_hist[256];
  __shared__ unsigned s_prefix;
  __shared__ int s_want, s_npos, s_base;
  __shared__ int s_wcnt[DN_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int t = blockIdx.x; t < count; t += gridDim.x) {
    const GxTask* T = plan.tasks + t;
    const int E = T->e_d;
    const float* v = edge_mask + T->edge_off;
    // positives
    if (tid == 0) s_npos = 0;
    __syncthreads();
    int c = 0;
    for (int e = tid; e < E; e += DN_THREADS) c += v[e] > 0.f ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0 && c) atomicAdd(&s_npos, c);
    __syncthreads();
    const int npos = s_npos;
    const int want0 = npos < k2 ? npos : k2;   // rank (from the top) of the threshold value
    if (want0 == 0) {   // no positive entry: nothing to keep (the reference's np.sort(...)[-0] raises here)
      if (tid == 0) { out_thr[t] = INFINITY; out_cnt[t] = 0; }
      __syncthreads();
      continue;
    }
    if (tid == 0) { s_prefix = 0u; s_want = want0; }
    __syncthreads();
    for (int pass = 3; pass >= 0; --pass) {
      const int shift = 8 * pass;
      const unsigned himask = pass == 3 ? 0u : (0xFFFFFFFFu << (shift + 8));
      s_hist[tid] = 0;
      __syncthreads();
      const unsigned prefix = s_prefix;
      for (int e = tid; e < E; e += DN_THREADS) {
        const float x = v[e];
        if (x > 0.f) {
          const unsigned b = __float_as_uint(x);
          if ((b & himask) == prefix) atomicAdd(&s_hist[(b >> shift) & 255u], 1);
        }
      }
      __syncthreads();
      if (tid == 0) {   // walk the buckets from the top until the wanted rank falls inside one
        int want = s_want, bkt = 255;
        for (; bkt > 0; --bkt) {
          if (s_hist[bkt] >= want) break;
          want -= s_hist[bkt];
        }
        s_want = want;
        s_prefix = prefix | ((unsigned)bkt << shift);
      }
      __syncthreads();
    }
    const float thr = __uint_as_float(s_prefix);
    // order-preserving compaction of the slots with value >= threshold
    if (tid == 0) s_base = 0;
    __syncthreads();
    const int32_t* rp = plan.sub_rowptr + T->rp_off;
    const int32_t* col = plan.sub_col + T->edge_off;
    const int32_t* nb = plan.nbrs + T->node_off;
    for (int e0 = 0; e0 < E; e0 += DN_THREADS) {
      const int e = e0 + tid;
      bool keep = e < E && v[e] >= thr;
      int row = 0;
      if (kEdges && keep) {
        row = slot_row(rp, T->n, e);
        keep = row < col[e];
      }
      const unsigned bal = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) s_wcnt[warp] = __popc(bal);
      __syncthreads();
      int off = s_base;
      for (int w = 0; w < warp; ++w) off += s_wcnt[w];
      if (keep) {
        const int pos = off + __popc(bal & ((1u << lane) - 1u));
        if (pos < cap) {
          const int64_t o = (int64_t)t * cap + pos;
          if (kEdges) {
            out_idx[2 * o] = nb[row];
            out_idx[2 * o + 1] = nb[col[e]];
          } else {
            out_idx[o] = e;
          }
          if (out_vals != nullptr) out_vals[o] = v[e];
        }
      }
      __syncthreads();
      if (tid == 0) { int tot = 0; for (int w = 0; w < DN_THREADS / 32; ++w) tot += s_wcnt[w]; s_base += tot; }
      __syncthreads();
    }
    if (tid == 0) { out_thr[t] = thr; out_cnt[t] = s_base; }
    __syncthreads();
  }
}

}  // namespace

cudaError_t gx_launch_denoise_topk(const GxPlanArrays& plan, int count, const float* edge_mask, int k2, int cap, float* out_thr,
                                   int32_t* out_cnt, int32_t* out_slots, float* out_vals, cudaStream_t s) {
  const int grid = count < GX_GRID_CAP ? count : GX_GRID_CAP;
  denoise_topk_kernel<false><<<grid, DN_THREADS, 0, s>>>(plan, count, edge_mask, k2, cap, out_thr, out_cnt, out_slots, out_vals);
  return cudaGetLastError();
}

cudaError_t gx_launch_denoise_topk_edges(const GxPlanArrays& plan, int count, const float* edge_mask, int k2, int cap, float* out_thr,
                                         int32_t* out_cnt, int32_t* out_uv, float* out_vals, cudaStream_t s) {
  const int grid = count < GX_GRID_CAP ? count : GX_GRID_CAP;
  denoise_topk_kernel<true><<<grid, DN_THREADS, 0, s>>>(plan, count, edge_mask, k2, cap, out_thr, out_cnt, out_uv, out_vals);
  return cudaGetLastError();
}
