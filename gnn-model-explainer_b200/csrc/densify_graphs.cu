// densify_graphs.cu -- the return value of graph mode on device: the packed edge masks of a list of padded graphs expanded to one dense
// (max_nodes, max_nodes) float64 array per graph, zero outside the graph's edges (explain.py:209-221 for explain.py:356-402).  It reads
// the uploaded batch CSR only, so it serves any packed result in list order -- gx_explain_graphs' output or a sharded run's gather.
#include <stdint.h>

#include "gnnx_internal.cuh"

namespace {

constexpr int kDensifyThreads = 256;

// One CTA per listed graph (grid-stride over the list).  Graph t's block out + t * n^2 is zero-filled with 16-byte stores (one scalar
// store in front when the block starts at an odd double, one behind when a double is left over), then the graph's CSR rows are
// scattered, one warp per row: slot s of the graph (its CSR entries in row-major order) is values[val_off[t] + s].  float -> double is
// exact, so the result is the host densify's bit for bit.
__global__ void __launch_bounds__(kDensifyThreads)
densify_graphs_kernel(GxGraphBatchDev gb, const int32_t* __restrict__ gids, int count, const int64_t* __restrict__ val_off,
                      const float* __restrict__ values, double* __restrict__ out) {
  const int n = gb.max_nodes;
  const int64_t nn = (int64_t)n * n;
  for (int t = blockIdx.x; t < count; t += gridDim.x) {
    double* o = out + (int64_t)t * nn;
    const int64_t head = ((uintptr_t)o & 15) ? 1 : 0;
    const int64_t pairs = (nn - head) / 2;
    double2* o2 = reinterpret_cast<double2*>(o + head);
    for (int64_t i = threadIdx.x; i < pairs; i += blockDim.x) o2[i] = make_double2(0.0, 0.0);
    if (threadIdx.x == 0) {
      if (head) o[0] = 0.0;
      if (head + 2 * pairs < nn) o[nn - 1] = 0.0;
    }
    __syncthreads();
    const int32_t* rp = gb.rowptr + (int64_t)gids[t] * n;
    const int32_t e0 = rp[0];
    const int64_t v0 = val_off[t];
    for (int r = threadIdx.x >> 5; r < n; r += blockDim.x >> 5)
      for (int32_t e = rp[r] + (threadIdx.x & 31); e < rp[r + 1]; e += 32)
        o[(int64_t)r * n + gb.col[e]] = (double)values[v0 + (e - e0)];
    // no barrier here: the next graph of this CTA lives in another block of out (a repeated id gets a block of its own, too)
  }
}

}  // namespace

cudaError_t gx_launch_densify_graphs(const GxGraphBatchDev& gb, const int32_t* gids, int count, const int64_t* val_off,
                                     const float* values, double* out, cudaStream_t s) {
  const int grid = count < GX_GRID_CAP ? count : GX_GRID_CAP;
  densify_graphs_kernel<<<grid > 0 ? grid : 1, kDensifyThreads, 0, s>>>(gb, gids, count, val_off, values, out);
  return cudaGetLastError();
}
