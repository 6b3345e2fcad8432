// khop.cu -- K1: batched k-hop neighbourhood extraction on CSR (integer, bit-exact).
//
// Replaces utils/graph_utils.py:147-158 (neighborhoods: dense (A + A^2 + .. + A^k) > 0) and
// explainer/explain.py:492-501 (extract_neighborhood: row -> nonzero -> fancy-index) of the
// reference.  One CTA per explained node; a level-synchronous frontier expansion marks the walk-
// reachable set in a per-CTA bitmap (the start node is NOT pre-marked: it is a member only if a
// closed walk of length <= k exists, exactly like the matrix powers), then the CTA emits
//   * the canonical description the reference API exposes (ascending neighbours, node_idx_new,
//     induced sub-adjacency as CSR in row-major nonzero order), and
//   * the internal description the explainer kernel consumes: nodes relabelled in
//     (distance-from-node, id) order so that every layer's receptive field is a prefix, rows with
//     columns ascending in that order, the undirected pair list with both directed slots.
#include "gnnx_internal.cuh"

namespace {

#ifndef GX_KH_THREADS
#define GX_KH_THREADS 512
#endif
constexpr int KH_THREADS = GX_KH_THREADS;   // threads per extraction CTA (one CTA per explained node): the big neighbourhoods are latency bound on per-row
                                             // dependent loads, 16 warps hide more of it than 8
constexpr int GX_RANK_SORT_MAX = 4096;  // O(n^2) rank sort of (level, degree) keys up to this many nodes

struct Slot {
  uint32_t* bm;
  int32_t* wpref;
  uint8_t* dist;
  int32_t* q;
  int32_t* loc;
  int32_t* cof;
  int32_t* pbase;
};

__device__ __forceinline__ Slot slot_of(const GxSlotWs& ws, int s, int64_t N) {
  Slot sl;
  sl.bm = ws.bm + (int64_t)s * ws.W;
  sl.wpref = ws.wpref + (int64_t)s * (ws.W + 1);
  sl.dist = ws.dist + (int64_t)s * N;
  sl.q = ws.q + (int64_t)s * (N + 1);
  sl.loc = ws.loc + (int64_t)s * N;
  sl.cof = ws.cof + (int64_t)s * N;
  sl.pbase = ws.pbase + (int64_t)s * (N + 1);
  return sl;
}

__device__ __forceinline__ bool member(const uint32_t* bm, int v) {
  return (__ldcg(bm + (v >> 5)) >> (v & 31)) & 1u;
}

// Row loops: the induced rows are short (a handful of neighbours), so a warp walks KH_GPW rows at a time, KH_GL lanes each -- four times
// as many dependent load chains in flight as one row per warp.  -DGX_KH_GL=32 restores one row per warp (A/B).
#ifndef GX_KH_GL
#define GX_KH_GL 8
#endif
constexpr int KH_GL = GX_KH_GL;
constexpr int KH_GPW = 32 / KH_GL;
__device__ __forceinline__ int group_sum_i(int x) {
#pragma unroll
  for (int o = KH_GL / 2; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}
__device__ __forceinline__ uint32_t group_bits(uint32_t ballot, int sub) {
  return KH_GL == 32 ? ballot : ((ballot >> (sub * KH_GL)) & ((1u << KH_GL) - 1u));
}

__device__ __forceinline__ int warp_sum_i(int x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

// In-place exclusive scan of data[0..len) by the whole CTA; returns the total.  s_w: >= 33 ints.
__device__ int block_excl_scan(int32_t* data, int len, int* s_w) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  int carry = 0;
  for (int base = 0; base < len; base += blockDim.x) {
    const int idx = base + tid;
    const int v = idx < len ? data[idx] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_w[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = lane < nwarps ? s_w[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      s_w[lane] = w;
    }
    __syncthreads();
    const int woff = warp > 0 ? s_w[warp - 1] : 0;
    const int total = s_w[nwarps - 1];
    if (idx < len) data[idx] = carry + woff + x - v;
    carry += total;
    __syncthreads();
  }
  return carry;
}

// Frontier expansion; returns the queue length (q[0] is a pseudo entry holding the start node; the
// members are q[1..tail)).  s_ctrl: 3 ints of shared memory.
__device__ int bfs_khop(const GxGraphDev& g, int root, int k, const Slot& sl, int* s_ctrl) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  if (tid == 0) {
    sl.q[0] = root;
    s_ctrl[0] = 0;
    s_ctrl[1] = 1;
    s_ctrl[2] = 1;
  }
  __syncthreads();
  for (int lvl = 0; lvl < k; ++lvl) {
    const int lo = s_ctrl[0], hi = s_ctrl[1];
    if (lo == hi) break;
    for (int idx = lo + warp; idx < hi; idx += nwarps) {
      const int u = sl.q[idx];
      const int e1 = g.rowptr[u + 1];
      for (int e = g.rowptr[u] + lane; e < e1; e += 32) {
        const int v = g.col[e];
        const uint32_t bit = 1u << (v & 31);
        const uint32_t old = atomicOr(sl.bm + (v >> 5), bit);
        if (!(old & bit)) {
          const int pos = atomicAdd(&s_ctrl[2], 1);
          sl.q[pos] = v;
          sl.dist[v] = (uint8_t)(lvl + 1);
        }
      }
    }
    __syncthreads();
    if (tid == 0) {
      s_ctrl[0] = hi;
      s_ctrl[1] = s_ctrl[2];
    }
    __syncthreads();
  }
  const int tail = s_ctrl[2];
  __syncthreads();
  return tail;
}

__device__ __forceinline__ void bfs_cleanup(const Slot& sl, int tail) {
  for (int idx = 1 + threadIdx.x; idx < tail; idx += blockDim.x) sl.bm[sl.q[idx] >> 5] = 0u;
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(KH_THREADS)
khop_count_kernel(GxGraphDev g, const int32_t* __restrict__ nodes, int count, int k, int row_lvl,
                  GxSlotWs ws, GxTask* __restrict__ tasks) {
  __shared__ int s_ctrl[3];
  __shared__ int s_cnt[GX_MAX_LEVELS + 1];
  __shared__ int s_e[4];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const Slot sl = slot_of(ws, blockIdx.x, g.N);
  for (int t = blockIdx.x; t < count; t += gridDim.x) {
    const int root = nodes[t];
    const int tail = bfs_khop(g, root, k, sl, s_ctrl);
    if (tid <= GX_MAX_LEVELS) s_cnt[tid] = 0;
    if (tid < 4) s_e[tid] = 0;
    __syncthreads();
    for (int idx0 = 1 + warp * KH_GPW; idx0 < tail; idx0 += nwarps * KH_GPW) {
      const int idx = idx0 + lane / KH_GL;
      const bool valid = idx < tail;
      const int u = valid ? sl.q[idx] : root;
      const int du = (u == root) ? 0 : (int)sl.dist[u];
      int cnt = 0, cnt_out = 0, loop = 0;
      if (valid) {
        const int e1 = g.rowptr[u + 1];
        for (int e = g.rowptr[u] + lane % KH_GL; e < e1; e += KH_GL) {
          const int v = g.col[e];
          if (v != u && member(sl.bm, v)) {
            ++cnt;
            const int dv = (v == root) ? 0 : (int)sl.dist[v];
            cnt_out += dv > row_lvl ? 1 : 0;
          }
          loop += v == u ? 1 : 0;
        }
      }
      cnt = group_sum_i(cnt);
      cnt_out = group_sum_i(cnt_out);
      loop = group_sum_i(loop);
      if (valid && lane % KH_GL == 0) {
        atomicAdd(&s_cnt[du], 1);
        atomicAdd(&s_e[0], cnt);
        if (loop) atomicAdd(&s_e[3], 1);
        if (du <= row_lvl) { atomicAdd(&s_e[1], cnt); atomicAdd(&s_e[2], cnt_out); }
      }
    }
    __syncthreads();
    if (tid == 0) {
      GxTask T;
      T.node = root;
      T.n = tail - 1;
      T.e_d = s_e[0];
      T.npairs = s_e[0] / 2;
      T.e1 = s_e[1];
      T.npairs_in = (s_e[1] - s_e[2]) / 2 + s_e[2];  // inner-inner pairs are seen from both ends
      T.idx_new = -1;
      T.gt_label = g.label ? g.label[root] : 0;
      T.status = member(sl.bm, root) ? 0 : 1;
      int c = 0;
      for (int l = 0; l <= GX_MAX_LEVELS; ++l) {
        c += s_cnt[l];
        T.cum[l] = c;
      }
      T.n2 = T.cum[row_lvl];
      T.n1 = row_lvl >= 1 ? T.cum[row_lvl - 1] : 0;
      T.smem_bytes = 0;
      T.n_norm = tail - 1;
      T.flags = 0;
      T.loops = s_e[3];
      T.node_off = T.edge_off = T.pair_off = T.rp_off = 0;
      tasks[t] = T;
    }
    __syncthreads();
    bfs_cleanup(sl, tail);
  }
}

// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int lower_bound_i(const int32_t* a, int lo, int hi, int key) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(KH_THREADS)
khop_fill_kernel(GxGraphDev g, int count, int k, GxSlotWs ws, GxPlanArrays P) {
  __shared__ int s_ctrl[3];
  __shared__ int s_w[33];
  __shared__ int s_cum[GX_MAX_LEVELS + 2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int sub = lane / KH_GL, gl = lane % KH_GL;   // row group of this lane inside its warp, lane inside the group
  const uint32_t lt_mask = (1u << gl) - 1u;
  const Slot sl = slot_of(ws, blockIdx.x, g.N);
  const int W = ws.W;
  for (int t = blockIdx.x; t < count; t += gridDim.x) {
    GxTask* T = P.tasks + t;
    if (T->status != 0) continue;  // uniform
    const int root = T->node;
    const int n = T->n;
    const int tail = bfs_khop(g, root, k, sl, s_ctrl);
    int32_t* nbrs = P.nbrs + T->node_off;
    int32_t* lo2gid = P.lo2gid + T->node_off;
    int32_t* srp = P.sub_rowptr + T->rp_off;
    int32_t* irp = P.irowptr + T->rp_off;
    int32_t* scol = P.sub_col + T->edge_off;
    int32_t* icol = P.icol + T->edge_off;
    if (tid <= GX_MAX_LEVELS) s_cum[tid + 1] = T->cum[tid];
    if (tid == 0) s_cum[0] = 0;

    // (1) word prefix of the membership bitmap -> canonical ranks
    for (int w = tid; w < W; w += blockDim.x) sl.wpref[w] = __popc(__ldcg(sl.bm + w));
    __syncthreads();
    block_excl_scan(sl.wpref, W, s_w);
    // (2) ascending neighbour list (explain.py:497 np.nonzero)
    for (int w = tid; w < W; w += blockDim.x) {
      uint32_t bits = __ldcg(sl.bm + w);
      int base = sl.wpref[w];
      while (bits) {
        const int b = __ffs(bits) - 1;
        nbrs[base++] = w * 32 + b;
        bits &= bits - 1;
      }
    }
    __syncthreads();
    auto canon = [&](int v) -> int {
      return sl.wpref[v >> 5] + __popc(__ldcg(sl.bm + (v >> 5)) & ((1u << (v & 31)) - 1u));
    };
    if (tid == 0) T->idx_new = canon(root);  // == sum(row[:node_idx]) (explain.py:496)
    // (3) induced degrees of the canonical rows
    for (int c0 = warp * KH_GPW; c0 < n; c0 += nwarps * KH_GPW) {
      const int c = c0 + sub;
      int cnt = 0;
      if (c < n) {
        const int u = nbrs[c];
        const int e1 = g.rowptr[u + 1];
        for (int e = g.rowptr[u] + gl; e < e1; e += KH_GL) {
          const int v = g.col[e];
          cnt += (v != u && member(sl.bm, v)) ? 1 : 0;
        }
      }
      cnt = group_sum_i(cnt);
      if (gl == 0 && c < n) srp[c] = cnt;
    }
    __syncthreads();
    // (4) level order: (distance from the node asc, induced degree desc, id asc).  Every layer's row
    //     set is a prefix, and inside a level rows of similar degree are adjacent (the explainer kernel
    //     processes rows in lane groups: similar degrees => little divergence, hubs first).
    if (n <= GX_RANK_SORT_MAX) {
      for (int c = tid; c < n; c += blockDim.x) {
        const int v = nbrs[c];
        const int dv = (v == root) ? 0 : (int)sl.dist[v];
        sl.pbase[c] = (dv << 24) | (0xFFFFFF - min(srp[c], 0xFFFFFF));
      }
      __syncthreads();
      for (int c = tid; c < n; c += blockDim.x) {
        const int key = sl.pbase[c];
        int rank = 0;
        for (int o = 0; o < n; ++o) {
          const int ko = sl.pbase[o];
          rank += (ko < key || (ko == key && o < c)) ? 1 : 0;
        }
        sl.loc[c] = rank;
        sl.cof[rank] = c;
        lo2gid[rank] = nbrs[c];
      }
      __syncthreads();
    } else {
      // large neighbourhoods: stable partition by level only (scan based, O(n) per level)
      int base_lo = 0;
      for (int lv = 0; lv <= k; ++lv) {
        for (int c = tid; c < n; c += blockDim.x) {
          const int v = nbrs[c];
          const int dv = (v == root) ? 0 : (int)sl.dist[v];
          sl.pbase[c] = (dv == lv) ? 1 : 0;
        }
        __syncthreads();
        const int tot = block_excl_scan(sl.pbase, n, s_w);
        for (int c = tid; c < n; c += blockDim.x) {
          const int v = nbrs[c];
          const int dv = (v == root) ? 0 : (int)sl.dist[v];
          if (dv == lv) {
            const int lo = base_lo + sl.pbase[c];
            sl.loc[c] = lo;
            sl.cof[lo] = c;
            lo2gid[lo] = v;
          }
        }
        base_lo += tot;
        __syncthreads();
      }
    }
    // canonical and level-order row pointers
    const int e_tot = block_excl_scan(srp, n, s_w);
    if (tid == 0) srp[n] = e_tot;
    __syncthreads();
    for (int i = tid; i < n; i += blockDim.x) {
      const int c = sl.cof[i];
      irp[i] = srp[c + 1] - srp[c];
    }
    __syncthreads();
    block_excl_scan(irp, n, s_w);
    if (tid == 0) irp[n] = e_tot;
    // (5) canonical columns: member neighbours in ascending id order (row-major nonzero order)
    for (int c0 = warp * KH_GPW; c0 < n; c0 += nwarps * KH_GPW) {
      const int c = c0 + sub;
      const bool valid = c < n;
      const int u = valid ? nbrs[c] : 0;
      int out = valid ? srp[c] : 0;
      const int e0 = valid ? g.rowptr[u] : 0, e1 = valid ? g.rowptr[u + 1] : 0;
      for (int eb = e0; __any_sync(0xffffffffu, eb < e1); eb += KH_GL) {
        const int e = eb + gl;
        int v = -1;
        bool keep = false;
        if (e < e1) {
          v = g.col[e];
          keep = (v != u) && member(sl.bm, v);
        }
        const uint32_t bal = group_bits(__ballot_sync(0xffffffffu, keep), sub);
        if (keep) scol[out + __popc(bal & lt_mask)] = canon(v);
        out += __popc(bal);
      }
    }
    __syncthreads();
    // (6) level-order rows: each canonical row partitioned by the level of the neighbour (columns within
    //     one hop of the explained node first: the backward only needs that prefix); the two slot maps
    //     canonical <-> internal are kept for the pair construction
    int32_t* cs2is = P.cs2is + T->edge_off;
    int32_t* is2cs = P.is2cs + T->edge_off;
    for (int i0 = warp * KH_GPW; i0 < n; i0 += nwarps * KH_GPW) {
      const int i = i0 + sub;
      const bool valid = i < n;
      const int c = valid ? sl.cof[i] : 0;
      const int r0 = valid ? srp[c] : 0, r1 = valid ? srp[c + 1] : 0;
      int out = valid ? irp[i] : 0;
      for (int lv = 0; lv <= k; ++lv) {
        const int lo_b = s_cum[lv], lo_e = s_cum[lv + 1];
        if (lo_b == lo_e) continue;
        for (int eb = r0; __any_sync(0xffffffffu, eb < r1); eb += KH_GL) {
          const int e = eb + gl;
          int lo = -1;
          if (e < r1) lo = sl.loc[scol[e]];
          const bool keep = lo >= lo_b && lo < lo_e;
          const uint32_t bal = group_bits(__ballot_sync(0xffffffffu, keep), sub);
          if (keep) {
            const int o = out + __popc(bal & lt_mask);
            icol[o] = lo;
            cs2is[e] = o;
            is2cs[o] = e;
          }
          out += __popc(bal);
        }
      }
    }
    __syncthreads();
    // (7) undirected pairs, owned by the endpoint with the smaller level-order id, in (i, slot) order:
    //     pairs touching the explained node / its neighbours come first, pairs between two
    //     outermost nodes last (uniform work per warp in the explainer's edge phase)
    for (int i0 = warp * KH_GPW; i0 < n; i0 += nwarps * KH_GPW) {
      const int i = i0 + sub;
      int cnt = 0;
      if (i < n)
        for (int kk = irp[i] + gl; kk < irp[i + 1]; kk += KH_GL) cnt += icol[kk] > i ? 1 : 0;
      cnt = group_sum_i(cnt);
      if (gl == 0 && i < n) sl.pbase[i] = cnt;
    }
    __syncthreads();
    block_excl_scan(sl.pbase, n, s_w);
    for (int i0 = warp * KH_GPW; i0 < n; i0 += nwarps * KH_GPW) {
      const int i = i0 + sub;
      const bool valid = i < n;
      const int r0 = valid ? irp[i] : 0, r1 = valid ? irp[i + 1] : 0;
      const int ci = valid ? sl.cof[i] : 0;
      int64_t out = T->pair_off + (valid ? sl.pbase[i] : 0);
      for (int kb = r0; __any_sync(0xffffffffu, kb < r1); kb += KH_GL) {
        const int kk = kb + gl;
        int j = -1;
        if (kk < r1) j = icol[kk];
        const bool keep = valid && j > i;
        const uint32_t bal = group_bits(__ballot_sync(0xffffffffu, keep), sub);
        if (keep) {
          const int64_t p = out + __popc(bal & lt_mask);
          const int cj = sl.cof[j];
          const int oji = lower_bound_i(scol, srp[cj], srp[cj + 1], ci);
          P.pair_i[p] = i;
          P.pair_j[p] = j;
          P.pair_pij[p] = kk;
          P.pair_pji[p] = cs2is[oji];
          P.pair_oij[p] = is2cs[kk];
          P.pair_oji[p] = oji;
        }
        out += __popc(bal);
      }
    }
    __syncthreads();
    bfs_cleanup(sl, tail);
  }
}

// graph_utils.neighborhoods rows: out_rows[t*N + v] = 1 for members (out pre-zeroed).
__global__ void __launch_bounds__(KH_THREADS)
hop_rows_kernel(GxGraphDev g, const int32_t* __restrict__ nodes, int count, int k, GxSlotWs ws,
                uint8_t* __restrict__ out_rows) {
  __shared__ int s_ctrl[3];
  const Slot sl = slot_of(ws, blockIdx.x, g.N);
  for (int t = blockIdx.x; t < count; t += gridDim.x) {
    const int tail = bfs_khop(g, nodes[t], k, sl, s_ctrl);
    uint8_t* row = out_rows + (int64_t)t * g.N;
    for (int idx = 1 + threadIdx.x; idx < tail; idx += blockDim.x) row[sl.q[idx]] = 1;
    __syncthreads();
    bfs_cleanup(sl, tail);
  }
}

// dense (n,n) float64 expansion of packed edge masks (explain.py:209-221 return value)
__global__ void __launch_bounds__(256)
densify_kernel(GxPlanArrays P, int count, const int64_t* __restrict__ dense_off,
               const float* __restrict__ edge_mask, double* __restrict__ out) {
  for (int t = blockIdx.x; t < count; t += gridDim.x) {
    const GxTask* T = P.tasks + t;
    const int n = T->n;
    double* o = out + dense_off[t];
    const int64_t nn = (int64_t)n * n;
    for (int64_t i = threadIdx.x; i < nn; i += blockDim.x) o[i] = 0.0;
    __syncthreads();
    const int32_t* srp = P.sub_rowptr + T->rp_off;
    const int32_t* scol = P.sub_col + T->edge_off;
    const float* em = edge_mask + T->edge_off;
    for (int r = threadIdx.x >> 5; r < n; r += blockDim.x >> 5)
      for (int e = srp[r] + (threadIdx.x & 31); e < srp[r + 1]; e += 32)
        o[(int64_t)r * n + scol[e]] = (double)em[e];
    __syncthreads();
  }
}

}  // namespace

static int khop_grid(int count, const GxSlotWs& ws) { return count < ws.slots ? count : ws.slots; }

cudaError_t gx_launch_khop_count(const GxGraphDev& g, const int32_t* nodes_dev, int count, int k,
                                 int row_lvl, GxSlotWs ws, GxTask* tasks, cudaStream_t s) {
  khop_count_kernel<<<khop_grid(count, ws), KH_THREADS, 0, s>>>(g, nodes_dev, count, k, row_lvl, ws, tasks);
  return cudaGetLastError();
}

cudaError_t gx_launch_khop_fill(const GxGraphDev& g, int count, int k, GxSlotWs ws, GxPlanArrays plan,
                                cudaStream_t s) {
  khop_fill_kernel<<<khop_grid(count, ws), KH_THREADS, 0, s>>>(g, count, k, ws, plan);
  return cudaGetLastError();
}

cudaError_t gx_launch_hop_rows(const GxGraphDev& g, const int32_t* nodes_dev, int count, int k,
                               GxSlotWs ws, uint8_t* out_rows, cudaStream_t s) {
  hop_rows_kernel<<<khop_grid(count, ws), KH_THREADS, 0, s>>>(g, nodes_dev, count, k, ws, out_rows);
  return cudaGetLastError();
}

cudaError_t gx_launch_densify(const GxPlanArrays& plan, int count, const int64_t* dense_off,
                              const float* edge_mask, double* out, cudaStream_t s) {
  const int grid = count < GX_GRID_CAP ? count : GX_GRID_CAP;
  densify_kernel<<<grid, 256, 0, s>>>(plan, count, dense_off, edge_mask, out);
  return cudaGetLastError();
}
