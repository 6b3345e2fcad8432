// explain_stream.cu -- K2s: the mask-optimisation kernel for explained nodes whose k-hop state does not fit the
// 227 KB of shared memory (wide features and/or 10^4..10^5-node neighbourhoods: BASELINE config 5).
//
// Same arithmetic contract as explain_node.cu (explainer/explain.py:137-146,665-715,740-808 + autograd + Adam,
// models.py:58-80,230-267,363-376), different data placement and a different contraction order:
//   * one persistent CTA (768 threads) per task, model weights and per-warp scratch in shared memory, every
//     per-node / per-edge array in a per-CTA global slab (L2 / HBM), the CSR and pair index arrays read in
//     place from the plan (no per-task copy);
//   * layer 1 is evaluated as A_m (X' W1) instead of (A_m X') W1: the d-wide feature row of a node is read
//     once per pass (F0: P = (X . sF) W1 for all nodes; B0: dL/dsF = sum_j X_j . (dP_j W1^T)) and every
//     per-edge operation is hid-wide (gathers of 80-byte rows, 20-float dots) -- for d = 128 that is 6.4x fewer
//     bytes per edge than the U = A_m X order the shared-memory kernel uses for d <= hid;
//   * dP = A_m^T dY1 needs, for every node j (also the outermost ones), its neighbours inside the layer-1 row
//     set: the plan's level-partitioned rows give that as a prefix of row j (cnt2).
//   * sparse aggregations stage the gathered hid-wide rows in shared memory with cp.async (LDGSTS, 16 B per lane,
//     no registers held by loads in flight): a warp streams its rows as chunks of up to 32 edges, two chunks in
//     flight across row boundaries, and reduces from shared memory (staged_rows);
//   * the two dense passes over the d-wide feature rows (F0, B0) keep four rows per warp in flight in registers.
// Phases per epoch (one __syncthreads each): F0 | F1 | F2 | S | B2 | B1 | B0 | P.
// Pairs between two outermost nodes are regulariser-only scalar recurrences (outer_pairs_kernel).
#include "explain_common.cuh"

namespace {

struct StreamSmem {
  int W1s, W1t, W1m, W2s, W2t, W3s, bs, sF, F, mF, vF, zs, dE, dZ3, logit, Wp, stage, astage, stage_per_warp, total;
};
constexpr int kStageBufs = 2;                                                   // chunks in flight per warp
__host__ __device__ constexpr int stage_chunk(int hid) { return hid <= 20 ? 32 : 16; }  // edges per chunk
constexpr int kTileRows = 4;                                                    // feature rows per tile of the dense passes
__host__ __device__ inline int tile_stride(int dp) { return gx_round_up(dp, 32) + 8; }  // bank-conflict-free row stride (floats)
__host__ __device__ inline StreamSmem stream_smem(int dp, int hid, int emb, int C, int nwarps) {
  StreamSmem S;
  int o = 0;
  auto take = [&](int words) { int r = o; o += gx_round_up(words, 4); return r; };
  S.W1s = take(dp * hid); S.W1t = take(hid * dp); S.W1m = take(dp * hid); S.W2s = take(hid * hid); S.W2t = take(hid * hid);
  S.W3s = take(hid * emb); S.bs = take(2 * hid + emb);
  S.sF = take(dp); S.F = take(dp); S.mF = take(dp); S.vF = take(dp);
  S.zs = take(nwarps * 128);
  S.dE = take(2 * hid); S.dZ3 = take(hid); S.logit = take(C < 32 ? 32 : C);
  S.Wp = take(C * (2 * hid + emb + 1) <= GX_WP_SMEM_MAX ? C * (2 * hid + emb + 1) : 0);
  // per warp: the gathered hid-wide rows of the sparse passes, or two 4-row tiles of d-wide feature rows (+ their dP rows)
  const int sp_rows = kStageBufs * stage_chunk(hid) * hid, sp_tiles = 2 * kTileRows * (tile_stride(dp) + hid);
  S.stage_per_warp = gx_round_up(sp_rows > sp_tiles ? sp_rows : sp_tiles, 4);
  S.stage = take(nwarps * S.stage_per_warp);
  S.astage = take(nwarps * kStageBufs * stage_chunk(hid));        // their edge values
  S.total = o;
  return S;
}

__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gsrc) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Sparse aggregation of the rows i = warp, warp + nwarps, ... < R of one warp:  z_i = sum_{e in [r0_i, r1_i)} a[e] f(src[icol[e]])
// with hid-wide source rows.  The rows are streamed as chunks of <= CH edges (a chunk never spans two rows, an empty row is
// one empty chunk).  Issuing side: lane l reads (icol, a) of edge l one chunk ahead into registers; H4 adjacent lanes then
// copy one source row into the warp's staging buffer with cp.async (one 128-byte line per row and instruction),
// kStageBufs chunks in flight across row boundaries.  Consuming side: lane = (edge slot, float4 index) reads the staged
// rows, reduces the edge slots through `red` (128 floats) at the end of a row and calls epi(i, z) with the warp converged;
// z is valid on lanes < H4 (lane q holds features 4q..4q+3).  bounds(i, r0, r1) returns the edge range of row i.
// kDot: additionally gout[e] = <src[icol[e]], dotsrc[i]> for every edge e of row i (the edge-gradient dots of the layer,
// taken while the gathered row is in shared memory anyway).
template <int HID, bool kRelu, bool kDot, typename Bounds, typename Epi>
__device__ __forceinline__ void staged_rows(int R, int warp, int nwarps, int lane, const int32_t* __restrict__ icol,
                                            const float* a, const float* src, float* stage, float* astage, float* red,
                                            const float* dotsrc, float* gout, Bounds bounds, Epi epi) {
  constexpr int HS = HID, H4 = HID / 4, EPL = 32 / H4, CH = stage_chunk(HID), NB = kStageBufs;
  constexpr int NK = (CH + EPL - 1) / EPL;
  const int es = lane / H4, q = lane - es * H4;
  const bool cons = es < EPL;
  const uint32_t stage_s = (uint32_t)__cvta_generic_to_shared(stage) + (uint32_t)(es * HS + 4 * q) * 4u;
  const char* const src_q = reinterpret_cast<const char*>(src) + 16 * q;
  int i_iss = warp, e_iss = 0, end_iss = 0;
  if (i_iss < R) bounds(i_iss, e_iss, end_iss);
  int i_con = i_iss, e_con = e_iss, end_con = end_iss;
  int nx0 = 0, nx1 = 0;                                   // edge range of the issuing side's NEXT row, loaded one row ahead
  if (i_iss + nwarps < R) bounds(i_iss + nwarps, nx0, nx1);
  int c_nx = 0;
  float a_nx = 0.f;
  auto prefetch = [&]() {
    const int e = e_iss + lane;
    if (i_iss < R && lane < CH && e < end_iss) { c_nx = __ldg(icol + e); a_nx = a[e]; }
  };
  auto issue = [&](int buf) {
    if (i_iss < R) {
      const int nvalid = min(CH, end_iss - e_iss);
      if (lane < nvalid) astage[buf * CH + lane] = a_nx;
#pragma unroll
      for (int k = 0; k < NK; ++k) {
        const int slot = k * EPL + es;
        const int c = __shfl_sync(0xffffffffu, c_nx, slot & 31);
        if (cons && slot < nvalid) {
          const uint32_t d = stage_s + (uint32_t)((buf * CH + k * EPL) * HS) * 4u;
          const char* g = src_q + (size_t)((uint32_t)c * (uint32_t)(HS * 4));
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(g) : "memory");
        }
      }
      e_iss += CH;
      if (e_iss >= end_iss) {
        i_iss += nwarps;
        e_iss = nx0; end_iss = nx1;
        if (i_iss + nwarps < R) bounds(i_iss + nwarps, nx0, nx1);
      }
    }
    cp_async_commit();
    prefetch();
  };
  prefetch();
#pragma unroll
  for (int b = 0; b < NB; ++b) issue(b);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 dv = make_float4(0.f, 0.f, 0.f, 0.f);
  if (kDot && i_con < R && lane < 32 && cons) dv = ld4(dotsrc + i_con * HS + 4 * q);
  int buf = 0;
  while (i_con < R) {
    cp_async_wait<NB - 1>();
    __syncwarp();
    const int cnt = min(CH, end_con - e_con);
    const float* st = stage + buf * CH * HS + 4 * q;
    const float* as_ = astage + buf * CH;
    const int nsteps = (cnt + EPL - 1) / EPL;   // warp-uniform (<= 0 for an empty row)
    for (int k = 0; k < nsteps; ++k) {
      const int sidx = k * EPL + es;
      const bool ok = cons && sidx < cnt;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      float av = 0.f;
      if (ok) { v = ld4(st + sidx * HS); av = as_[sidx]; }
      if (kRelu) v = relu4(v);
      fma4(acc, av, v);
      if (kDot) {
        float pd = fmaf(v.x, dv.x, fmaf(v.y, dv.y, fmaf(v.z, dv.z, v.w * dv.w)));
        if (H4 == 8) {
          pd += __shfl_xor_sync(0xffffffffu, pd, 1); pd += __shfl_xor_sync(0xffffffffu, pd, 2); pd += __shfl_xor_sync(0xffffffffu, pd, 4);
        } else {   // H4 == 5: lanes es*5 .. es*5+4; only the q == 0 lane's sum is used
          const float t1 = pd + __shfl_down_sync(0xffffffffu, pd, 1);
          const float t2 = t1 + __shfl_down_sync(0xffffffffu, t1, 2);
          pd = t2 + __shfl_down_sync(0xffffffffu, pd, 4);
        }
        if (ok && q == 0) gout[e_con + sidx] = pd;
      }
    }
    e_con += CH;
    const bool row_done = e_con >= end_con;
    __syncwarp();
    issue(buf);
    buf = buf + 1 == NB ? 0 : buf + 1;
    if (row_done) {
      st4(red + lane * 4, acc);
      __syncwarp();
      float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      if (lane < H4) {
#pragma unroll
        for (int s2 = 0; s2 < EPL; ++s2) { const float4 o = ld4(red + (s2 * H4 + lane) * 4); z.x += o.x; z.y += o.y; z.z += o.z; z.w += o.w; }
      }
      __syncwarp();
      epi(i_con, z);
      acc = make_float4(0.f, 0.f, 0.f, 0.f);
      i_con += nwarps;
      if (i_con < R) {
        bounds(i_con, e_con, end_con);
        if (kDot && cons) dv = ld4(dotsrc + i_con * HS + 4 * q);
      }
    }
  }
  cp_async_wait<0>();
}

// this lane's float4 (features 4q..4q+3) of a feature row of the full graph
__device__ __forceinline__ float4 load_x4(const float* __restrict__ row, int q, int d, bool vec) {
  if (vec) return __ldg(reinterpret_cast<const float4*>(row) + q);
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  const int f = 4 * q;
  if (f < d) v.x = __ldg(row + f);
  if (f + 1 < d) v.y = __ldg(row + f + 1);
  if (f + 2 < d) v.z = __ldg(row + f + 2);
  if (f + 3 < d) v.w = __ldg(row + f + 3);
  return v;
}

// F0, vector path: P[j] = X[j] (sF (.) W1) for all nodes.  A warp takes tiles of kTileRows feature rows, copied with
// cp.async into its staging area (two tiles in flight); lane = (row r of the tile, feature slice s = f mod 8) keeps all
// HID outputs of its row in registers, so one pass over W1m (shared memory) serves the four rows of the tile.
template <int HID>
__device__ __forceinline__ void dense_forward_tiles(int n, int d, int dp, int warp, int nwarps, int lane,
                                                    const float* __restrict__ feat, const int32_t* __restrict__ lo2gid,
                                                    const float* W1m, float* xb, float* P) {
  constexpr int HS = HID, H4 = HID / 4, TR = kTileRows;
  const int D4 = dp / 4, xs = tile_stride(dp);
  const int ntile = (n + TR - 1) / TR;
  const int r = lane >> 3, sl = lane & 7;
  int t_iss = warp;
  auto gid_of = [&](int t) { const int row = t * TR + lane; return (t < ntile && lane < TR && row < n) ? __ldg(lo2gid + row) : -1; };
  int g_nx = gid_of(t_iss);
  auto issue = [&](int buf) {
    if (t_iss < ntile) {
#pragma unroll
      for (int rr = 0; rr < TR; ++rr) {
        const int gid = __shfl_sync(0xffffffffu, g_nx, rr);
        if (gid >= 0 && lane < D4) cp_async16(xb + (buf * TR + rr) * xs + 4 * lane, feat + (int64_t)gid * d + 4 * lane);
      }
      t_iss += nwarps;
      g_nx = gid_of(t_iss);
    }
    cp_async_commit();
  };
  issue(0);
  issue(1);
  int buf = 0;
  for (int t = warp; t < ntile; t += nwarps) {
    cp_async_wait<1>();
    __syncwarp();
    float acc[HID];
#pragma unroll
    for (int h = 0; h < HID; ++h) acc[h] = 0.f;
    const float* xr = xb + (buf * TR + r) * xs;
    for (int f = sl; f < dp; f += 8) {
      const float xv = xr[f];
      const float* w = W1m + f * HS;
#pragma unroll
      for (int h4 = 0; h4 < H4; ++h4) {
        const float4 w4 = ld4(w + 4 * h4);
        acc[4 * h4] = fmaf(xv, w4.x, acc[4 * h4]); acc[4 * h4 + 1] = fmaf(xv, w4.y, acc[4 * h4 + 1]);
        acc[4 * h4 + 2] = fmaf(xv, w4.z, acc[4 * h4 + 2]); acc[4 * h4 + 3] = fmaf(xv, w4.w, acc[4 * h4 + 3]);
      }
    }
#pragma unroll
    for (int h = 0; h < HID; ++h) {
      acc[h] += __shfl_xor_sync(0xffffffffu, acc[h], 1);
      acc[h] += __shfl_xor_sync(0xffffffffu, acc[h], 2);
      acc[h] += __shfl_xor_sync(0xffffffffu, acc[h], 4);
    }
    const int row = t * TR + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int h4 = 0; h4 < H4; ++h4)
      if (sl == h4) v = make_float4(acc[4 * h4], acc[4 * h4 + 1], acc[4 * h4 + 2], acc[4 * h4 + 3]);
    if (row < n && sl < H4) st4(P + row * HS + 4 * sl, v);
    __syncwarp();
    issue(buf);
    buf ^= 1;
  }
  cp_async_wait<0>();
}

// B0, vector path: this warp's share of dL/dsF = sum_j X_j (.) (dP_j W1^T).  Same tiling; lane l owns features 4l..4l+3
// and keeps the four rows' products in registers, so one pass over W1t serves the tile.
template <int HID>
__device__ __forceinline__ float4 dense_backward_tiles(int n, int d, int dp, int warp, int nwarps, int lane,
                                                       const float* __restrict__ feat, const int32_t* __restrict__ lo2gid,
                                                       const float* W1t, float* xb, const float* dP) {
  constexpr int HS = HID, H4 = HID / 4, TR = kTileRows;
  const int D4 = dp / 4, xs = tile_stride(dp);
  float* const pb = xb + 2 * TR * xs;
  const int ntile = (n + TR - 1) / TR;
  int t_iss = warp;
  auto gid_of = [&](int t) { const int row = t * TR + lane; return (t < ntile && lane < TR && row < n) ? __ldg(lo2gid + row) : -1; };
  int g_nx = gid_of(t_iss);
  auto issue = [&](int buf) {
    if (t_iss < ntile) {
#pragma unroll
      for (int rr = 0; rr < TR; ++rr) {
        const int gid = __shfl_sync(0xffffffffu, g_nx, rr);
        if (gid >= 0 && lane < D4) cp_async16(xb + (buf * TR + rr) * xs + 4 * lane, feat + (int64_t)gid * d + 4 * lane);
      }
      if (lane < TR * H4) {
        const int rr = lane / H4, c = lane - rr * H4, row = t_iss * TR + rr;
        if (row < n) cp_async16(pb + (buf * TR + rr) * HS + 4 * c, dP + row * HS + 4 * c);
      }
      t_iss += nwarps;
      g_nx = gid_of(t_iss);
    }
    cp_async_commit();
  };
  issue(0);
  issue(1);
  float4 gacc = make_float4(0.f, 0.f, 0.f, 0.f);
  int buf = 0;
  for (int t = warp; t < ntile; t += nwarps) {
    cp_async_wait<1>();
    __syncwarp();
    if (lane < D4) {
      float4 tq[TR];
#pragma unroll
      for (int rr = 0; rr < TR; ++rr) tq[rr] = make_float4(0.f, 0.f, 0.f, 0.f);
      const float* pr = pb + buf * TR * HS;
#pragma unroll 4
      for (int h = 0; h < HID; ++h) {
        const float4 w4 = ld4(W1t + h * dp + 4 * lane);
#pragma unroll
        for (int rr = 0; rr < TR; ++rr) fma4(tq[rr], pr[rr * HS + h], w4);
      }
#pragma unroll
      for (int rr = 0; rr < TR; ++rr) {
        if (t * TR + rr < n) {
          const float4 x = ld4(xb + (buf * TR + rr) * xs + 4 * lane);
          gacc.x = fmaf(tq[rr].x, x.x, gacc.x); gacc.y = fmaf(tq[rr].y, x.y, gacc.y);
          gacc.z = fmaf(tq[rr].z, x.z, gacc.z); gacc.w = fmaf(tq[rr].w, x.w, gacc.w);
        }
      }
    }
    __syncwarp();
    issue(buf);
    buf ^= 1;
  }
  cp_async_wait<0>();
  return gacc;
}

// first slot in [r0,r1) whose column is >= bound (columns are partitioned by level, so the predicate is monotone)
__device__ __forceinline__ int prefix_below(const int32_t* __restrict__ icol, int r0, int r1, int bound) {
  int lo = r0, hi = r1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(icol + mid) < bound) lo = mid + 1; else hi = mid;
  }
  return lo - r0;
}

template <int HID, int EMB, int NT, bool kTrace>
__global__ void __launch_bounds__(NT, 1) explain_stream_kernel(const ExplainArgs A) {
  extern __shared__ __align__(16) float sm[];
  __shared__ int s_task;
  __shared__ float s_tr[kTrace ? (NT / 32) * 4 + 4 : 1];   // trace: per-warp partial sums of the edge phase + (pred loss, p[gt], feat-size term)
  __shared__ long long s_ph[9];   // debug: per-phase cycle sums of the CTA's first task + last stamp
  static_assert((HID == 20 || HID == 32) && EMB % 4 == 0 && EMB <= 32, "hidden width 20 or 32 (others are zero-padded to 32 by gx_set_model)");
  constexpr int HS = HID, H4 = HID / 4, PD = 2 * HID + EMB;
  constexpr int nwarps = NT / 32;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const GxModelDev& m = A.m;
  const GxHparamsDev& hp = A.hp;
  const int d = m.d, C = m.C;
  const bool ieee = (hp.flags & GX_HP_IEEE_EDGE) != 0;
  const int dp = gx_round_up(d, 4), D4 = dp / 4;
  const bool xvec = (d % 4 == 0) && ((reinterpret_cast<uintptr_t>(A.g.feat) & 15) == 0);
  const StreamSmem S = stream_smem(dp, HID, EMB, C, nwarps);
  float* const W1s = sm + S.W1s; float* const W1t = sm + S.W1t; float* const W2s = sm + S.W2s; float* const W2t = sm + S.W2t;
  float* const W3s = sm + S.W3s; float* const bs = sm + S.bs; float* const sF = sm + S.sF; float* const Fm = sm + S.F;
  float* const mF = sm + S.mF; float* const vF = sm + S.vF; float* const zw = sm + S.zs + warp * 128;
  float* const stage = sm + S.stage + warp * S.stage_per_warp;
  float* const W1m = sm + S.W1m;
  float* const astage = sm + S.astage + warp * (kStageBufs * stage_chunk(HID));
  float* const dE = sm + S.dE; float* const dZ3 = sm + S.dZ3; float* const logit = sm + S.logit;
  const bool wp_smem = C * (PD + 1) <= GX_WP_SMEM_MAX;
  const float* const Wpp = wp_smem ? sm + S.Wp : m.Wp;
  const float* const bpp = wp_smem ? sm + S.Wp + C * PD : m.bp;

  // model weights: once per CTA
  for (int idx = tid; idx < dp * HS; idx += NT) { const int f = idx / HS, c = idx - f * HS; W1s[idx] = f < d ? __ldg(m.W[0] + f * HID + c) : 0.f; }
  for (int idx = tid; idx < HID * dp; idx += NT) { const int c = idx / dp, f = idx - c * dp; W1t[idx] = f < d ? __ldg(m.Wt[0] + c * d + f) : 0.f; }
  for (int idx = tid; idx < HID * HS; idx += NT) { W2s[idx] = __ldg(m.W[1] + idx); W2t[idx] = __ldg(m.Wt[1] + idx); }
  for (int idx = tid; idx < HID * EMB; idx += NT) W3s[idx] = __ldg(m.W[2] + idx);
  for (int idx = tid; idx < HID; idx += NT) { bs[idx] = __ldg(m.b[0] + idx); bs[HID + idx] = __ldg(m.b[1] + idx); }
  for (int idx = tid; idx < EMB; idx += NT) bs[2 * HID + idx] = __ldg(m.b[2] + idx);
  if (wp_smem) {
    float* const Wps = sm + S.Wp;
    for (int idx = tid; idx < C * PD; idx += NT) Wps[idx] = __ldg(m.Wp + idx);
    for (int idx = tid; idx < C; idx += NT) Wps[C * PD + idx] = __ldg(m.bp + idx);
  }

  // lane groups of 8: a group owns one hid-wide row (q < H4 lanes carry a float4 each)
  Grp G;
  G.GW = 8; G.epi = 4; G.lane = lane; G.grp = lane >> 3; G.q = lane & 7; G.gbase = G.grp * 8;
  constexpr int epi = 4;
  const int q = G.q;
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
    const int n = Tp->n, n1 = Tp->n1, n2 = Tp->n2, e_d = Tp->e_d, np = Tp->npairs_in;
    const int gt = hp.mode ? __ldg(A.g.pred_label + Tp->node) : Tp->gt_label;   // gradient baseline: predicted label (explain.py:130)
    const int64_t node_off = Tp->node_off, rp_off = Tp->rp_off, edge_off = Tp->edge_off, pair_off = Tp->pair_off;
    const GxStreamLayout L = gx_make_stream_layout(n, n1, n2, e_d, np, d, HID, nwarps);
    const int32_t* __restrict__ lo2gid = A.plan.lo2gid + node_off;
    const int32_t* const irp = A.plan.irowptr + rp_off;
    const int32_t* const icol = A.plan.icol + edge_off;
    const int32_t* __restrict__ pi = A.plan.pair_i + pair_off; const int32_t* __restrict__ pj = A.plan.pair_j + pair_off;
    const int32_t* __restrict__ ppij = A.plan.pair_pij + pair_off; const int32_t* __restrict__ ppji = A.plan.pair_pji + pair_off;
    const int32_t* __restrict__ poij = A.plan.pair_oij + pair_off; const int32_t* __restrict__ poji = A.plan.pair_oji + pair_off;
    float* const a = slab + L.a; float* const P = slab + L.P; float* const Yh1 = slab + L.Yh1; float* const q1 = slab + L.q1;
    float* const dY1 = slab + L.dY1; float* const Yh2 = slab + L.Yh2; float* const q2 = slab + L.q2; float* const dZ2 = slab + L.dZ2;
    float* const lapg = slab + L.lapg; float* const gFp = slab + L.gFp;
    int32_t* const cnt1 = reinterpret_cast<int32_t*>(slab + L.cnt1); int32_t* const cnt2 = reinterpret_cast<int32_t*>(slab + L.cnt2);
    float* const dP = slab + L.dP; float* const gE = slab + L.gE;
    float2* const MM = MM0; float2* const mm = MM + np; float2* const vv = mm + np; float2* const SS = vv + np;
    const float nn = (float)n * (float)n;
    const float ent_over_nn = hp.c_ent / nn;
    const float lap_over_nn = hp.c_lap / nn;

    // ------------------------------------------------------------------ per-task state
    const bool resume = hp.init == GX_INIT_STATE && !hp.mode;   // optimiser state supplied by the caller (gx_explain_io)
    for (int f = tid; f < dp; f += NT) {
      sF[f] = hp.mode ? 1.0f : 0.5f; Fm[f] = 0.f; mF[f] = 0.f; vF[f] = 0.f;   // feat_mask = 0 (explain.py:633-643)
      if (resume && A.x.feat_state_in != nullptr && f < d) {
        const float* fs = A.x.feat_state_in + (int64_t)task_id * 3 * d;
        Fm[f] = fs[f]; mF[f] = fs[d + f]; vF[f] = fs[2 * d + f];
        sF[f] = sigmoid_f(fs[f]);
      }
      if (hp.out_iter == 0 && !hp.mode && f < d) {
        if (A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = sF[f];
        if (A.x.feat_state_out != nullptr) {
          float* fo = A.x.feat_state_out + (int64_t)task_id * 3 * d;
          fo[f] = Fm[f]; fo[d + f] = mF[f]; fo[2 * d + f] = vF[f];
        }
      }
    }
    {
      const float m0_std = sqrtf(2.0f / (float)n);  // gain('relu') * sqrt(2/(n+n)) (explain.py:647-651)
      for (int p = tid; p < np; p += NT) {
        const int oij = poij[p], oji = poji[p];
        float Mi, Mj;
        if (hp.mode) {
          Mi = Mj = 0.f;
        } else if (hp.init == GX_INIT_PHILOX) {
          Mi = 1.0f + m0_std * philox_normal(hp.seed, (uint32_t)Tp->node, (uint32_t)oij);
          Mj = 1.0f + m0_std * philox_normal(hp.seed, (uint32_t)Tp->node, (uint32_t)oji);
        } else {
          Mi = __ldg(A.m0 + edge_off + oij);
          Mj = __ldg(A.m0 + edge_off + oji);
        }
        float2 m2 = make_float2(0.f, 0.f), v2 = m2;
        if (resume) {
          m2 = make_float2(__ldg(A.x.adam_m_in + edge_off + oij), __ldg(A.x.adam_m_in + edge_off + oji));
          v2 = make_float2(__ldg(A.x.adam_v_in + edge_off + oij), __ldg(A.x.adam_v_in + edge_off + oji));
        }
        MM[p] = make_float2(Mi, Mj);
        mm[p] = m2;
        vv[p] = v2;
        const float Si = resume ? sigmoid_fast(Mi, ieee) : sigmoid_f(Mi), Sj = resume ? sigmoid_fast(Mj, ieee) : sigmoid_f(Mj);   // a resumed state came out of the edge phase: same sigmoid as there, so that a split run equals the straight one bit for bit
        SS[p] = make_float2(Si, Sj);
        const float a0 = hp.mode ? 1.0f : 0.5f * (Si + Sj);  // explain.py:665-678 ; gradient baseline: the adjacency itself
        a[ppij[p]] = a0;
        a[ppji[p]] = a0;
        {   // d/dA_ij + d/dA_ji of y^T (D - A) y / n^2 (explain.py:780-793): constant over the epochs
          const float yd = (float)__ldg(A.g.pred_label + lo2gid[pi[p]]) - (float)__ldg(A.g.pred_label + lo2gid[pj[p]]);
          lapg[p] = lap_over_nn * yd * yd;
        }
        if (hp.out_iter == 0 && !hp.mode) {
          A.out_mask[edge_off + oij] = a0;
          A.out_mask[edge_off + oji] = a0;
          if (A.x.mask_param_out != nullptr) { A.x.mask_param_out[edge_off + oij] = Mi; A.x.mask_param_out[edge_off + oji] = Mj; }
          if (A.x.adam_m_out != nullptr) { A.x.adam_m_out[edge_off + oij] = m2.x; A.x.adam_m_out[edge_off + oji] = m2.y; }
          if (A.x.adam_v_out != nullptr) { A.x.adam_v_out[edge_off + oij] = v2.x; A.x.adam_v_out[edge_off + oji] = v2.y; }
        }
      }
    }
    for (int e = tid; e < e_d; e += NT) gE[e] = 0.f;   // slots outside the < n2 prefixes are never written and must read as 0
    for (int i = tid; i < n; i += NT) {
      const int r0 = irp[i], r1 = irp[i + 1];
      cnt2[i] = prefix_below(icol, r0, r1, n2);
      if (i < n2) cnt1[i] = prefix_below(icol, r0, r1, n1);
    }
    __syncthreads();

    const int np1 = prefix_below(pi, 0, np, n1);   // pairs are sorted by i: the first np1 touch rows < n1 (layer-2/3 terms)
    // ------------------------------------------------------------------ epochs
    const bool timed = A.dbg != nullptr && qi == 0;
#define GXS_MARK(k) if (timed && warp == 0) { const long long c_ = clock64(); if (lane == 0) { s_ph[k] += c_ - s_ph[8]; s_ph[8] = c_; } __syncwarp(); }
    if (timed && warp == 0) { const long long c_ = clock64(); if (lane == 0) { for (int k = 0; k < 8; ++k) s_ph[k] = 0; s_ph[8] = c_; } __syncwarp(); }
    for (int it = 1; it <= hp.iters; ++it) {
      // ---- F0: all nodes: P = (X . sigmoid(feat_mask)) W1                         (explain.py:707, models.py:70-71)
      if (xvec) {
        for (int idx = tid; idx < dp * HS; idx += NT) W1m[idx] = W1s[idx] * sF[idx / HS];   // fold the feature mask into W1
        __syncthreads();
        dense_forward_tiles<HID>(n, d, dp, warp, nwarps, lane, A.g.feat, lo2gid, W1m, stage, P);
      } else {
        const float4 s4 = lane < D4 ? ld4(sF + 4 * lane) : make_float4(0.f, 0.f, 0.f, 0.f);
        const int chunk = (D4 + epi - 1) / epi;            // the four lane groups split the feature axis
        const int f0 = G.grp * chunk, f1 = min(D4, f0 + chunk);
        for (int j = warp; j < n; j += nwarps) {     // (rare path: d % 4 != 0, scalar feature loads)
          const float4 x = lane < D4 ? load_x4(A.g.feat + (int64_t)lo2gid[j] * d, lane, d, false) : make_float4(0.f, 0.f, 0.f, 0.f);
          if (lane < D4) st4(zw + 4 * lane, make_float4(x.x * s4.x, x.y * s4.y, x.z * s4.z, x.w * s4.w));
          __syncwarp();
          float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
          if (q < H4 && f0 < f1) acc = group_dense(zw + 4 * f0, f1 - f0, W1s + 4 * f0 * HS, HS, q, acc);
#pragma unroll
          for (int o = 8; o <= 16; o <<= 1) {
            acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
            acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
          }
          if (G.grp == 0 && q < H4) st4(P + j * HS + 4 * q, acc);
          __syncwarp();
        }
      }
      __syncthreads();
      GXS_MARK(0)
      // ---- F1: rows [0,n2): Y1 = A_m P + b1 ; row normalise                                   (models.py:70-78)
      staged_rows<HID, false, false>(n2, warp, nwarps, lane, icol, a, P, stage, astage, zw, nullptr, nullptr,
        [&](int i, int& r0, int& r1) { r0 = irp[i]; r1 = irp[i + 1]; },
        [&](int i, float4 z) {
          float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
          if (lane < H4) { const float4 b = ld4(bs + 4 * lane); y = make_float4(z.x + b.x, z.y + b.y, z.z + b.z, z.w + b.w); }
          const float ss = warp_sum(y.x * y.x + y.y * y.y + y.z * y.z + y.w * y.w);
          const float qn = fmaxf(sqrtf(ss), 1e-12f);  // F.normalize(p=2, dim=2), eps 1e-12
          if (lane < H4) st4(Yh1 + i * HS + 4 * lane, make_float4(y.x / qn, y.y / qn, y.z / qn, y.w / qn));
          if (lane == 0) q1[i] = qn;
        });
      __syncthreads();
      GXS_MARK(1)
      // ---- F2: rows [0,n1): Y2 = (A_m relu(Yh1)) W2 + b2 ; row normalise
      staged_rows<HID, true, false>(n1, warp, nwarps, lane, icol, a, Yh1, stage, astage, zw, nullptr, nullptr,
        [&](int i, int& r0, int& r1) { r0 = irp[i]; r1 = irp[i + 1]; },
        [&](int i, float4 z) {
          if (lane < H4) st4(zw + 4 * lane, z);
          __syncwarp();
          float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
          if (lane < H4) y = group_dense(zw, H4, W2s, HS, lane, ld4(bs + HID + 4 * lane));
          const float ss = warp_sum(y.x * y.x + y.y * y.y + y.z * y.z + y.w * y.w);
          const float qn = fmaxf(sqrtf(ss), 1e-12f);
          if (lane < H4) st4(Yh2 + i * HS + 4 * lane, make_float4(y.x / qn, y.y / qn, y.z / qn, y.w / qn));
          if (lane == 0) q2[i] = qn;
          __syncwarp();
        });
      __syncthreads();
      GXS_MARK(2)
      // ---- S: row r (= level-order id 0): layer 3, readout, softmax, -log p[gt], layer-3 backward
      if (warp == 0) {
        {
          const int r0 = irp[0], r1 = irp[1];
          float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
          if (q < H4) acc = gather_row<int32_t, true, 4>(r0 + G.grp, r1, epi, icol, a, Yh2, HS, q);
          st4(zw + lane * 4, acc);
        }
        __syncwarp();
        float z = 0.f;
        if (lane < HID)
          for (int g2 = 0; g2 < epi; ++g2) z += zw[(g2 * 8 + (lane >> 2)) * 4 + (lane & 3)];
        __syncwarp();
        if (lane < HID) zw[lane] = z;
        __syncwarp();
        float y3 = lane < EMB ? bs[2 * HID + lane] : 0.f;
        if (lane < EMB)
          for (int f = 0; f < HID; ++f) y3 = fmaf(zw[f], W3s[f * EMB + lane], y3);
        const float ss = warp_sum(lane < EMB ? y3 * y3 : 0.f);
        const float q3 = fmaxf(sqrtf(ss), 1e-12f);
        const float yh3 = lane < EMB ? y3 / q3 : 0.f;
        const float e1v = lane < HID ? fmaxf(Yh1[lane], 0.f) : 0.f;  // row 0 of H1
        const float e2v = lane < HID ? fmaxf(Yh2[lane], 0.f) : 0.f;  // row 0 of H2
        // logits = pred_model(concat) (models.py:260,375), softmax over classes (explain.py:714)
        for (int c = 0; c < C; ++c) {
          const float* wp = Wpp + c * PD;
          float t = 0.f;
          if (lane < HID) t = fmaf(e1v, wp[lane], fmaf(e2v, wp[HID + lane], t));
          if (lane < EMB) t = fmaf(yh3, wp[2 * HID + lane], t);
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
        if (kTrace) {
          float* const tr = s_tr + (NT / 32) * 4;
          if (lane == 0) { const float lg = logit[gt]; tr[0] = -((lg - mx) - logf(se)); tr[1] = expf(lg - mx) / se; }
          if (A.x.trace_pred != nullptr) {
            float* trp = A.x.trace_pred + ((int64_t)task_id * A.x.epochs + (it - 1)) * C;
            for (int c = lane; c < C; c += 32) trp[c] = expf(logit[c] - mx) / se;
          }
          float fs = 0.f;   // feat_size_loss = coeff * mean(sigmoid(feat_mask)) (explain.py:763-766)
          for (int f = lane; f < d; f += 32) fs += sF[f];
          fs = warp_sum(fs);
          if (lane == 0) tr[2] = hp.c_feat_size * fs / (float)d;
          __syncwarp();
        }
        for (int c = lane; c < C; c += 32)
          logit[c] = expf(logit[c] - mx) / se - (c == gt ? 1.f : 0.f);  // dL/dlogits = p - onehot(gt) (explain.py:750-753)
        __syncwarp();
        float d1 = 0.f, d2 = 0.f, d3 = 0.f;
        for (int c = 0; c < C; ++c) {
          const float gc = logit[c];
          const float* wp = Wpp + c * PD;
          if (lane < HID) { d1 = fmaf(gc, wp[lane], d1); d2 = fmaf(gc, wp[HID + lane], d2); }
          if (lane < EMB) d3 = fmaf(gc, wp[2 * HID + lane], d3);
        }
        if (lane < HID) { dE[lane] = d1; dE[HS + lane] = d2; }
        // backward of y/max(|y|,eps): dY = (dYh - Yh <Yh,dYh>)/q ; dZ3 = dY3 W3^T
        const float s3 = warp_sum(yh3 * d3);
        const float dy3 = lane < EMB ? (d3 - yh3 * s3) / q3 : 0.f;
        __syncwarp();
        if (lane < EMB) zw[lane] = dy3;
        __syncwarp();
        if (lane < HID) dZ3[lane] = dot_v4(zw, W3s + lane * EMB, EMB / 4);
      }
      __syncthreads();
      GXS_MARK(3)
      // ---- B2: rows {r} U N(r): dYh2 = dEmb2 (row r) + a[r,j] dZ3 (j in N(r)), relu', normalise', dZ2 = dY2 W2^T
      {
        const int r0 = irp[0];
        const int items = 1 + irp[1] - r0;
        const int ntask = (items + epi - 1) / epi;
        for (int t = warp; t < ntask; t += nwarps) {
          const int item = t * epi + G.grp;
          const bool act = item < items;
          int j = 0;
          float coef = 1.f;
          const float* dsrc = dE + HS;
          if (act && item > 0) {
            const int e = r0 + item - 1;
            j = icol[e];
            coef = a[e];
            dsrc = dZ3;
          }
          float4 yh = make_float4(0.f, 0.f, 0.f, 0.f), dy = yh;
          if (act && q < H4) {
            yh = ld4(Yh2 + j * HS + 4 * q);
            const float4 g4 = ld4(dsrc + 4 * q);
            dy.x = yh.x > 0.f ? coef * g4.x : 0.f;   // relu backward: grad where input > 0
            dy.y = yh.y > 0.f ? coef * g4.y : 0.f;
            dy.z = yh.z > 0.f ? coef * g4.z : 0.f;
            dy.w = yh.w > 0.f ? coef * g4.w : 0.f;
          }
          const float sdot = group_sum(yh.x * dy.x + yh.y * dy.y + yh.z * dy.z + yh.w * dy.w, G);
          if (act && q < H4) {
            const float qn = q2[j];
            st4(zw + lane * 4, make_float4((dy.x - yh.x * sdot) / qn, (dy.y - yh.y * sdot) / qn,
                                           (dy.z - yh.z * sdot) / qn, (dy.w - yh.w * sdot) / qn));
          }
          __syncwarp();
          if (act && q < H4)
            st4(dZ2 + j * HS + 4 * q, group_dense(zw + G.gbase * 4, H4, W2t, HS, q, make_float4(0.f, 0.f, 0.f, 0.f)));
          __syncwarp();
        }
      }
      __syncthreads();
      GXS_MARK(4)
      // ---- B1: rows [0,n2): dH1 = A_m^T dZ2 (only columns < n1 carry gradient), relu', normalise' -> dY1
      staged_rows<HID, false, false>(n2, warp, nwarps, lane, icol, a, dZ2, stage, astage, zw, nullptr, nullptr,
        [&](int i, int& r0, int& r1) { r0 = irp[i]; r1 = r0 + cnt1[i]; },
        [&](int i, float4 dh) {
          float4 yh = make_float4(0.f, 0.f, 0.f, 0.f), dy = yh;
          if (lane < H4) {
            yh = ld4(Yh1 + i * HS + 4 * lane);
            if (i == 0) { const float4 e4 = ld4(dE + 4 * lane); dh.x += e4.x; dh.y += e4.y; dh.z += e4.z; dh.w += e4.w; }
            dy.x = yh.x > 0.f ? dh.x : 0.f; dy.y = yh.y > 0.f ? dh.y : 0.f;
            dy.z = yh.z > 0.f ? dh.z : 0.f; dy.w = yh.w > 0.f ? dh.w : 0.f;
          }
          const float sdot = warp_sum(yh.x * dy.x + yh.y * dy.y + yh.z * dy.z + yh.w * dy.w);
          if (lane < H4) {
            const float qn = q1[i];
            st4(dY1 + i * HS + 4 * lane, make_float4((dy.x - yh.x * sdot) / qn, (dy.y - yh.y * sdot) / qn,
                                                     (dy.z - yh.z * sdot) / qn, (dy.w - yh.w * sdot) / qn));
          }
        });
      __syncthreads();
      GXS_MARK(5)
      // ---- B0: all nodes: dP = A_m^T dY1 (columns < n2 of row j), then dL/dsF += X_j (.) (dP_j W1^T) for the warp's own rows
      {
        staged_rows<HID, false, true>(n, warp, nwarps, lane, icol, a, dY1, stage, astage, zw, P, gE,
          [&](int i, int& r0, int& r1) { r0 = irp[i]; r1 = r0 + cnt2[i]; },
          [&](int i, float4 z) { if (lane < H4) st4(dP + i * HS + 4 * lane, z); });
        __syncthreads();   // the tiles below read dP rows written by other warps
        float4 gacc = make_float4(0.f, 0.f, 0.f, 0.f);
        if (xvec) {
          gacc = dense_backward_tiles<HID>(n, d, dp, warp, nwarps, lane, A.g.feat, lo2gid, W1t, stage, dP);
        } else {
          for (int j = warp; j < n; j += nwarps) {
            if (lane < H4) st4(zw + 4 * lane, ld4(dP + j * HS + 4 * lane));
            __syncwarp();
            if (lane < D4) {
              const float4 o = group_dense(zw, H4, W1t, dp, lane, make_float4(0.f, 0.f, 0.f, 0.f));
              const float4 x = load_x4(A.g.feat + (int64_t)lo2gid[j] * d, lane, d, false);
              gacc.x = fmaf(o.x, x.x, gacc.x); gacc.y = fmaf(o.y, x.y, gacc.y);
              gacc.z = fmaf(o.z, x.z, gacc.z); gacc.w = fmaf(o.w, x.w, gacc.w);
            }
            __syncwarp();
          }
        }
        if (lane < D4) st4(gFp + warp * dp + 4 * lane, gacc);  // per-warp partial, summed in warp order below
      }
      __syncthreads();
      GXS_MARK(6)
      // ---- P: per undirected edge: dA_ij, dA_ji, symmetrise, regularisers, Adam, next mask value
      {
        const float2 tab = __ldg(hp.adam_tab + (it - 1));
        const float step = tab.x, bc2s = tab.y, bc2s_inv = 1.0f / tab.y;
        const bool last = (it == hp.out_iter);   // the mask built after this update is the one the reference returns
        // feature mask: dL/dF = sF(1-sF) (sum_j X_j (.) dX'_j + feat_size/d) ; Adam (explain.py:766, train_utils.py:10)
        for (int f = tid; f < d && !hp.mode; f += NT) {
          float gsum = 0.f;
          for (int w = 0; w < nwarps; ++w) gsum += gFp[w * dp + f];
          const float s = sF[f];
          const float g = s * (1.f - s) * (gsum + hp.c_feat_size / (float)d);
          float mf = mF[f], vf = vF[f], Fv = Fm[f];
          mf = mf + (g - mf) * hp.one_minus_b1;
          vf = vf * hp.b2 + hp.one_minus_b2 * g * g;
          Fv = Fv - step * (mf / (sqrtf(vf) / bc2s + hp.eps));
          mF[f] = mf; vF[f] = vf; Fm[f] = Fv;
          const float sn = sigmoid_f(Fv);
          sF[f] = sn;
          if (last) {
            if (A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = sn;
            if (A.x.feat_state_out != nullptr) {
              float* fo = A.x.feat_state_out + (int64_t)task_id * 3 * d;
              fo[f] = Fv; fo[d + f] = mf; fo[2 * d + f] = vf;
            }
          }
        }
        float trS = 0.f, trH = 0.f, trL = 0.f, trD = 0.f;   // trace: this thread's share of sum S, sum H(S), sum a (y_i-y_j)^2, sum 2a'
        // The layer-1 dots <dY1[i], P[j]> and <dY1[j], P[i]> were taken in B0 while the gathered rows were staged (gE);
        // only the few pairs touching rows < n1 (listed first) carry layer-2/3 terms.
        if (hp.mode) {
          // gradient baseline (explain.py:125-133): mask_ij = sigmoid(|dL/dA_ij| + |dL/dA_ji|) on the edges
          for (int p = tid; p < np; p += NT) {
            float gij = gE[ppji[p]], gji = gE[ppij[p]];
            if (p < np1) {
              const int i = pi[p], j = pj[p];
              gij += dot_relu_v4(dZ2 + i * HS, Yh1 + j * HS, H4);
              if (j < n1) gji += dot_relu_v4(dZ2 + j * HS, Yh1 + i * HS, H4);
              if (i == 0) gij += dot_relu_v4(dZ3, Yh2 + j * HS, H4);
            }
            const float an = sigmoid_f(fabsf(gij) + fabsf(gji));
            A.out_mask[edge_off + poij[p]] = an;
            A.out_mask[edge_off + poji[p]] = an;
          }
        } else
        for (int p = tid; p < np; p += NT) {
          const int sij = ppij[p], sji = ppji[p];
          float Gd = lapg[p] + gE[sji] + gE[sij];
          if (p < np1) {
            const int i = pi[p], j = pj[p];   // i < j, i < n1
            Gd += dot_relu_v4(dZ2 + i * HS, Yh1 + j * HS, H4);
            if (j < n1) Gd += dot_relu_v4(dZ2 + j * HS, Yh1 + i * HS, H4);
            if (i == 0) Gd += dot_relu_v4(dZ3, Yh2 + j * HS, H4);
          }
          Gd *= 0.5f;  // sym_mask = (S + S^T)/2 (explain.py:671)
          float2 Mv = MM[p];
          const float2 Sv = SS[p];
          if (kTrace) {
            trS += Sv.x + Sv.y; trH += bern_entropy(Sv.x) + bern_entropy(Sv.y);
            if (lap_over_nn > 0.f) trL += 0.5f * (Sv.x + Sv.y) * (lapg[p] / lap_over_nn);   // lapg = c_lap/n^2 (y_i-y_j)^2
          }
          // size: coeff*sum(S) ; entropy: mean over n^2 of H(S), dH/dM = -M S(1-S) (explain.py:755-770)
          const float gi = Sv.x * (1.f - Sv.x) * (Gd + hp.c_size - ent_over_nn * Mv.x);
          const float gj = Sv.y * (1.f - Sv.y) * (Gd + hp.c_size - ent_over_nn * Mv.y);
          float2 m2 = mm[p], v2 = vv[p];
          m2.x = m2.x + (gi - m2.x) * hp.one_minus_b1;
          m2.y = m2.y + (gj - m2.y) * hp.one_minus_b1;
          v2.x = v2.x * hp.b2 + hp.one_minus_b2 * gi * gi;
          v2.y = v2.y * hp.b2 + hp.one_minus_b2 * gj * gj;
          Mv.x = Mv.x - adam_delta_fast(m2.x, v2.x, step, bc2s, bc2s_inv, hp.eps, ieee);
          Mv.y = Mv.y - adam_delta_fast(m2.y, v2.y, step, bc2s, bc2s_inv, hp.eps, ieee);
          const float2 Sn = make_float2(sigmoid_fast(Mv.x, ieee), sigmoid_fast(Mv.y, ieee));
          MM[p] = Mv; mm[p] = m2; vv[p] = v2; SS[p] = Sn;
          const float an = 0.5f * (Sn.x + Sn.y);
          if (kTrace) trD += 2.0f * an;
          a[sij] = an;
          a[sji] = an;
          if (last) {
            const int64_t oij = edge_off + poij[p], oji = edge_off + poji[p];
            A.out_mask[oij] = an;
            A.out_mask[oji] = an;
            if (A.x.mask_param_out != nullptr) { A.x.mask_param_out[oij] = Mv.x; A.x.mask_param_out[oji] = Mv.y; }
            if (A.x.adam_m_out != nullptr) { A.x.adam_m_out[oij] = m2.x; A.x.adam_m_out[oji] = m2.y; }
            if (A.x.adam_v_out != nullptr) { A.x.adam_v_out[oij] = v2.x; A.x.adam_v_out[oji] = v2.y; }
          }
        }
        if (kTrace) {
          trS = warp_sum(trS); trH = warp_sum(trH); trL = warp_sum(trL); trD = warp_sum(trD);
          if (lane == 0) { s_tr[warp * 4 + 0] = trS; s_tr[warp * 4 + 1] = trH; s_tr[warp * 4 + 2] = trL; s_tr[warp * 4 + 3] = trD; }
        }
      }
      __syncthreads();
      if (kTrace && tid == 0) {   // raw terms of epoch it-1 over the INNER pairs (trace_finalize_kernel assembles the columns)
        float sS = 0.f, sH = 0.f, sLp = 0.f, sD = 0.f;
        for (int w = 0; w < nwarps; ++w) { sS += s_tr[w * 4]; sH += s_tr[w * 4 + 1]; sLp += s_tr[w * 4 + 2]; sD += s_tr[w * 4 + 3]; }
        float* row = A.x.trace + ((int64_t)task_id * A.x.epochs + (it - 1)) * GX_TRACE_COLS;
        const float* const tr = s_tr + (NT / 32) * 4;
        row[0] = sS; row[1] = tr[0]; row[2] = sH; row[3] = sLp; row[4] = sD; row[5] = tr[2]; row[6] = 0.f; row[7] = tr[1];
      }
      GXS_MARK(7)
    }
    if (timed && tid == 0) {
      float* o = A.dbg + (1 << 19);
      for (int k = 0; k < 8; ++k) o[k] = (float)s_ph[k];
      o[8] = (float)n; o[9] = (float)n1; o[10] = (float)n2; o[11] = (float)np; o[12] = (float)e_d; o[13] = (float)NT;
    }
  }
}

template <int HID, int EMB, int NT, bool kTrace>
cudaError_t launch_stream_nt(const GxExplainLaunch& cfg, const ExplainArgs& args, cudaStream_t s) {
  auto kern = explain_stream_kernel<HID, EMB, NT, kTrace>;
  const StreamSmem S = stream_smem(gx_round_up(args.m.d, 4), HID, EMB, args.m.C, NT / 32);
  const int bytes = S.total * 4;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return e;
  kern<<<cfg.grid, NT, bytes, s>>>(args);
  return cudaGetLastError();
}
template <int HID, int EMB>
cudaError_t launch_stream(const GxExplainLaunch& cfg, const ExplainArgs& args, cudaStream_t s) {
  if (args.x.trace != nullptr) return launch_stream_nt<HID, EMB, GX_STREAM_THREADS, true>(cfg, args, s);
  return launch_stream_nt<HID, EMB, GX_STREAM_THREADS, false>(cfg, args, s);
}

}  // namespace

cudaError_t gx_launch_explain_stream(const GxExplainLaunch& cfg, const GxGraphDev& g, const GxModelDev& m,
                                     const GxHparamsDev& hp, const GxPlanArrays& plan, const float* m0,
                                     float* out_mask, float* out_feat, cudaStream_t s) {
  const ExplainArgs args = explain_args(cfg, g, m, hp, plan, m0, out_mask, out_feat);
  if (m.hid == 20 && m.emb == 20) return launch_stream<20, 20>(cfg, args, s);
  if (m.hid == 32 && m.emb == 32) return launch_stream<32, 32>(cfg, args, s);   // any width <= 32, zero-padded by gx_set_model
  return cudaErrorInvalidValue;
}
