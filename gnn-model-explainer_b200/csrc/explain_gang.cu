// explain_gang.cu -- K2g: the streaming mask-optimisation kernel for explained nodes whose k-hop state does not fit shared memory
// (BASELINE config 5: 10^4..10^5-node neighbourhoods, d = 128), second generation.
//
// Same arithmetic contract as explain_node.cu / explain_stream.cu (explainer/explain.py:137-146,665-715,740-808 + autograd + Adam,
// models.py:58-80,230-267,363-376); what changed against explain_stream.cu (one CTA per task, cp.async staging, FP32 FMA GEMMs):
//   * GANGS: G co-resident CTAs (one per SM, cooperative launch) share ONE task; rows, pairs and feature tiles are dealt over the
//     gang's warps, phases are separated by a gang barrier (one atomic counter in L2 + fence).  G is chosen per launch so that the
//     randomly accessed state of the tasks in flight (a, gE, P, dP, dY1: 8 B per directed edge + 240 B per node) stays L2 resident:
//     for the 100 000-node graphs one task spans all 132 SMs and HBM only sees the sequential streams (CSR, pair state).
//     Nothing in the arithmetic depends on G (row sums are taken by one warp, the dL/dsF reduction runs over fixed 128-node blocks),
//     so a sharded multi-GPU run stays bit-identical to the single-GPU run whatever G the launches pick.
//   * SPARSE PASSES: a warp owns a row and walks it six edges at a time (lane = (edge slot, float4 of the 80-byte source row)):
//     one coalesced index/value load and one 16-byte L2 gather per lane and step, four steps in flight, no staging through shared
//     memory; ~2 instructions per edge instead of ~12.  Rows longer than kLongEdges are sliced over all warps of their CTA.
//   * DENSE FEATURE PASSES on the tensor cores: P = X (sF (.) W1) (F0) and dL/dsF = colsum(X (.) (dP W1^T)) (B0) are
//     mma.sync m16n8k8 TF32 with the 3xTF32 split (x = hi + lo; lo*hi + hi*lo + hi*hi, FP32 accumulate: FP32-grade accuracy);
//     the 16-node feature tiles are staged by the TMA engine (cp.async.bulk global -> shared, one 512-byte row per copy,
//     completion on an mbarrier, double buffered per warp).
// Phases per epoch (gang barrier each): F0 | F1 | F2 | S (every CTA, redundantly) | B2 | B1 | B0s | B0d | P.
// Supported: feature widths d <= 128 (wider inputs keep explain_stream.cu), hidden width 20 or 32.
#include "explain_common.cuh"
#include "mma_tf32.cuh"

namespace {

#ifndef GXG_UNROLL
#define GXG_UNROLL 4   // steps of six edges a warp keeps in flight in the sparse passes
#endif
constexpr int kGangThreads = 512;    // 16 warps, 128 registers per thread (the tensor-core passes hold 24 A fragments + 32 accumulators)
#ifndef GXG_DENSE_WARPS
#define GXG_DENSE_WARPS 6
#endif
#ifndef GXG_TILE_BUFS
#define GXG_TILE_BUFS 2
#endif
constexpr int kTileBufs = GXG_TILE_BUFS;   // tile buffers per dense warp (2 = the next tile is in flight while the current one is consumed)
constexpr int kDenseWarps = GXG_DENSE_WARPS;       // warps of a CTA that run the TMA + tensor-core feature passes (two 8.4 KB tiles each; 8 would not fit 227 KB at d = 128)
constexpr int kLongEdges = 512;      // rows with more edges are sliced over all warps of one CTA
constexpr int kBlockTiles = 8;       // dL/dsF is reduced over fixed blocks of 8 tiles (128 nodes): independent of the gang size

struct GangSmem {
  int W1s, Whi, Wlo, Thi, Tlo, W2s, W2t, W3s, bs, sF, F, mF, vF, zs, dE, dZ3, logit, Wp, part, red, xt, pt, bar, total;
  int xs, ldb, ldt, dp8, ntl;
};
__host__ __device__ inline GangSmem gang_smem(int d, int hid, int emb, int C, int nwarps) {
  GangSmem S;
  const int dp = gx_round_up(d, 4), dp8 = gx_round_up(d, 8);
  const int ntl = (hid + 7) / 8, n8 = ntl * 8;
  S.dp8 = dp8; S.ntl = ntl;
  S.xs = dp8 + 4;                          // feature-tile row stride (floats): = 4 mod 8 -> conflict-free A fragments
  S.ldb = n8 + (n8 % 32 == 0 ? 8 : 0);     // row stride of the (k = feature, n = hidden) operand
  S.ldt = dp8 + 8;                         // row stride of the (k = hidden, n = feature) operand
  int o = 0;
  auto take = [&](int words) { int r = o; o += gx_round_up(words, 4); return r; };
  S.W1s = take(dp * hid);
  S.Whi = take(dp8 * S.ldb); S.Wlo = take(dp8 * S.ldb);   // tf32 hi / lo of sF (.) W1, rebuilt every epoch
  S.Thi = take(n8 * S.ldt); S.Tlo = take(n8 * S.ldt);     // tf32 hi / lo of W1^T (rows >= hid are zero)
  S.W2s = take(hid * hid); S.W2t = take(hid * hid); S.W3s = take(hid * emb); S.bs = take(2 * hid + emb);
  S.sF = take(dp); S.F = take(dp); S.mF = take(dp); S.vF = take(dp);
  S.zs = take(nwarps * 128);
  S.dE = take(2 * hid); S.dZ3 = take(hid); S.logit = take(C < 32 ? 32 : C);
  S.Wp = take(C * (2 * hid + emb + 1) <= GX_WP_SMEM_MAX ? C * (2 * hid + emb + 1) : 0);
  S.part = take(nwarps * hid);             // long rows: per-warp partial aggregates
  S.red = take(kGangThreads > dp ? kGangThreads : dp);   // dL/dsF: slice partials
  S.xt = take(kDenseWarps * kTileBufs * 16 * S.xs);      // feature tiles (TMA destination), kTileBufs per dense warp
  S.pt = take(kDenseWarps * kTileBufs * 16 * hid);       // dP tiles
  S.bar = take(kDenseWarps * 2 * 2);                     // one mbarrier (8 bytes) per tile buffer
  S.total = o;
  return S;
}

// ------------------------------------------------------------------------------------------------ gang barrier
// Monotonic counter in global memory; every CTA of the gang arrives once per barrier.  __syncthreads + fence + atomic is the
// release, the spin + fence the acquire (the fence also invalidates this SM's L1, so plain loads see the other CTAs' stores).
struct GangBar {
  unsigned long long* ctr;
  unsigned long long target;
  int G;
  __device__ __forceinline__ void sync() {
    if (G == 1) { __syncthreads(); return; }
    __syncthreads();
    if (threadIdx.x == 0) {
      target += (unsigned long long)G;
      __threadfence();
      atomicAdd(ctr, 1ull);
      unsigned long long v;
      do { asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(ctr) : "memory"); } while (v < target);
      __threadfence();
    }
    __syncthreads();
  }
};

// ------------------------------------------------------------------------------------------------ TMA (bulk copy) + mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tWAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
// global -> shared bulk copy by the TMA engine (UBLKCP in SASS); bytes % 16 == 0, both addresses 16-byte aligned
__device__ __forceinline__ void tma_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t l2_policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(l2_policy) : "memory");
}

__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }

// ------------------------------------------------------------------------------------------------ L2 residency control
// One task streams ~0.4 GB per epoch through the 126 MB L2 (CSR indices, pair indices and optimiser state, feature rows) while its
// randomly accessed arrays (a, gE: 8 B per directed edge; P, dP, dY1: 240 B per node) are touched 4-byte-wise from all SMs: without
// a hint the streams evict them and every scattered access becomes a DRAM read-modify-write (the edge phase was DRAM-latency
// bound).  Streams are therefore loaded / stored with an evict_first policy, the scattered arrays with evict_last.
struct L2Pol { uint64_t first, last; };
__device__ __forceinline__ L2Pol make_l2pol() {
  L2Pol p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p.first));
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p.last));
  return p;
}
__device__ __forceinline__ int ld_i32_stream(const int32_t* a, uint64_t pol) { int v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s32 %0, [%1], %2;" : "=r"(v) : "l"(a), "l"(pol)); return v; }
__device__ __forceinline__ float ld_f32_pol(const float* a, uint64_t pol) { float v; asm volatile("ld.global.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(a), "l"(pol) : "memory"); return v; }
__device__ __forceinline__ float4 ld_v4_pol(const float* a, uint64_t pol) {
  float4 v;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(a), "l"(pol) : "memory");
  return v;
}
__device__ __forceinline__ float2 ld_v2_pol(const float2* a, uint64_t pol) {
  float2 v;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.f32 {%0,%1}, [%2], %3;" : "=f"(v.x), "=f"(v.y) : "l"(a), "l"(pol) : "memory");
  return v;
}
__device__ __forceinline__ void st_f32_pol(float* a, float v, uint64_t pol) { asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(a), "f"(v), "l"(pol) : "memory"); }
__device__ __forceinline__ void st_v2_pol(float2* a, float2 v, uint64_t pol) { asm volatile("st.global.L2::cache_hint.v2.f32 [%0], {%1,%2}, %3;" ::"l"(a), "f"(v.x), "f"(v.y), "l"(pol) : "memory"); }
__device__ __forceinline__ void st_v4_pol(float* a, float4 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}

// ------------------------------------------------------------------------------------------------ sparse passes
// One row segment [r0,r1) by one warp: lane = (edge slot es, float4 index q); returns this lane's partial aggregate
//   sum_{e = r0 + es, step EPL} a[e] f(src[icol[e]])[4q..4q+3]
// kDot: gout[e] = <src[icol[e]], dv> for every edge (dv = this lane's float4 of the row's dot vector).
#ifdef GXG_OUTLINE_SEGMENT
#define GXG_SEG_INLINE __noinline__
#else
#define GXG_SEG_INLINE __forceinline__
#endif
template <int HID, bool kRelu, bool kDot>
__device__ GXG_SEG_INLINE float4 row_segment(int r0, int r1, int lane, const int32_t* __restrict__ icol, const float* a, const float* src,
                                              float4 dv, float* gout, const L2Pol pol) {
  constexpr int H4 = HID / 4, EPL = 32 / H4, UN = GXG_UNROLL;
  const int es = lane / H4, q = lane - es * H4;
  const bool act = es < EPL;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  const float* const src_q = src + 4 * q;
  // software pipeline: the indices / values of step k+1 are loaded while the gathers of step k are in flight, so a step costs one
  // memory latency instead of two (the loop is latency bound: 16 warps x 24 edges in flight per SM)
  int cn[UN];
  float an[UN];
#pragma unroll
  for (int k = 0; k < UN; ++k) {
    const int ek = r0 + es + k * EPL;
    const bool ok = act && ek < r1;
    cn[k] = ok ? ld_i32_stream(icol + ek, pol.first) : -1;
    an[k] = ok ? ld_f32_pol(a + ek, pol.last) : 0.f;
  }
#pragma unroll 1
  for (int e = r0 + es; e - es < r1; e += UN * EPL) {
    int c[UN];
    float av[UN];
    float4 v[UN];
#pragma unroll
    for (int k = 0; k < UN; ++k) { c[k] = cn[k]; av[k] = an[k]; }
#pragma unroll
    for (int k = 0; k < UN; ++k) v[k] = c[k] >= 0 ? ld_v4_pol(src_q + (size_t)c[k] * HID, pol.last) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < UN; ++k) {
      const int ek = e + (UN + k) * EPL;
      const bool ok = act && ek < r1;
      cn[k] = ok ? ld_i32_stream(icol + ek, pol.first) : -1;
      an[k] = ok ? ld_f32_pol(a + ek, pol.last) : 0.f;
    }
#pragma unroll
    for (int k = 0; k < UN; ++k) {
      if (kRelu) v[k] = relu4(v[k]);
      fma4(acc, av[k], v[k]);
      if (kDot) {
        float pd = fmaf(v[k].x, dv.x, fmaf(v[k].y, dv.y, fmaf(v[k].z, dv.z, v[k].w * dv.w)));
        if (H4 == 8) {
          pd += __shfl_xor_sync(0xffffffffu, pd, 1); pd += __shfl_xor_sync(0xffffffffu, pd, 2); pd += __shfl_xor_sync(0xffffffffu, pd, 4);
        } else {   // H4 == 5: lanes es*5 .. es*5+4; only the q == 0 lane's sum is used
          const float t1 = pd + __shfl_down_sync(0xffffffffu, pd, 1);
          const float t2 = t1 + __shfl_down_sync(0xffffffffu, t1, 2);
          pd = t2 + __shfl_down_sync(0xffffffffu, pd, 4);
        }
        if (c[k] >= 0 && q == 0) st_f32_pol(gout + e + k * EPL, pd, pol.last);
      }
    }
  }
  return acc;
}
// sum of the edge slots' partials; valid on lanes < H4 (lane q holds features 4q..4q+3)
template <int HID>
__device__ __forceinline__ float4 slot_reduce(float4 z) {
  constexpr int H4 = HID / 4;
  if (H4 == 8) {
#pragma unroll
    for (int o = 8; o <= 16; o <<= 1) {
      z.x += __shfl_xor_sync(0xffffffffu, z.x, o); z.y += __shfl_xor_sync(0xffffffffu, z.y, o);
      z.z += __shfl_xor_sync(0xffffffffu, z.z, o); z.w += __shfl_xor_sync(0xffffffffu, z.w, o);
    }
  } else {   // six slots of five lanes: (s, s+3) first, then s = 0,1,2
    z.x += __shfl_down_sync(0xffffffffu, z.x, 15); z.y += __shfl_down_sync(0xffffffffu, z.y, 15);
    z.z += __shfl_down_sync(0xffffffffu, z.z, 15); z.w += __shfl_down_sync(0xffffffffu, z.w, 15);
    const float x1 = __shfl_down_sync(0xffffffffu, z.x, 5), x2 = __shfl_down_sync(0xffffffffu, z.x, 10);
    const float y1 = __shfl_down_sync(0xffffffffu, z.y, 5), y2 = __shfl_down_sync(0xffffffffu, z.y, 10);
    const float z1 = __shfl_down_sync(0xffffffffu, z.z, 5), z2 = __shfl_down_sync(0xffffffffu, z.z, 10);
    const float w1 = __shfl_down_sync(0xffffffffu, z.w, 5), w2 = __shfl_down_sync(0xffffffffu, z.w, 10);
    z.x = (z.x + x1) + x2; z.y = (z.y + y1) + y2; z.z = (z.z + z1) + z2; z.w = (z.w + w1) + w2;
  }
  return z;
}

// z_i = sum_{e in bounds(i)} a[e] f(src[icol[e]]) for the rows i < Rn of this gang (and the long rows among Rn .. R-1), then epi(i, z) with the warp converged
// (z valid on lanes < H4).  Long rows (full degree > kLongEdges, listed in longlist) are sliced over the warps of the CTA
// that owns them; every other row is taken by one warp.  bounds(i, r0, r1) gives the edge range of row i in this pass.
template <int HID, bool kRelu, bool kDot, typename Bounds, typename Epi>
__device__ __forceinline__ void row_pass(int R, int Rn, int G, int grank, int warp, int nwarps, int lane, const int32_t* __restrict__ irp,
                                         const int32_t* __restrict__ icol, const float* a, const float* src, const float* dotsrc, float* gout,
                                         const int32_t* longlist, int nlong, float* part, int* row_ctr, const L2Pol pol, Bounds bounds, Epi epi) {
  constexpr int H4 = HID / 4, EPL = 32 / H4;
  const int q = lane % H4;
  // long rows of this CTA
  for (int k = grank; k < nlong; k += G) {
    const int i = longlist[k];
    if (i >= R) continue;   // (CTA-uniform)
    int r0, r1;
    bounds(i, r0, r1);
    const int len = r1 - r0;
    const int per = gx_round_up((len + nwarps - 1) / nwarps, 4 * EPL);   // (a multiple of the slot count; independent of the unroll depth)
    const int s0 = min(r1, r0 + warp * per), s1 = min(r1, s0 + per);
    float4 dv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (kDot && lane < EPL * H4) dv = ldcg4(dotsrc + (size_t)i * HID + 4 * q);
    float4 z = slot_reduce<HID>(row_segment<HID, kRelu, kDot>(s0, s1, lane, icol, a, src, dv, gout, pol));
    if (lane < H4) st4(part + warp * HID + 4 * lane, z);
    __syncthreads();
    if (warp == 0) {
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
      if (lane < H4)
        for (int w = 0; w < nwarps; ++w) { const float4 o = ld4(part + w * HID + 4 * lane); t.x += o.x; t.y += o.y; t.z += o.z; t.w += o.w; }
      epi(i, t);
    }
    __syncthreads();
  }
  // everything else: one warp per row.  Row i belongs to CTA i mod G; inside the CTA the warps draw the next row from a shared
  // counter (rows are sorted by degree inside a level, so this is longest-first scheduling; a row's result does not depend on
  // which warp takes it).
  (void)nwarps;
  for (;;) {
    int k = 0;
    if (lane == 0) k = atomicAdd(row_ctr, 1);
    k = __shfl_sync(0xffffffffu, k, 0);
    const int i = k * G + grank;
    if (i >= Rn) break;   // (rows Rn .. R-1: only the long ones, above)
    if (nlong > 0 && irp[i + 1] - irp[i] > kLongEdges) continue;
    int r0, r1;
    bounds(i, r0, r1);
    float4 dv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (kDot && lane < EPL * H4) dv = ldcg4(dotsrc + (size_t)i * HID + 4 * q);
    const float4 z = slot_reduce<HID>(row_segment<HID, kRelu, kDot>(r0, r1, lane, icol, a, src, dv, gout, pol));
    epi(i, z);
  }
}

// Row-parallel variant for SHORT rows (B0 on the outermost nodes: a handful of gradient-carrying neighbours per row): every
// edge slot of the warp (H4 lanes) owns one row and walks its edges with four gathers in flight, so a warp keeps EPL rows in
// flight instead of one; no cross-slot reduction.  out[i] = sum_e a[e] src[icol[e]], gout[e] = <src[icol[e]], dotsrc[i]>.
// Rows R0 .. R-1 of this gang; rows whose full degree exceeds kLongEdges are left to the whole-CTA path of row_pass.
template <int HID, typename Bounds>
__device__ __forceinline__ void short_rows_pass(int R0, int R, int G, int grank, int lane, const int32_t* __restrict__ irp,
                                                const int32_t* __restrict__ icol, const float* a, const float* src, const float* dotsrc,
                                                float* gout, float* out, int nlong, int* row_ctr, const L2Pol pol, Bounds bounds) {
  constexpr int H4 = HID / 4, EPL = 32 / H4, UN = 4;
  const int es = lane / H4, q = lane - es * H4;
  const bool act = es < EPL;
  for (;;) {
    int k = 0;
    if (lane == 0) k = atomicAdd(row_ctr, EPL);
    k = __shfl_sync(0xffffffffu, k, 0);
    if (R0 + k * G + grank >= R) break;   // (rows of this CTA: R0 + grank, R0 + grank + G, ...)
    const int i = R0 + (k + es) * G + grank;
    int r0 = 0, r1 = 0;
    bool mine = act && i < R;
    if (mine && nlong > 0 && irp[i + 1] - irp[i] > kLongEdges) mine = false;
    if (mine) bounds(i, r0, r1);
    const float4 dv = mine ? ldcg4(dotsrc + (size_t)i * HID + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int wl = r1 - r0;   // warp-wide longest row: uniform trip count (the dot reduction shuffles need every lane)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wl = max(wl, __shfl_xor_sync(0xffffffffu, wl, o));
    const float* const src_q = src + 4 * q;
    for (int e0 = 0; e0 < wl; e0 += UN) {
      int c[UN];
      float av[UN];
      float4 v[UN];
#pragma unroll
      for (int u = 0; u < UN; ++u) {
        const int e = r0 + e0 + u;
        const bool ok = e < r1;
        c[u] = ok ? ld_i32_stream(icol + e, pol.first) : -1;
        av[u] = ok ? ld_f32_pol(a + e, pol.last) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < UN; ++u) v[u] = c[u] >= 0 ? ld_v4_pol(src_q + (size_t)c[u] * HID, pol.last) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < UN; ++u) {
        fma4(acc, av[u], v[u]);
        float pd = fmaf(v[u].x, dv.x, fmaf(v[u].y, dv.y, fmaf(v[u].z, dv.z, v[u].w * dv.w)));
        if (H4 == 8) {
          pd += __shfl_xor_sync(0xffffffffu, pd, 1); pd += __shfl_xor_sync(0xffffffffu, pd, 2); pd += __shfl_xor_sync(0xffffffffu, pd, 4);
        } else {
          const float t1 = pd + __shfl_down_sync(0xffffffffu, pd, 1);
          const float t2 = t1 + __shfl_down_sync(0xffffffffu, t1, 2);
          pd = t2 + __shfl_down_sync(0xffffffffu, pd, 4);
        }
        if (c[u] >= 0 && q == 0) st_f32_pol(gout + r0 + e0 + u, pd, pol.last);
      }
    }
    if (mine) st_v4_pol(out + (size_t)i * HID + 4 * q, acc, pol.last);
  }
}

// ------------------------------------------------------------------------------------------------ dense feature passes
// Tile pipeline of one dense warp: tiles of 16 consecutive level-order nodes, taken in blocks of kBlockTiles; the feature rows of
// a tile are gathered by the TMA engine (one bulk copy per node: its d floats) into the warp's two tile buffers.
struct TileIter {
  int b, k, nb, ntile, step;
  __device__ __forceinline__ bool valid() const { return b < nb; }
  __device__ __forceinline__ int tile() const { return b * kBlockTiles + k; }
  __device__ __forceinline__ void next() {
    ++k;
    if (k == kBlockTiles || b * kBlockTiles + k >= ntile) { b += step; k = 0; }
  }
};

// issue the loads of tile t into buffer `buf` (whole warp; one lane talks to the TMA engine).  The task's feature rows were copied
// once into level order with the shared-memory tile pitch (xlo), so a tile is ONE contiguous bulk copy that lands in the padded,
// bank-conflict-free layout; with_dp: also the tile's 16 x HID block of dP (contiguous as well).
template <int HID>
__device__ __forceinline__ void tile_issue(int t, int n, int xs, bool with_dp, int lane, const float* xlo, const float* dP,
                                           float* xt, float* pt, uint32_t bar, const L2Pol pol) {
  const int rows = min(16, n - t * 16);
  if (lane == 0) {
    mbar_expect_tx(bar, (uint32_t)(16 * xs * 4 + (with_dp ? rows * HID * 4 : 0)));
    tma_load_1d((uint32_t)__cvta_generic_to_shared(xt), xlo + (size_t)t * 16 * xs, (uint32_t)(16 * xs * 4), bar, pol.first);   // the feature rows stream
    if (with_dp) tma_load_1d((uint32_t)__cvta_generic_to_shared(pt), dP + (size_t)t * 16 * HID, (uint32_t)(rows * HID * 4), bar, pol.last);
  }
  __syncwarp();
}

// F0: P[j] = X[j] (sF (.) W1) for the tiles of this dense warp                                        (explain.py:707, models.py:70-71)
template <int HID>
__device__ __forceinline__ void dense_forward(int n, const GangSmem& S, int dwarp, int G, int grank, int lane,
                                              const float* xlo, const float* Whi, const float* Wlo,
                                              float* xt0, uint32_t bar0, uint32_t& phase, float* P, const L2Pol pol) {
  constexpr int NTL = (HID + 7) / 8;
  const int xs = S.xs, ldb = S.ldb, dp8 = S.dp8;
  const int ntile = (n + 15) / 16, nb = (ntile + kBlockTiles - 1) / kBlockTiles;
  const int g = lane >> 2, t4 = lane & 3;
  TileIter it{dwarp * G + grank, 0, nb, ntile, kDenseWarps * G};
  TileIter nx = it;
  int buf = 0;
  if (kTileBufs == 2 && nx.valid()) { tile_issue<HID>(nx.tile(), n, xs, false, lane, xlo, nullptr, xt0, nullptr, bar0, pol); nx.next(); }
  while (it.valid()) {
    if (kTileBufs == 1) { tile_issue<HID>(it.tile(), n, xs, false, lane, xlo, nullptr, xt0, nullptr, bar0, pol); }
    else if (nx.valid()) { tile_issue<HID>(nx.tile(), n, xs, false, lane, xlo, nullptr, xt0 + (buf ^ 1) * 16 * xs, nullptr, bar0 + (buf ^ 1) * 8, pol); nx.next(); }
    mbar_wait(bar0 + buf * 8, (phase >> buf) & 1u); phase ^= 1u << buf;
    const float* xr = xt0 + buf * 16 * xs;
    // 3xTF32 with two accumulators per n-tile (small terms lo*hi + hi*lo, big term hi*hi) and the MMAs of the n-tiles interleaved:
    // back-to-back MMAs into ONE accumulator serialise on the ~35-cycle MMA latency (the first version spent 3/4 of F0 there)
    float cs[NTL][4], cb[NTL][4];
#pragma unroll
    for (int nt = 0; nt < NTL; ++nt) { cs[nt][0] = cs[nt][1] = cs[nt][2] = cs[nt][3] = 0.f; cb[nt][0] = cb[nt][1] = cb[nt][2] = cb[nt][3] = 0.f; }
    for (int k0 = 0; k0 < dp8; k0 += 8) {
      uint32_t ahi[4], alo[4];
      tf32_split(xr[g * xs + k0 + t4], ahi[0], alo[0]);
      tf32_split(xr[(g + 8) * xs + k0 + t4], ahi[1], alo[1]);
      tf32_split(xr[g * xs + k0 + t4 + 4], ahi[2], alo[2]);
      tf32_split(xr[(g + 8) * xs + k0 + t4 + 4], ahi[3], alo[3]);
      uint32_t bh0[NTL], bh1[NTL], bl0[NTL], bl1[NTL];
#pragma unroll
      for (int nt = 0; nt < NTL; ++nt) {
        const int o0 = (k0 + t4) * ldb + nt * 8 + g, o1 = o0 + 4 * ldb;
        bh0[nt] = __float_as_uint(Whi[o0]); bh1[nt] = __float_as_uint(Whi[o1]); bl0[nt] = __float_as_uint(Wlo[o0]); bl1[nt] = __float_as_uint(Wlo[o1]);
      }
#pragma unroll
      for (int nt = 0; nt < NTL; ++nt) mma_tf32(cs[nt], alo, bh0[nt], bh1[nt]);
#pragma unroll
      for (int nt = 0; nt < NTL; ++nt) mma_tf32(cb[nt], ahi, bh0[nt], bh1[nt]);
#pragma unroll
      for (int nt = 0; nt < NTL; ++nt) mma_tf32(cs[nt], ahi, bl0[nt], bl1[nt]);
    }
    float c[NTL][4];
#pragma unroll
    for (int nt = 0; nt < NTL; ++nt) { c[nt][0] = cs[nt][0] + cb[nt][0]; c[nt][1] = cs[nt][1] + cb[nt][1]; c[nt][2] = cs[nt][2] + cb[nt][2]; c[nt][3] = cs[nt][3] + cb[nt][3]; }
    const int row0 = it.tile() * 16 + g;
#pragma unroll
    for (int nt = 0; nt < NTL; ++nt) {
      const int col = nt * 8 + 2 * t4;
      if (col < HID) {
        if (row0 < n) *reinterpret_cast<float2*>(P + (size_t)row0 * HID + col) = make_float2(c[nt][0], c[nt][1]);
        if (row0 + 8 < n) *reinterpret_cast<float2*>(P + (size_t)(row0 + 8) * HID + col) = make_float2(c[nt][2], c[nt][3]);
      }
    }
    __syncwarp();   // every lane is done with this buffer before the next issue overwrites it
    if (kTileBufs == 2) buf ^= 1;
    it.next();
  }
}

// B0 (dense half): per 128-node block b the partial  gFb[b][f] = sum_{j in block} X[j][f] (dP_j W1^T)[f]        (dL/dsF, explain.py:707)
// NF8 = feature n-tiles kept in registers (dp8 / 8 <= 16).
template <int HID, int NF8>
__device__ __forceinline__ void dense_backward(int n, int dp, const GangSmem& S, int dwarp, int G, int grank, int lane,
                                               const float* xlo, const float* Thi, const float* Tlo,
                                               const float* dP, float* xt0, float* pt0, uint32_t bar0, uint32_t& phase, float* gFb, const L2Pol pol) {
  constexpr int NTL = (HID + 7) / 8;
  const int xs = S.xs, ldt = S.ldt, dp8 = S.dp8;
  const int nf8 = dp8 / 8;
  const int ntile = (n + 15) / 16, nb = (ntile + kBlockTiles - 1) / kBlockTiles;
  const int g = lane >> 2, t4 = lane & 3;
  TileIter it{dwarp * G + grank, 0, nb, ntile, kDenseWarps * G};
  TileIter nx = it;
  int buf = 0;
  float ga[NF8][2];
#pragma unroll
  for (int nt = 0; nt < NF8; ++nt) { ga[nt][0] = 0.f; ga[nt][1] = 0.f; }
  if (kTileBufs == 2 && nx.valid()) { tile_issue<HID>(nx.tile(), n, xs, true, lane, xlo, dP, xt0, pt0, bar0, pol); nx.next(); }
  while (it.valid()) {
    if (kTileBufs == 1) { tile_issue<HID>(it.tile(), n, xs, true, lane, xlo, dP, xt0, pt0, bar0, pol); }
    else if (nx.valid()) {
      tile_issue<HID>(nx.tile(), n, xs, true, lane, xlo, dP, xt0 + (buf ^ 1) * 16 * xs, pt0 + (buf ^ 1) * 16 * HID, bar0 + (buf ^ 1) * 8, pol);
      nx.next();
    }
    mbar_wait(bar0 + buf * 8, (phase >> buf) & 1u); phase ^= 1u << buf;
    const float* xr = xt0 + buf * 16 * xs;
    const float* pr = pt0 + buf * 16 * HID;
    const int rows = min(16, n - it.tile() * 16);
    const bool v0 = g < rows, v1 = g + 8 < rows;
    // A = the tile's dP rows (16 x HID, K padded to 8 NTL with zeros); rows past the end of the graph are zeroed
    uint32_t ahi[NTL][4], alo[NTL][4];
#pragma unroll
    for (int ks = 0; ks < NTL; ++ks) {
      const int k0 = ks * 8 + t4, k1 = k0 + 4;
      tf32_split((v0 && k0 < HID) ? pr[g * HID + k0] : 0.f, ahi[ks][0], alo[ks][0]);
      tf32_split((v1 && k0 < HID) ? pr[(g + 8) * HID + k0] : 0.f, ahi[ks][1], alo[ks][1]);
      tf32_split((v0 && k1 < HID) ? pr[g * HID + k1] : 0.f, ahi[ks][2], alo[ks][2]);
      tf32_split((v1 && k1 < HID) ? pr[(g + 8) * HID + k1] : 0.f, ahi[ks][3], alo[ks][3]);
    }
    // feature n-tiles two at a time, two accumulators each (small / big 3xTF32 terms): four independent MMA chains in flight
#pragma unroll
    for (int np2 = 0; np2 < NF8; np2 += 2) {
      if (np2 < nf8) {
        float cs[2][4], cb[2][4];
#pragma unroll
        for (int j = 0; j < 2; ++j) { cs[j][0] = cs[j][1] = cs[j][2] = cs[j][3] = 0.f; cb[j][0] = cb[j][1] = cb[j][2] = cb[j][3] = 0.f; }
#pragma unroll
        for (int ks = 0; ks < NTL; ++ks) {
          uint32_t bh0[2], bh1[2], bl0[2], bl1[2];
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int nt = np2 + j < nf8 ? np2 + j : np2;   // (odd tile count: the second lane of the pair repeats the first, its result is dropped)
            const int o0 = (ks * 8 + t4) * ldt + nt * 8 + g, o1 = o0 + 4 * ldt;
            bh0[j] = __float_as_uint(Thi[o0]); bh1[j] = __float_as_uint(Thi[o1]); bl0[j] = __float_as_uint(Tlo[o0]); bl1[j] = __float_as_uint(Tlo[o1]);
          }
          mma_tf32(cs[0], alo[ks], bh0[0], bh1[0]); mma_tf32(cs[1], alo[ks], bh0[1], bh1[1]);
          mma_tf32(cb[0], ahi[ks], bh0[0], bh1[0]); mma_tf32(cb[1], ahi[ks], bh0[1], bh1[1]);
          mma_tf32(cs[0], ahi[ks], bl0[0], bl1[0]); mma_tf32(cs[1], ahi[ks], bl0[1], bl1[1]);
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int nt = np2 + j;
          if (nt < nf8) {
            const float c0 = cs[j][0] + cb[j][0], c1 = cs[j][1] + cb[j][1], c2 = cs[j][2] + cb[j][2], c3 = cs[j][3] + cb[j][3];
            const int col = nt * 8 + 2 * t4;
            const float2 x0 = v0 ? *reinterpret_cast<const float2*>(xr + g * xs + col) : make_float2(0.f, 0.f);
            const float2 x1 = v1 ? *reinterpret_cast<const float2*>(xr + (g + 8) * xs + col) : make_float2(0.f, 0.f);
            ga[nt][0] = fmaf(c0, x0.x, ga[nt][0]); ga[nt][1] = fmaf(c1, x0.y, ga[nt][1]);
            ga[nt][0] = fmaf(c2, x1.x, ga[nt][0]); ga[nt][1] = fmaf(c3, x1.y, ga[nt][1]);
          }
        }
      }
    }
    __syncwarp();
    const int b = it.b;
    if (kTileBufs == 2) buf ^= 1;
    it.next();
    if (!it.valid() || it.b != b) {   // end of the block: sum the eight row groups (fixed order) and write the block partial
#pragma unroll
      for (int nt = 0; nt < NF8; ++nt) {
        if (nt < nf8) {
#pragma unroll
          for (int o = 4; o <= 16; o <<= 1) {
            ga[nt][0] += __shfl_xor_sync(0xffffffffu, ga[nt][0], o);
            ga[nt][1] += __shfl_xor_sync(0xffffffffu, ga[nt][1], o);
          }
          const int col = nt * 8 + 2 * t4;
          if (g == 0) {
            if (col < dp) gFb[(size_t)b * dp + col] = ga[nt][0];
            if (col + 1 < dp) gFb[(size_t)b * dp + col + 1] = ga[nt][1];
          }
          ga[nt][0] = 0.f; ga[nt][1] = 0.f;
        }
      }
    }
  }
}

// first slot in [r0,r1) whose column is >= bound (columns are partitioned by level, so the predicate is monotone)
__device__ __forceinline__ int prefix_below_g(const int32_t* __restrict__ icol, int r0, int r1, int bound) {
  int lo = r0, hi = r1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(icol + mid) < bound) lo = mid + 1; else hi = mid;
  }
  return lo - r0;
}

struct GangArgs {
  ExplainArgs A;
  int G;                          // CTAs per gang
  unsigned long long* bars;       // [ngangs] barrier counters (zeroed before the launch)
  int32_t* mail;                  // [ngangs * 2] task mailbox + long-row counter
};

template <int HID, int EMB, bool kTrace>
__global__ void __launch_bounds__(kGangThreads, 1) explain_gang_kernel(const GangArgs GA) {
  extern __shared__ __align__(16) float sm[];
  __shared__ float s_tr[kTrace ? 8 : 1];
  __shared__ long long s_ph[11];   // debug: per-phase cycle sums of the first task + last stamp
  __shared__ int s_rowctr[5];      // next row of this CTA in each of the sparse passes of an epoch
  static_assert((HID == 20 || HID == 32) && EMB == HID, "hidden width 20 or 32 (others are zero-padded to 32 by gx_set_model)");
  constexpr int HS = HID, H4 = HID / 4, PD = 2 * HID + EMB, NT = kGangThreads;
  constexpr int nwarps = NT / 32;
  const ExplainArgs& A = GA.A;
  const int G = GA.G;
  const int gang = blockIdx.x / G, grank = blockIdx.x - gang * G;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const GxModelDev& m = A.m;
  const GxHparamsDev& hp = A.hp;
  const int d = m.d, C = m.C;
  const bool ieee = (hp.flags & GX_HP_IEEE_EDGE) != 0;
  const int dp = gx_round_up(d, 4);
  const GangSmem S = gang_smem(d, HID, EMB, C, nwarps);
  float* const W1s = sm + S.W1s; float* const Whi = sm + S.Whi; float* const Wlo = sm + S.Wlo; float* const Thi = sm + S.Thi; float* const Tlo = sm + S.Tlo;
  float* const W2s = sm + S.W2s; float* const W2t = sm + S.W2t; float* const W3s = sm + S.W3s; float* const bs = sm + S.bs;
  float* const sF = sm + S.sF; float* const Fm = sm + S.F; float* const mF = sm + S.mF; float* const vF = sm + S.vF;
  float* const zw = sm + S.zs + warp * 128;
  float* const dE = sm + S.dE; float* const dZ3 = sm + S.dZ3; float* const logit = sm + S.logit;
  float* const part = sm + S.part; float* const red = sm + S.red;
  const bool wp_smem = C * (PD + 1) <= GX_WP_SMEM_MAX;
  const float* const Wpp = wp_smem ? sm + S.Wp : m.Wp;
  const float* const bpp = wp_smem ? sm + S.Wp + C * PD : m.bp;
  float* const xt0 = sm + S.xt + (warp < kDenseWarps ? warp : 0) * kTileBufs * 16 * S.xs;
  float* const pt0 = sm + S.pt + (warp < kDenseWarps ? warp : 0) * kTileBufs * 16 * HID;
  const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(sm + S.bar) + (warp < kDenseWarps ? warp : 0) * 16;
  uint32_t tile_phase = 0;

  // model weights: once per CTA
  for (int idx = tid; idx < dp * HS; idx += NT) { const int f = idx / HS, c = idx - f * HS; W1s[idx] = f < d ? __ldg(m.W[0] + f * HID + c) : 0.f; }
  for (int idx = tid; idx < S.ntl * 8 * S.ldt; idx += NT) {   // W1^T as the (k = hidden, n = feature) operand, tf32 hi / lo
    const int c = idx / S.ldt, f = idx - c * S.ldt;
    const float w = (c < HID && f < d) ? __ldg(m.Wt[0] + c * d + f) : 0.f;
    uint32_t hi, lo;
    tf32_split(w, hi, lo);
    Thi[idx] = __uint_as_float(hi); Tlo[idx] = __uint_as_float(lo);
  }
  for (int idx = tid; idx < S.dp8 * S.ldb; idx += NT) { Whi[idx] = 0.f; Wlo[idx] = 0.f; }
  for (int idx = tid; idx < HID * HS; idx += NT) { W2s[idx] = __ldg(m.W[1] + idx); W2t[idx] = __ldg(m.Wt[1] + idx); }
  for (int idx = tid; idx < HID * EMB; idx += NT) W3s[idx] = __ldg(m.W[2] + idx);
  for (int idx = tid; idx < HID; idx += NT) { bs[idx] = __ldg(m.b[0] + idx); bs[HID + idx] = __ldg(m.b[1] + idx); }
  for (int idx = tid; idx < EMB; idx += NT) bs[2 * HID + idx] = __ldg(m.b[2] + idx);
  if (wp_smem) {
    float* const Wps = sm + S.Wp;
    for (int idx = tid; idx < C * PD; idx += NT) Wps[idx] = __ldg(m.Wp + idx);
    for (int idx = tid; idx < C; idx += NT) Wps[C * PD + idx] = __ldg(m.bp + idx);
  }
  for (int idx = tid; idx < kDenseWarps * kTileBufs * 16 * S.xs; idx += NT) sm[S.xt + idx] = 0.f;   // the pad columns [d, dp8) stay zero
  if (tid < kDenseWarps * 2) mbar_init((uint32_t)__cvta_generic_to_shared(sm + S.bar) + tid * 8, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();

  Grp G8;   // lane groups of 8 (phase S and B2)
  G8.GW = 8; G8.epi = 4; G8.lane = lane; G8.grp = lane >> 3; G8.q = lane & 7; G8.gbase = G8.grp * 8;
  constexpr int epi = 4;
  const int q = G8.q;
  float* const slab = A.gws + (int64_t)gang * A.gws_stride_words;
  float2* const MM0 = reinterpret_cast<float2*>(A.pws + (int64_t)gang * A.pws_stride_words);
  GangBar bar{GA.bars + gang, 0ull, G};
  const L2Pol pol = make_l2pol();
  int32_t* const mail = GA.mail + gang * 2;
  const int gtid = grank * NT + tid, gthreads = G * NT;
  const int gnw = nwarps * G;

  for (;;) {
    if (grank == 0 && tid == 0) { mail[0] = atomicAdd(A.counter, 1); mail[1] = 0; }
    bar.sync();
    const int qi = __ldcg(mail);
    if (qi >= A.ntasks) break;
    const int task_id = A.order[qi];
    const GxTask* __restrict__ Tp = A.plan.tasks + task_id;
    const int n = Tp->n, n1 = Tp->n1, n2 = Tp->n2, e_d = Tp->e_d, np = Tp->npairs_in;
    const int gt = hp.mode ? __ldg(A.g.pred_label + Tp->node) : Tp->gt_label;   // gradient baseline: predicted label (explain.py:130)
    const int64_t node_off = Tp->node_off, rp_off = Tp->rp_off, edge_off = Tp->edge_off, pair_off = Tp->pair_off;
    const GxStreamLayout L = gx_make_stream_layout(n, n1, n2, e_d, np, d, HID, nwarps);
    const int32_t* __restrict__ lo2gid = A.plan.lo2gid + node_off;
    const int32_t* __restrict__ irp = A.plan.irowptr + rp_off;
    const int32_t* __restrict__ icol = A.plan.icol + edge_off;
    const int32_t* __restrict__ pi = A.plan.pair_i + pair_off; const int32_t* __restrict__ pj = A.plan.pair_j + pair_off;
    const int32_t* __restrict__ ppij = A.plan.pair_pij + pair_off; const int32_t* __restrict__ ppji = A.plan.pair_pji + pair_off;
    const int32_t* __restrict__ poij = A.plan.pair_oij + pair_off; const int32_t* __restrict__ poji = A.plan.pair_oji + pair_off;
    float* const a = slab + L.a; float* const P = slab + L.P; float* const Yh1 = slab + L.Yh1; float* const q1 = slab + L.q1;
    float* const dY1 = slab + L.dY1; float* const Yh2 = slab + L.Yh2; float* const q2 = slab + L.q2; float* const dZ2 = slab + L.dZ2;
    float* const lapg = slab + L.lapg; float* const gFb = slab + L.gFb;
    int32_t* const cnt1 = reinterpret_cast<int32_t*>(slab + L.cnt1); int32_t* const cnt2 = reinterpret_cast<int32_t*>(slab + L.cnt2);
    int32_t* const longlist = reinterpret_cast<int32_t*>(slab + L.longlist);
    float* const dP = slab + L.dP; float* const gE = slab + L.gE;
    float* const xlo = slab + L.xlo;
    float2* const MM = MM0; float2* const mm = MM + np; float2* const vv = mm + np;   // (sigmoid(M) is recomputed, not stored)
    const float nn = (float)n * (float)n;
    const float ent_over_nn = hp.c_ent / nn;
    const float lap_over_nn = hp.c_lap / nn;
    const int nblk = ((n + 15) / 16 + kBlockTiles - 1) / kBlockTiles;

    // ------------------------------------------------------------------ per-task state (every CTA: the feature mask; gang: the rest)
    const bool resume = hp.init == GX_INIT_STATE && !hp.mode;   // optimiser state supplied by the caller (gx_explain_io)
    for (int f = tid; f < dp; f += NT) {
      sF[f] = hp.mode ? 1.0f : 0.5f; Fm[f] = 0.f; mF[f] = 0.f; vF[f] = 0.f;   // feat_mask = 0 (explain.py:633-643)
      if (resume && A.x.feat_state_in != nullptr && f < d) {
        const float* fs = A.x.feat_state_in + (int64_t)task_id * 3 * d;
        Fm[f] = fs[f]; mF[f] = fs[d + f]; vF[f] = fs[2 * d + f];
        sF[f] = sigmoid_f(fs[f]);
      }
      if (grank == 0 && hp.out_iter == 0 && !hp.mode && f < d) {
        if (A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = sF[f];
        if (A.x.feat_state_out != nullptr) {
          float* fo = A.x.feat_state_out + (int64_t)task_id * 3 * d;
          fo[f] = Fm[f]; fo[d + f] = mF[f]; fo[2 * d + f] = vF[f];
        }
      }
    }
    {
      const float m0_std = sqrtf(2.0f / (float)n);  // gain('relu') * sqrt(2/(n+n)) (explain.py:647-651)
      for (int p = gtid; p < np; p += gthreads) {
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
    // the task's feature rows in level order at the tile pitch (pad columns zero; the 16 rows past the end belong to the last tile)
    for (int j = warp * G + grank; j < n + 16; j += gnw) {   // a warp per row: coalesced read of the node's d floats, coalesced write
      const float* const row = j < n ? A.g.feat + (size_t)__ldg(lo2gid + j) * d : nullptr;
      for (int f = lane; f < S.xs; f += 32) xlo[(size_t)j * S.xs + f] = (row != nullptr && f < d) ? __ldg(row + f) : 0.f;
    }
    for (int e = gtid; e < e_d; e += gthreads) gE[e] = 0.f;   // slots outside the < n2 prefixes are never written and must read as 0
    for (int i = gtid; i < n; i += gthreads) {
      const int r0 = irp[i], r1 = irp[i + 1];
      cnt2[i] = prefix_below_g(icol, r0, r1, n2);
      if (i < n2) cnt1[i] = prefix_below_g(icol, r0, r1, n1);
      if (r1 - r0 > kLongEdges) longlist[atomicAdd(mail + 1, 1)] = i;   // (any order: a row's result does not depend on its position)
    }
    bar.sync();
    const int nlong = __ldcg(mail + 1);
    const int np1 = prefix_below_g(pi, 0, np, n1);   // pairs are sorted by i: the first np1 touch rows < n1 (layer-2/3 terms)

    // ------------------------------------------------------------------ epochs
    const bool timed = A.dbg != nullptr && qi == 0 && grank == 0;
#define GXG_MARK(k) if (timed && warp == 0) { const long long c_ = clock64(); if (lane == 0) { s_ph[k] += c_ - s_ph[10]; s_ph[10] = c_; } __syncwarp(); }
    if (timed && warp == 0) { const long long c_ = clock64(); if (lane == 0) { for (int k = 0; k < 10; ++k) s_ph[k] = 0; s_ph[10] = c_; } __syncwarp(); }
    for (int it = 1; it <= hp.iters; ++it) {
      // ---- F0: all nodes: P = (X . sigmoid(feat_mask)) W1 on the tensor cores               (explain.py:707, models.py:70-71)
      if (tid < 5) s_rowctr[tid] = 0;
      for (int idx = tid; idx < dp * HID; idx += NT) {   // fold the feature mask into W1, split into tf32 hi / lo
        const int f = idx / HID, c = idx - f * HID;
        uint32_t hi, lo;
        tf32_split(W1s[idx] * sF[f], hi, lo);
        Whi[f * S.ldb + c] = __uint_as_float(hi); Wlo[f * S.ldb + c] = __uint_as_float(lo);
      }
      __syncthreads();
      if (warp < kDenseWarps) {
        asm volatile("fence.proxy.async.global;" ::: "memory");   // xlo was written with ordinary stores, the TMA engine reads it
        dense_forward<HID>(n, S, warp, G, grank, lane, xlo, Whi, Wlo, xt0, bar0, tile_phase, P, pol);
      }
      bar.sync();
      GXG_MARK(0)
      // ---- F1: rows [0,n2): Y1 = A_m P + b1 ; row normalise                                   (models.py:70-78)
      row_pass<HID, false, false>(n2, n2, G, grank, warp, nwarps, lane, irp, icol, a, P, nullptr, nullptr, longlist, nlong, part, s_rowctr + 0, pol,
        [&](int i, int& r0, int& r1) { r0 = irp[i]; r1 = irp[i + 1]; },
        [&](int i, float4 z) {
          float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
          if (lane < H4) { const float4 b = ld4(bs + 4 * lane); y = make_float4(z.x + b.x, z.y + b.y, z.z + b.z, z.w + b.w); }
          const float ss = warp_sum(y.x * y.x + y.y * y.y + y.z * y.z + y.w * y.w);
          const float qn = fmaxf(sqrtf(ss), 1e-12f);  // F.normalize(p=2, dim=2), eps 1e-12
          if (lane < H4) st4(Yh1 + (size_t)i * HS + 4 * lane, make_float4(y.x / qn, y.y / qn, y.z / qn, y.w / qn));
          if (lane == 0) q1[i] = qn;
        });
      bar.sync();
      GXG_MARK(1)
      // ---- F2: rows [0,n1): Y2 = (A_m relu(Yh1)) W2 + b2 ; row normalise
      row_pass<HID, true, false>(n1, n1, G, grank, warp, nwarps, lane, irp, icol, a, Yh1, nullptr, nullptr, longlist, nlong, part, s_rowctr + 1, pol,
        [&](int i, int& r0, int& r1) { r0 = irp[i]; r1 = irp[i + 1]; },
        [&](int i, float4 z) {
          if (lane < H4) st4(zw + 4 * lane, z);
          __syncwarp();
          float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
          if (lane < H4) y = group_dense(zw, H4, W2s, HS, lane, ld4(bs + HID + 4 * lane));
          const float ss = warp_sum(y.x * y.x + y.y * y.y + y.z * y.z + y.w * y.w);
          const float qn = fmaxf(sqrtf(ss), 1e-12f);
          if (lane < H4) st4(Yh2 + (size_t)i * HS + 4 * lane, make_float4(y.x / qn, y.y / qn, y.z / qn, y.w / qn));
          if (lane == 0) q2[i] = qn;
          __syncwarp();
        });
      bar.sync();
      GXG_MARK(2)
      // ---- S: row r (= level-order id 0): layer 3, readout, softmax, -log p[gt], layer-3 backward -- every CTA for itself
      {
        // the explained node can be a hub (BASELINE configs[4]: thousands of neighbours): every warp of the CTA gathers a slice of its row,
        // warp 0 adds the partials in warp order and carries on alone
        const int r0 = irp[0], r1 = irp[1];
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        if (q < H4) acc = gather_row<int32_t, true, 4>(r0 + warp * epi + G8.grp, r1, epi * nwarps, icol, a, Yh2, HS, q);
        st4(zw + lane * 4, acc);
      }
      __syncthreads();
      if (warp == 0) {
        float z = 0.f;
        if (lane < HID)
          for (int w = 0; w < nwarps; ++w) {
            const float* const zo = sm + S.zs + w * 128;
            for (int g2 = 0; g2 < epi; ++g2) z += zo[(g2 * 8 + (lane >> 2)) * 4 + (lane & 3)];
          }
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
          if (lane == 0) { const float lg = logit[gt]; s_tr[4] = -((lg - mx) - logf(se)); s_tr[5] = expf(lg - mx) / se; }
          if (A.x.trace_pred != nullptr && grank == 0) {
            float* trp = A.x.trace_pred + ((int64_t)task_id * A.x.epochs + (it - 1)) * C;
            for (int c = lane; c < C; c += 32) trp[c] = expf(logit[c] - mx) / se;
          }
          float fs = 0.f;   // feat_size_loss = coeff * mean(sigmoid(feat_mask)) (explain.py:763-766)
          for (int f = lane; f < d; f += 32) fs += sF[f];
          fs = warp_sum(fs);
          if (lane == 0) s_tr[6] = hp.c_feat_size * fs / (float)d;
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
      GXG_MARK(3)
      // ---- B2: rows {r} U N(r): dYh2 = dEmb2 (row r) + a[r,j] dZ3 (j in N(r)), relu', normalise', dZ2 = dY2 W2^T
      {
        const int r0 = irp[0];
        const int items = 1 + irp[1] - r0;
        const int ntask = (items + epi - 1) / epi;
        // a handful of rows: every CTA computes all of them for itself (identical values, benign duplicate stores) -- saves a gang barrier
        for (int t = warp; t < ntask; t += nwarps) {
          const int item = t * epi + G8.grp;
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
            yh = ld4(Yh2 + (size_t)j * HS + 4 * q);
            const float4 g4 = ld4(dsrc + 4 * q);
            dy.x = yh.x > 0.f ? coef * g4.x : 0.f;   // relu backward: grad where input > 0
            dy.y = yh.y > 0.f ? coef * g4.y : 0.f;
            dy.z = yh.z > 0.f ? coef * g4.z : 0.f;
            dy.w = yh.w > 0.f ? coef * g4.w : 0.f;
          }
          const float sdot = group_sum(yh.x * dy.x + yh.y * dy.y + yh.z * dy.z + yh.w * dy.w, G8);
          if (act && q < H4) {
            const float qn = q2[j];
            st4(zw + lane * 4, make_float4((dy.x - yh.x * sdot) / qn, (dy.y - yh.y * sdot) / qn,
                                           (dy.z - yh.z * sdot) / qn, (dy.w - yh.w * sdot) / qn));
          }
          __syncwarp();
          if (act && q < H4)
            st4(dZ2 + (size_t)j * HS + 4 * q, group_dense(zw + G8.gbase * 4, H4, W2t, HS, q, make_float4(0.f, 0.f, 0.f, 0.f)));
          __syncwarp();
        }
      }
      __threadfence();
      __syncthreads();
      GXG_MARK(4)
      // ---- B1: rows [0,n2): dH1 = A_m^T dZ2 (only columns < n1 carry gradient), relu', normalise' -> dY1
      row_pass<HID, false, false>(n2, n2, G, grank, warp, nwarps, lane, irp, icol, a, dZ2, nullptr, nullptr, longlist, nlong, part, s_rowctr + 2, pol,
        [&](int i, int& r0, int& r1) { r0 = irp[i]; r1 = r0 + cnt1[i]; },
        [&](int i, float4 dh) {
          float4 yh = make_float4(0.f, 0.f, 0.f, 0.f), dy = yh;
          if (lane < H4) {
            yh = ld4(Yh1 + (size_t)i * HS + 4 * lane);
            if (i == 0) { const float4 e4 = ld4(dE + 4 * lane); dh.x += e4.x; dh.y += e4.y; dh.z += e4.z; dh.w += e4.w; }
            dy.x = yh.x > 0.f ? dh.x : 0.f; dy.y = yh.y > 0.f ? dh.y : 0.f;
            dy.z = yh.z > 0.f ? dh.z : 0.f; dy.w = yh.w > 0.f ? dh.w : 0.f;
          }
          const float sdot = warp_sum(yh.x * dy.x + yh.y * dy.y + yh.z * dy.z + yh.w * dy.w);
          if (lane < H4) {
            const float qn = q1[i];
            st4(dY1 + (size_t)i * HS + 4 * lane, make_float4((dy.x - yh.x * sdot) / qn, (dy.y - yh.y * sdot) / qn,
                                                             (dy.z - yh.z * sdot) / qn, (dy.w - yh.w * sdot) / qn));
          }
        });
      bar.sync();
      GXG_MARK(5)
      // ---- B0 (sparse half): all nodes: dP = A_m^T dY1 (columns < n2 of row j); layer-1 edge dots <dY1[col], P[row]> on the way
      //      rows < n2 (hub-heavy, long gradient-carrying prefixes): a warp per row; the outermost rows (a few edges each): a row per edge slot
      row_pass<HID, false, true>(n, n2, G, grank, warp, nwarps, lane, irp, icol, a, dY1, P, gE, longlist, nlong, part, s_rowctr + 3, pol,
        [&](int i, int& r0, int& r1) { r0 = irp[i]; r1 = r0 + cnt2[i]; },
        [&](int i, float4 z) { if (lane < H4) st4(dP + (size_t)i * HS + 4 * lane, z); });
      short_rows_pass<HID>(n2, n, G, grank, lane, irp, icol, a, dY1, P, gE, dP, nlong, s_rowctr + 4, pol,
        [&](int i, int& r0, int& r1) { r0 = irp[i]; r1 = r0 + cnt2[i]; });
      bar.sync();   // the tiles below read dP rows written by other warps / CTAs
      GXG_MARK(6)
      // ---- B0 (dense half): per 128-node block: sum_j X_j (.) (dP_j W1^T) on the tensor cores
      if (!hp.mode && warp < kDenseWarps) {
        asm volatile("fence.proxy.async.global;" ::: "memory");   // dP (and, first epoch, xlo) were written with ordinary stores, the TMA engine reads them
        dense_backward<HID, 16>(n, dp, S, warp, G, grank, lane, xlo, Thi, Tlo, dP, xt0, pt0, bar0, tile_phase, gFb, pol);
      }
      bar.sync();
      GXG_MARK(7)
      // ---- P: per undirected edge: dA_ij, dA_ji, symmetrise, regularisers, Adam, next mask value
      {
        const float2 tab = __ldg(hp.adam_tab + (it - 1));
        const float step = tab.x, bc2s = tab.y, bc2s_inv = 1.0f / tab.y;
        const bool last = (it == hp.out_iter);   // the mask built after this update is the one the reference returns
        // feature mask (every CTA keeps its own copy, all identical): dL/dF = sF(1-sF) (sum_j X_j (.) dX'_j + feat_size/d) ; Adam
        if (!hp.mode) {
          const int slices = NT / dp > 0 ? NT / dp : 1;
          for (int idx = tid; idx < slices * dp; idx += NT) {
            const int s = idx / dp, f = idx - s * dp;
            // (sixteen independent loads in flight, added in block order: the loop was a chain of ~200 dependent L2 round trips)
            float t = 0.f;
            int b = s;
            for (; b + 15 * slices < nblk; b += 16 * slices) {
              float v[16];
#pragma unroll
              for (int u = 0; u < 16; ++u) v[u] = __ldcg(gFb + (size_t)(b + u * slices) * dp + f);
#pragma unroll
              for (int u = 0; u < 16; ++u) t += v[u];
            }
            for (; b < nblk; b += slices) t += __ldcg(gFb + (size_t)b * dp + f);
            red[idx] = t;
          }
          __syncthreads();
          for (int f = tid; f < d; f += NT) {
            float gsum = 0.f;
            for (int s = 0; s < slices; ++s) gsum += red[s * dp + f];
            const float s = sF[f];
            const float g = s * (1.f - s) * (gsum + hp.c_feat_size / (float)d);
            float mf = mF[f], vf = vF[f], Fv = Fm[f];
            mf = mf + (g - mf) * hp.one_minus_b1;
            vf = vf * hp.b2 + hp.one_minus_b2 * g * g;
            Fv = Fv - step * (mf / (sqrtf(vf) / bc2s + hp.eps));
            mF[f] = mf; vF[f] = vf; Fm[f] = Fv;
            const float sn = sigmoid_f(Fv);
            sF[f] = sn;
            if (last && grank == 0) {
              if (A.out_feat != nullptr) A.out_feat[(int64_t)task_id * d + f] = sn;
              if (A.x.feat_state_out != nullptr) {
                float* fo = A.x.feat_state_out + (int64_t)task_id * 3 * d;
                fo[f] = Fv; fo[d + f] = mf; fo[2 * d + f] = vf;
              }
            }
          }
        }
        float trS = 0.f, trH = 0.f, trL = 0.f, trD = 0.f;   // trace: this thread's share of sum S, sum H(S), sum a (y_i-y_j)^2, sum 2a'
        // The layer-1 dots <dY1[i], P[j]> and <dY1[j], P[i]> were taken in B0 (gE); only the few pairs touching rows < n1
        // (listed first) carry layer-2/3 terms.
        if (hp.mode) {
          // gradient baseline (explain.py:125-133): mask_ij = sigmoid(|dL/dA_ij| + |dL/dA_ji|) on the edges
          for (int p = (warp * G + grank) * 32 + lane; p < np; p += gthreads) {
            float gij = __ldcg(gE + ppji[p]), gji = __ldcg(gE + ppij[p]);
            if (p < np1) {
              const int i = pi[p], j = pj[p];
              gij += dot_relu_v4(dZ2 + (size_t)i * HS, Yh1 + (size_t)j * HS, H4);
              if (j < n1) gji += dot_relu_v4(dZ2 + (size_t)j * HS, Yh1 + (size_t)i * HS, H4);
              if (i == 0) gij += dot_relu_v4(dZ3, Yh2 + (size_t)j * HS, H4);
            }
            const float an = sigmoid_f(fabsf(gij) + fabsf(gji));
            A.out_mask[edge_off + poij[p]] = an;
            A.out_mask[edge_off + poji[p]] = an;
          }
        } else
        for (int p = (warp * G + grank) * 32 + lane; p < np; p += gthreads) {
          // streams (pair indices, optimiser state) pass through the L2 with evict_first, the scattered a / gE accesses keep their lines
          const int sij = ld_i32_stream(ppij + p, pol.first), sji = ld_i32_stream(ppji + p, pol.first);
          float2 Mv = ld_v2_pol(MM + p, pol.first);
          // sigmoid(M) is recomputed instead of streamed (16 B less per pair and epoch): bit-identical to the value the previous
          // epoch's update produced (same function of the same M); the first epoch of a fresh run uses the IEEE form like the init
          const bool s_ieee = ieee || (it == 1 && !resume);
          const float2 Sv = make_float2(s_ieee ? sigmoid_f(Mv.x) : sigmoid_fast(Mv.x, false), s_ieee ? sigmoid_f(Mv.y) : sigmoid_fast(Mv.y, false));
          float2 m2 = ld_v2_pol(mm + p, pol.first), v2 = ld_v2_pol(vv + p, pol.first);
          float Gd = ld_f32_pol(lapg + p, pol.first) + ld_f32_pol(gE + sji, pol.last) + ld_f32_pol(gE + sij, pol.last);
          if (p < np1) {
            const int i = pi[p], j = pj[p];   // i < j, i < n1
            Gd += dot_relu_v4(dZ2 + (size_t)i * HS, Yh1 + (size_t)j * HS, H4);
            if (j < n1) Gd += dot_relu_v4(dZ2 + (size_t)j * HS, Yh1 + (size_t)i * HS, H4);
            if (i == 0) Gd += dot_relu_v4(dZ3, Yh2 + (size_t)j * HS, H4);
          }
          Gd *= 0.5f;  // sym_mask = (S + S^T)/2 (explain.py:671)
          if (kTrace) {
            trS += Sv.x + Sv.y; trH += bern_entropy(Sv.x) + bern_entropy(Sv.y);
            if (lap_over_nn > 0.f) trL += 0.5f * (Sv.x + Sv.y) * (lapg[p] / lap_over_nn);   // lapg = c_lap/n^2 (y_i-y_j)^2
          }
          // size: coeff*sum(S) ; entropy: mean over n^2 of H(S), dH/dM = -M S(1-S) (explain.py:755-770)
          const float gi = Sv.x * (1.f - Sv.x) * (Gd + hp.c_size - ent_over_nn * Mv.x);
          const float gj = Sv.y * (1.f - Sv.y) * (Gd + hp.c_size - ent_over_nn * Mv.y);
          m2.x = m2.x + (gi - m2.x) * hp.one_minus_b1;
          m2.y = m2.y + (gj - m2.y) * hp.one_minus_b1;
          v2.x = v2.x * hp.b2 + hp.one_minus_b2 * gi * gi;
          v2.y = v2.y * hp.b2 + hp.one_minus_b2 * gj * gj;
          Mv.x = Mv.x - adam_delta_fast(m2.x, v2.x, step, bc2s, bc2s_inv, hp.eps, ieee);
          Mv.y = Mv.y - adam_delta_fast(m2.y, v2.y, step, bc2s, bc2s_inv, hp.eps, ieee);
          const float2 Sn = make_float2(sigmoid_fast(Mv.x, ieee), sigmoid_fast(Mv.y, ieee));
          st_v2_pol(MM + p, Mv, pol.first); st_v2_pol(mm + p, m2, pol.first); st_v2_pol(vv + p, v2, pol.first);
          const float an = 0.5f * (Sn.x + Sn.y);
          if (kTrace) trD += 2.0f * an;
          st_f32_pol(a + sij, an, pol.last);
          st_f32_pol(a + sji, an, pol.last);
          if (last) {
            const int64_t oij = edge_off + poij[p], oji = edge_off + poji[p];
            A.out_mask[oij] = an;
            A.out_mask[oji] = an;
            if (A.x.mask_param_out != nullptr) { A.x.mask_param_out[oij] = Mv.x; A.x.mask_param_out[oji] = Mv.y; }
            if (A.x.adam_m_out != nullptr) { A.x.adam_m_out[oij] = m2.x; A.x.adam_m_out[oji] = m2.y; }
            if (A.x.adam_v_out != nullptr) { A.x.adam_v_out[oij] = v2.x; A.x.adam_v_out[oji] = v2.y; }
          }
        }
        if (kTrace) {   // per-warp partials of the gang, summed in warp order by (gang rank 0, thread 0) after the barrier
          trS = warp_sum(trS); trH = warp_sum(trH); trL = warp_sum(trL); trD = warp_sum(trD);
          float* tw = slab + L.trw + (size_t)(warp * G + grank) * 4;
          if (lane == 0) { tw[0] = trS; tw[1] = trH; tw[2] = trL; tw[3] = trD; }
        }
      }
      bar.sync();
      if (kTrace && tid == 0 && grank == 0) {   // raw terms of epoch it-1 over the INNER pairs (trace_finalize_kernel assembles the columns)
        float sS = 0.f, sH = 0.f, sLp = 0.f, sD = 0.f;
        const float* tw = slab + L.trw;
        for (int w = 0; w < gnw; ++w) { sS += __ldcg(tw + w * 4); sH += __ldcg(tw + w * 4 + 1); sLp += __ldcg(tw + w * 4 + 2); sD += __ldcg(tw + w * 4 + 3); }
        float* row = A.x.trace + ((int64_t)task_id * A.x.epochs + (it - 1)) * GX_TRACE_COLS;
        row[0] = sS; row[1] = s_tr[4]; row[2] = sH; row[3] = sLp; row[4] = sD; row[5] = s_tr[6]; row[6] = 0.f; row[7] = s_tr[5];
      }
      GXG_MARK(8)
    }
    if (timed && tid == 0) {
      float* o = A.dbg + (1 << 19);
      for (int k = 0; k < 9; ++k) o[k] = (float)s_ph[k];
      o[9] = (float)n; o[10] = (float)n1; o[11] = (float)n2; o[12] = (float)np; o[13] = (float)e_d; o[14] = (float)NT; o[15] = (float)G; o[16] = (float)nlong;
    }
  }
}

template <int HID, int EMB, bool kTrace>
cudaError_t launch_gang_t(const GxExplainLaunch& cfg, const ExplainArgs& args, cudaStream_t s) {
  auto kern = explain_gang_kernel<HID, EMB, kTrace>;
  const GangSmem S = gang_smem(args.m.d, HID, EMB, args.m.C, kGangThreads / 32);
  const int bytes = S.total * 4;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return e;
  GangArgs ga;
  ga.A = args;
  ga.G = cfg.gang;
  ga.bars = cfg.gang_bars;
  ga.mail = cfg.gang_mail;
  if (cfg.gang <= 1) {
    kern<<<cfg.grid, kGangThreads, bytes, s>>>(ga);
    return cudaGetLastError();
  }
  // gangs spin on each other: the whole grid must be resident at once -> cooperative launch (fails instead of deadlocking)
  void* params[] = {&ga};
  return cudaLaunchCooperativeKernel((const void*)kern, dim3((unsigned)cfg.grid), dim3(kGangThreads), params, (size_t)bytes, s);
}

}  // namespace

int gx_gang_smem_bytes(int d, int hid, int C) {
  const int h = hid <= 20 ? 20 : 32;
  return gang_smem(d, h, h, C, kGangThreads / 32).total * 4;
}

cudaError_t gx_launch_explain_gang(const GxExplainLaunch& cfg, const GxGraphDev& g, const GxModelDev& m,
                                   const GxHparamsDev& hp, const GxPlanArrays& plan, const float* m0,
                                   float* out_mask, float* out_feat, cudaStream_t s) {
  const ExplainArgs args = explain_args(cfg, g, m, hp, plan, m0, out_mask, out_feat);
  const bool trace = args.x.trace != nullptr;
  if (m.d > 128) return cudaErrorInvalidValue;   // wider inputs: explain_stream.cu
  if (m.hid == 20 && m.emb == 20) return trace ? launch_gang_t<20, 20, true>(cfg, args, s) : launch_gang_t<20, 20, false>(cfg, args, s);
  if (m.hid == 32 && m.emb == 32) return trace ? launch_gang_t<32, 32, true>(cfg, args, s) : launch_gang_t<32, 32, false>(cfg, args, s);
  return cudaErrorInvalidValue;
}
