// explain_common.cuh -- device primitives shared by the node-mode and graph-mode explainer kernels
// (lane-group row tasks, float4 gathers, dense products from a warp scratch row, Philox init, edge-phase math).
#pragma once
#include "gnnx_internal.cuh"

namespace {

#ifndef GX_SHORT_DEPTH
#define GX_SHORT_DEPTH 1   // edges in flight per lane group on short rows in the small launch classes (2 measured slower: 3.93 -> 4.33 ms, more registers/instructions)
#endif
constexpr int kLongRow = 32;  // rows with more edges than this are aggregated by a whole warp

__device__ __forceinline__ float warp_sum(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}
__device__ __forceinline__ float warp_max(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, o));
  return x;
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }
// Edge-phase arithmetic (2 sigmoids, 2 square roots, 4 divisions per undirected edge and epoch) uses the
// hardware approximations (ex2/rcp/rsqrt, <= 2 ulp): the phase is instruction-issue bound and IEEE
// division/sqrt sequences were a third of its instructions.  The row-normalised forward/backward keeps
// IEEE arithmetic.  Effect on parity: none measurable (tests/test_gpu_parity.py thresholds unchanged).
// `ieee` (GxHparamsDev::flags & GX_HP_IEEE_EDGE, test knob gx_debug_ieee_edge) selects the IEEE sequences instead, so the parity
// tests can measure what the approximations move (tools/parity_report.py).
__device__ __forceinline__ float sigmoid_fast(float x, bool ieee) {
  return ieee ? 1.0f / (1.0f + expf(-x)) : __fdividef(1.0f, 1.0f + __expf(-x));
}
__device__ __forceinline__ float adam_delta_fast(float m, float v, float step, float bc2s, float bc2s_inv, float eps, bool ieee) {
  return ieee ? step * (m / (sqrtf(v) / bc2s + eps)) : step * __fdividef(m, fmaf(__fsqrt_rn(v), bc2s_inv, eps));
}

// One optimiser step on a scalar parameter for the optimisers other than Adam (utils/train_utils.py:11-16 with torch's defaults):
// SGD(momentum 0.95): buf = 0.95 buf + g (= g at the first step, buf starts at 0); RMSprop(alpha 0.99, eps 1e-8); Adagrad(eps 1e-10).
// m = momentum buffer, v = squared-gradient accumulator, lr = this epoch's learning rate (scheduler applied on the host).
__device__ __forceinline__ void opt_step_other(int opt, float& P, float g, float& m, float& v, float lr) {
  if (opt == GX_OPT_SGD) { m = fmaf(0.95f, m, g); P -= lr * m; }
  else if (opt == GX_OPT_RMSPROP) { v = fmaf(0.99f, v, 0.01f * g * g); P -= lr * (g / (sqrtf(v) + 1e-8f)); }
  else { v = fmaf(g, g, v); P -= lr * (g / (sqrtf(v) + 1e-10f)); }
}

// Philox4x32-10 (Salmon et al. 2011), used only for GX_INIT_PHILOX.
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                              uint32_t k0, uint32_t k1, uint32_t* out) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
__device__ __forceinline__ float philox_normal(uint64_t seed, uint32_t node, uint32_t slot) {
  uint32_t r[4];
  philox4x32_10(slot, node, 0x67u, 0x6e78u, (uint32_t)seed, (uint32_t)(seed >> 32), r);
  const float u1 = ((float)(r[0] >> 8) + 0.5f) * (1.0f / 16777216.0f);
  const float u2 = ((float)(r[1] >> 8) + 0.5f) * (1.0f / 16777216.0f);
  return sqrtf(-2.0f * logf(u1)) * cosf(6.28318530717958647692f * u2);
}

template <typename IdxT> struct IdxTraits;
template <> struct IdxTraits<uint16_t> { static constexpr uint16_t kNone = 0xFFFFu; };
template <> struct IdxTraits<int32_t> { static constexpr int32_t kNone = -1; };

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, const float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 relu4(float4 v) {
  return make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
}
__device__ __forceinline__ void fma4(float4& acc, float s, const float4 v) {
  acc.x = fmaf(s, v.x, acc.x); acc.y = fmaf(s, v.y, acc.y); acc.z = fmaf(s, v.z, acc.z); acc.w = fmaf(s, v.w, acc.w);
}

// dot of two length-(4*n4) vectors / dot(a, relu(b)).  kMaxN4 > 0: n4 <= kMaxN4, unrolled to that bound with k < n4 as a predicate
template <int kMaxN4 = 0>
__device__ __forceinline__ float dot_v4(const float* a, const float* b, int n4) {
  float s = 0.f;
  const auto step = [&](int k) {
    const float4 x = ld4(a + 4 * k), y = ld4(b + 4 * k);
    s = fmaf(x.x, y.x, s); s = fmaf(x.y, y.y, s); s = fmaf(x.z, y.z, s); s = fmaf(x.w, y.w, s);
  };
  if constexpr (kMaxN4 > 0) {
#pragma unroll
    for (int k = 0; k < kMaxN4; ++k)
      if (k < n4) step(k);
  } else {
    for (int k = 0; k < n4; ++k) step(k);
  }
  return s;
}
__device__ __forceinline__ float dot_relu_v4(const float* a, const float* b, int n4) {
  float s = 0.f;
  for (int k = 0; k < n4; ++k) {
    const float4 x = ld4(a + 4 * k), y = relu4(ld4(b + 4 * k));
    s = fmaf(x.x, y.x, s); s = fmaf(x.y, y.y, s); s = fmaf(x.z, y.z, s); s = fmaf(x.w, y.w, s);
  }
  return s;
}

struct ExplainArgs {
  const int32_t* order;
  int32_t ntasks;
  int32_t* counter;
  float* gws;
  int64_t gws_stride_words;
  float* pws;
  int64_t pws_stride_words;
  GxGraphDev g;
  GxModelDev m;
  GxHparamsDev hp;
  GxPlanArrays plan;
  const float* m0;
  float* out_mask;
  float* out_feat;
  float* dbg;  // optional debug dump of the shared-memory arrays of task 0 after the backward of epoch 1
  GxExtra x;   // optional trace / optimiser-state buffers (gx_explain_io)
};

// ---------------------------------------------------------------------------------------------
// Thread-block clusters (explain_node.cu, cluster launch class): the CS CTAs of a cluster work on ONE task.  Every CTA keeps a
// full copy of the task's shared-memory state; a row (or pair) is computed by exactly one CTA, which stores the result into
// every CTA's copy (st.shared::cluster through the DSMEM window), so all reads stay local.  Phases are separated by the
// hardware cluster barrier (release/acquire makes the remote stores visible).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_id_x() { uint32_t r; asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
template <int CS> __device__ __forceinline__ void phase_sync() {
  if (CS == 1) __syncthreads(); else cluster_sync_all();
}
// Peer<CS>: byte offsets from this CTA's shared window to the other CTAs' windows (shared::cluster addresses)
template <int CS> struct Peer {
  uint32_t delta[CS > 1 ? CS - 1 : 1];
  __device__ __forceinline__ void init(const void* any_smem, uint32_t crank) {
    if (CS > 1) {
      const uint32_t a = (uint32_t)__cvta_generic_to_shared(any_smem);
#pragma unroll
      for (int k = 1; k < CS; ++k) {
        const uint32_t r = (crank + k) % CS;
        uint32_t ra;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(a), "r"(r));
        delta[k - 1] = ra - a;
      }
    }
  }
  // store to the local copy and to every peer's copy
  __device__ __forceinline__ void st4(float* p, const float4 v) const {
    *reinterpret_cast<float4*>(p) = v;
    if (CS > 1) {
      const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
#pragma unroll
      for (int k = 0; k < CS - 1; ++k)
        asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a + delta[k]), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
    }
  }
  __device__ __forceinline__ void st1(float* p, const float v) const {
    *p = v;
    if (CS > 1) {
      const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
#pragma unroll
      for (int k = 0; k < CS - 1; ++k) asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(a + delta[k]), "f"(v) : "memory");
    }
  }
  __device__ __forceinline__ void sti(int* p, const int v) const {
    *p = v;
    if (CS > 1) {
      const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
#pragma unroll
      for (int k = 0; k < CS - 1; ++k) asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(a + delta[k]), "r"(v) : "memory");
    }
  }
};

// entropy of a Bernoulli(s) in nats, as the reference writes it (explain.py:769): no guard at s -> 0/1, like torch
__device__ __forceinline__ float bern_entropy(float s) { return -s * logf(s) - (1.0f - s) * logf(1.0f - s); }

// ---------------------------------------------------------------------------------------------
// Lane-group primitives.  A warp = epi groups of GW lanes; lane = grp*GW + q.
// ---------------------------------------------------------------------------------------------
struct Grp {
  int GW, epi, grp, q, gbase, lane;
};

// sum of v over the GW lanes of the caller's group (every lane of the warp must call this).  kGW > 0: GW == kGW is known
// at compile time, so the shuffles are issued together; the adds keep their left-to-right order either way.
template <int kGW = 0>
__device__ __forceinline__ float group_sum(float v, const Grp& G) {
  float s = 0.f;
  if constexpr (kGW > 0) {
    float t[kGW];
#pragma unroll
    for (int k = 0; k < kGW; ++k) t[k] = __shfl_sync(0xffffffffu, v, min(G.gbase + k, 31));
#pragma unroll
    for (int k = 0; k < kGW; ++k) s += t[k];
  } else {
    for (int k = 0; k < G.GW; ++k) s += __shfl_sync(0xffffffffu, v, min(G.gbase + k, 31));
  }
  return s;
}

__device__ __forceinline__ void group_dense_step(const float* zrow, int f4, const float* W, int ldw, int q, float4& acc) {
  const float4 z = ld4(zrow + 4 * f4);
  const float* w = W + (4 * f4) * ldw + 4 * q;
  fma4(acc, z.x, ld4(w));
  fma4(acc, z.y, ld4(w + ldw));
  fma4(acc, z.z, ld4(w + 2 * ldw));
  fma4(acc, z.w, ld4(w + 3 * ldw));
}
// out4 = init + sum_{f < 4*F4} z[f] * W[f][4q .. 4q+3]   (z: F4 float4 in the group's scratch row).  kMaxF4 > 0: F4 <= kMaxF4,
// and the loop is unrolled to that bound with f4 < F4 as a predicate.
template <int kMaxF4 = 0>
__device__ __forceinline__ float4 group_dense(const float* zrow, int F4, const float* W, int ldw, int q, float4 acc) {
  if constexpr (kMaxF4 > 0) {
#pragma unroll
    for (int f4 = 0; f4 < kMaxF4; ++f4)
      if (f4 < F4) group_dense_step(zrow, f4, W, ldw, q, acc);
  } else {
    for (int f4 = 0; f4 < F4; ++f4) group_dense_step(zrow, f4, W, ldw, q, acc);
  }
  return acc;
}

// this lane's float4 slice of  sum_{e = r0, r0+estep, .. < r1} a[e] * f(src[col[e]]).  Four edges are kept in
// flight: the loop is a chain of two dependent shared-memory loads per edge, so without this a lane
// group waits ~2 LDS latencies per edge (hub rows: thousands of cycles).
template <typename IdxT, bool kRelu, int kDepth>
__device__ __forceinline__ float4 gather_row(int r0, int r1, int estep, const IdxT* icol, const float* a,
                                             const float* src, int src_stride, int q) {
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  int e = r0;
  if (kDepth >= 4)
#pragma unroll 1
  for (; e + 3 * estep < r1; e += 4 * estep) {
    const int c0 = icol[e], c1 = icol[e + estep], c2 = icol[e + 2 * estep], c3 = icol[e + 3 * estep];
    const float a0 = a[e], a1 = a[e + estep], a2 = a[e + 2 * estep], a3 = a[e + 3 * estep];
    float4 v0 = ld4(src + c0 * src_stride + 4 * q), v1 = ld4(src + c1 * src_stride + 4 * q);
    float4 v2 = ld4(src + c2 * src_stride + 4 * q), v3 = ld4(src + c3 * src_stride + 4 * q);
    if (kRelu) { v0 = relu4(v0); v1 = relu4(v1); v2 = relu4(v2); v3 = relu4(v3); }
    fma4(acc, a0, v0); fma4(acc, a1, v1); fma4(acc, a2, v2); fma4(acc, a3, v3);
  }
  if (kDepth >= 2)
#pragma unroll 1
  for (; e + estep < r1; e += 2 * estep) {
    const int c0 = icol[e], c1 = icol[e + estep];
    const float a0 = a[e], a1 = a[e + estep];
    float4 v0 = ld4(src + c0 * src_stride + 4 * q), v1 = ld4(src + c1 * src_stride + 4 * q);
    if (kRelu) { v0 = relu4(v0); v1 = relu4(v1); }
    fma4(acc, a0, v0); fma4(acc, a1, v1);
  }
#pragma unroll 1
  for (; e < r1; e += estep) {
    float4 v = ld4(src + (int)icol[e] * src_stride + 4 * q);
    if (kRelu) v = relu4(v);
    fma4(acc, a[e], v);
  }
  return acc;
}

// A "row task" of a phase: either one long row taken by the whole warp (edges split across the groups,
// partial sums reduced into group 0 through the scratch) or a chunk of epi short rows, one per group.
// Returns the row id (or -1) and this lane's float4 of the aggregate; W4 = source width in float4.
template <typename IdxT, bool kRelu, int kShortDepth>
__device__ __forceinline__ int row_task_gather(int t, int nlong, const IdxT* llist, int R, const Grp& G, int W4,
                                               const IdxT* irp, const IdxT* icol, const float* a,
                                               const float* src, int src_stride, const IdxT* cnt, float* zs,
                                               float4& z) {
  z = make_float4(0.f, 0.f, 0.f, 0.f);
  if (t < nlong) {
    const int i = llist[t];
    const int r0 = irp[i], r1 = cnt != nullptr ? r0 + (int)cnt[i] : (int)irp[i + 1];
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (G.grp < G.epi && G.q < W4)
      acc = gather_row<IdxT, kRelu, 4>(r0 + G.grp, r1, G.epi, icol, a, src, src_stride, G.q);
    st4(zs + G.lane * 4, acc);
    __syncwarp();
    if (G.grp == 0 && G.q < W4) {
      z = acc;
      for (int g2 = 1; g2 < G.epi; ++g2) {
        const float4 o = ld4(zs + (g2 * G.GW + G.q) * 4);
        z.x += o.x; z.y += o.y; z.z += o.z; z.w += o.w;
      }
    }
    __syncwarp();
    return G.grp == 0 ? i : -1;
  }
  const int i = (t - nlong) * G.epi + G.grp;
  if (G.grp >= G.epi || i >= R) return -1;
  const int r0 = irp[i], r1 = cnt != nullptr ? r0 + (int)cnt[i] : (int)irp[i + 1];
  if (nlong > 0 && r1 - r0 > kLongRow) return -1;  // taken by a whole warp above
  if (G.q < W4) z = gather_row<IdxT, kRelu, kShortDepth>(r0, r1, 1, icol, a, src, src_stride, G.q);
  return i;
}


// The kernel arguments every explainer launcher takes from its GxExplainLaunch and call: work queue, pair slabs, model,
// hyper-parameters, plan and masks.  Args is ExplainArgs or a graph-mode kernel's argument struct.
template <typename Args>
inline void fill_queue_args(Args& a, const GxExplainLaunch& cfg, const GxModelDev& m, const GxHparamsDev& hp, const GxPlanArrays& plan,
                            const float* m0, float* out_mask, float* out_feat) {
  a.order = cfg.order; a.ntasks = cfg.ntasks; a.counter = cfg.counter;
  a.pws = cfg.pws; a.pws_stride_words = cfg.pws_stride_words;
  a.m = m; a.hp = hp; a.plan = plan;
  a.m0 = m0; a.out_mask = out_mask; a.out_feat = out_feat;
}
inline ExplainArgs explain_args(const GxExplainLaunch& cfg, const GxGraphDev& g, const GxModelDev& m, const GxHparamsDev& hp,
                                const GxPlanArrays& plan, const float* m0, float* out_mask, float* out_feat) {
  ExplainArgs a;
  fill_queue_args(a, cfg, m, hp, plan, m0, out_mask, out_feat);
  a.g = g; a.gws = cfg.gws; a.gws_stride_words = cfg.gws_stride_words; a.dbg = cfg.dbg; a.x = cfg.x;
  return a;
}

}  // namespace
