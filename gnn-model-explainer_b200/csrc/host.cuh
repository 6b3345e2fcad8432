// host.cuh -- private to the host side of libgnnx.so (api.cu, node_mode.cu, graph_mode.cu): the handle and the device buffers it
// owns, the launch-class table and the helpers the entry points share.  No device code.
#pragma once
#include <stdio.h>

#include <algorithm>
#include <chrono>
#include <vector>

#include "gnnx_internal.cuh"

// A device allocation that grows on demand (with 25 % headroom) and is freed with its owner.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 4 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct LaunchClass {
  int cap_bytes;  // dynamic shared memory per CTA (0: the slab class, whose tasks keep their state in a global slab)
  int threads;
  int ctas_per_sm;
};
// Node-mode launch classes.  k CTAs per SM share 227 KB (1 KB per CTA is reserved by the system).  GNNX_CLASS_THREADS overrides the
// threads of a handle's copy.
constexpr LaunchClass kNodeClasses[] = {
    {13 * 1024, 128, 16}, {27 * 1024, 256, 8}, {55 * 1024, 256, 4},
    {112 * 1024, 512, 2}, {226 * 1024, 512, 1}, {0, 512, 1}, {226 * 1024, 512, 1}};
constexpr int kNumClasses = sizeof(kNodeClasses) / sizeof(kNodeClasses[0]);
constexpr int kStreamClass = 5;    // the slab class: explain_gang.cu / explain_stream.cu, or explain_var.cu for model variants
constexpr int kClusterClass = 6;   // explain_node.cu with a thread-block cluster per task: the most expensive shared-memory tasks
constexpr int kOneClass = 4, kTwoClass = 3;
// Cluster class (gx_debug_set_cluster / GNNX_CLUSTER_SIZE): off by default, so that a task's masks never depend on the batch it is in;
// 0 = latency mode, gx_plan_nodes moves the most expensive tasks of a batch that leaves SMs idle to clusters; 2 / 4 = every task above
// cluster_cost.  A full 700-node batch is throughput bound: splitting its tasks only adds barrier and DSMEM overhead,
// so the latency mode gives it none.

inline double now_us() { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

struct AdamKey { float lr, b1, b2, decay_rate; int32_t opt, sched, decay_step, restart, iters, start; };

struct gx_handle {
  int device = 0;
  int num_sms = 132;
  int64_t l2_bytes = (int64_t)50 << 20;
  cudaStream_t stream = nullptr;           // the caller's stream (gx_set_stream), not owned
  cudaStream_t side[kNumClasses] = {};     // one per launch class
  cudaEvent_t ev_fork = nullptr;
  cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;
  bool timed = false;
  float* dbg = nullptr;
  // knobs, read from the environment by gx_create; the gx_debug_* entry points set the test knobs later
  LaunchClass classes[kNumClasses];   // kNodeClasses with GNNX_CLASS_THREADS applied
  int exclusive_topk = 30;    // GNNX_EXCLUSIVE_TOPK: tasks of the 2-per-SM class that may get an SM of their own (syn1 sweep, DESIGN section 6)
  bool host_timing = false;   // GNNX_HOST_TIMING=1: stderr breakdown of the host side (tools/)
  bool ieee_edge = false;     // test knob (gx_debug_ieee_edge / GNNX_IEEE_EDGE): IEEE arithmetic in the edge phase
  bool node_generic = false;  // test / A-B knob (GNNX_NODE_GENERIC=1): explain_node.cu keeps the run-time lane-group shape for every input width
  int gang_override = 0;      // test knob (gx_debug_set_gang / GNNX_GANG): CTAs per task of explain_gang.cu, 0 = automatic, -1 = explain_stream.cu
  int cluster_size = 1;       // gx_debug_set_cluster / GNNX_CLUSTER_SIZE: 1 = never (default: results independent of the batch composition), 0 = automatic, 2 / 4 = forced
  int64_t cluster_cost = 0;   // GNNX_CLUSTER_COST
  int plan_cluster = 1;       // cluster size the current plan was classified with
  bool force_stream = false;  // test knob (gx_debug_force_stream / GNNX_FORCE_STREAM): every task goes to the streaming class
  cudaEvent_t ev_join[kNumClasses] = {}, ev_begin[kNumClasses] = {};
  bool class_used[kNumClasses] = {};   // launch classes of the last explain call (gx_last_class_ms)
  int64_t launches = 0;

  // graph
  bool has_graph = false;
  GxGraphDev g{};
  DevBuf g_rowptr, g_col, g_feat, g_label, g_pred;
  // model
  bool has_model = false;
  GxModelDev m{};
  GxHeadDev head{};   // the MLP prediction head of a gx_set_model_head model (k = 0: none); its block lies in m_buf
  DevBuf m_buf;
  // plan (node mode, or graph mode: one task per graph)
  bool has_plan = false;
  int count = 0, n_hops = 0;
  int64_t total_n = 0, total_e = 0;
  std::vector<GxTask> tasks;
  AdamKey adam_key{};
  bool adam_valid = false;
  bool tasks_fetched = true;   // false: idx_new of the host copy is stale (filled on the device by khop_fill, fetched by gx_plan_fetch)
  std::vector<int32_t> class_order[kNumClasses];   // tasks per launch class, most expensive first; d_order holds them class by class
  DevBuf d_nodes, d_tasks, d_nbrs, d_lo2gid, d_srp, d_scol, d_irp, d_icol, d_pairs, d_order, d_counters;
  DevBuf d_pws, d_gws, d_adam, d_m0, d_out, d_feat, d_dense_off, d_dense, d_rows;
  DevBuf d_trace, d_trpred, d_trouter, d_min, d_vin, d_fsin, d_Mout, d_mout, d_vout, d_fsout, d_m0dense, d_offedge;   // gx_explain_io staging (GX_HOST)
  DevBuf d_dn_thr, d_dn_cnt, d_dn_slots, d_dn_vals, d_us, d_gang, d_fwd;
  DevBuf d_uorder, d_mdense;   // unconstrained.cu: its work order (the plan's d_order stays for the constrained kernels), mask_dense staging
  GxComm* comm = nullptr;
  int32_t label_min = 0, label_max = 0, pred_min = 0, pred_max = 0;   // ranges of the uploaded labels (checked against num_classes at plan time)
  bool has_label = false;
  GxPlanArrays plan{};
  // graph-classification mode
  bool has_batch = false, has_gplan = false;
  GxGraphBatchDev gb{};
  DevBuf gb_rowptr, gb_col, gb_feat, gb_label;
  DevBuf d_dgraph;   // gx_densify_graphs: the value offsets and ids of its list
  DevBuf d_glabel;   // gx_grad_graphs: the loss label of every planned graph
  std::vector<int32_t> gb_h_rowptr, gb_h_label;
  // slot workspace
  DevBuf ws_buf;
  GxSlotWs ws{};

  gx_handle() = default;
  gx_handle(const gx_handle&) = delete;
  gx_handle& operator=(const gx_handle&) = delete;
  ~gx_handle() {   // the device buffers free themselves after this
    gx_comm_impl_destroy(comm);
    for (int i = 0; i < kNumClasses; ++i) {
      if (side[i]) cudaStreamDestroy(side[i]);
      if (ev_join[i]) cudaEventDestroy(ev_join[i]);
      if (ev_begin[i]) cudaEventDestroy(ev_begin[i]);
    }
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_t0) cudaEventDestroy(ev_t0);
    if (ev_t1) cudaEventDestroy(ev_t1);
  }
};

// Device views of a gx_explain_io: identity for GX_DEVICE, staged through handle-owned buffers for GX_HOST.
struct IoDev {
  const float* m0 = nullptr;
  float* out = nullptr;
  float* feat = nullptr;
  GxExtra x{};
};

// GX_HOST staging: stage_in uploads n elements (dev = nullptr when there are none), stage_out points dev at a device buffer for n
// elements (nullptr when host is), stage_back copies n elements back.  All on h->stream.
template <typename T> cudaError_t stage_in(gx_handle* h, DevBuf& b, const T* host, size_t n, const T** dev) {
  *dev = nullptr;
  if (!host || n == 0) return cudaSuccess;
  cudaError_t e = b.reserve(n * sizeof(T));
  if (e != cudaSuccess) return e;
  e = cudaMemcpyAsync(b.p, host, n * sizeof(T), cudaMemcpyHostToDevice, h->stream);
  *dev = b.as<T>();
  return e;
}
template <typename T> cudaError_t stage_out(DevBuf& b, T* host, size_t n, T** dev) {
  *dev = nullptr;
  if (!host) return cudaSuccess;
  cudaError_t e = b.reserve(std::max<size_t>(n, 1) * sizeof(T));
  *dev = b.as<T>();
  return e;
}
template <typename T> cudaError_t stage_back(gx_handle* h, T* host, const T* dev, size_t n) {
  if (!host || !dev || n == 0) return cudaSuccess;
  return cudaMemcpyAsync(host, dev, n * sizeof(T), cudaMemcpyDeviceToHost, h->stream);
}

// shared checks (api.cu); each reports through gx_set_error with `who` as the prefix and returns a GX_ status
int check_node_list(const gx_handle* h, const char* who, const int32_t* nodes, int32_t count, int32_t n_hops, int min_hops);
int check_explain_hparams(const char* who, const gx_hparams* hp, int mode, bool var, const gx_explain_io* io, bool init_first);
int check_optimiser(const char* who, const gx_hparams* hp);

// shared explain steps (api.cu)
int io_prepare(gx_handle* h, const char* who, const gx_hparams* hp, int mode, gx_memspace space, const gx_explain_io* io, int count,
               int64_t te, int d, int C, IoDev* D);
int io_finish(gx_handle* h, const gx_hparams* hp, gx_memspace space, const gx_explain_io* io, int count, int64_t te, int d, int C, const IoDev& D);
int upload_adam_table(gx_handle* h, const gx_hparams* hp, int iters, int start);
void fill_hparams(const gx_handle* h, const gx_hparams* hp, int mode, bool trace, GxHparamsDev* hd);
int upload_dense_offsets(gx_handle* h, int64_t* total);
int begin_timing(gx_handle* h);

// Pair-state slab of one CTA: 8 floats of optimiser state per inner pair (all pairs in graph mode) of the largest task it may take,
// and 2 words for the pair's four 16-bit indices (explain_node.cu).  Slabs are per CTA and the work queue is dynamic, so the stride
// never changes a result.
inline int64_t pair_slab_words(int max_pairs) { return ((int64_t)max_pairs * 10 + 3) / 4 * 4; }

// Places the pair slabs of n launches one after another in d_pws (launch c: slabs[c] slabs of cfg[c].pws_stride_words) and points
// cfg[c].pws at them.
int place_pair_slabs(gx_handle* h, GxExplainLaunch* cfg, const int* slabs, int n);

// A persistent launch whose CTAs each keep the task they work on in a global slab of slab_words(task) words, next to its pair slab:
// min(#ids, max_ctas) CTAs, fewer when the slabs would take more than 80 % of the free device memory.  Reserves the task slabs (d_gws)
// and fills cfg's grid, gws and slab strides; place_pair_slabs places the pair slabs.
template <typename SlabWords>
int size_slab_launch(gx_handle* h, const char* who, const std::vector<int32_t>& ids, SlabWords slab_words, int max_ctas,
                     GxExplainLaunch* cfg) {
  int64_t words = 4;
  int maxnp = 0;
  for (int32_t t : ids) {
    words = std::max<int64_t>(words, slab_words(h->tasks[t]));
    maxnp = std::max(maxnp, h->tasks[t].npairs_in);
  }
  cfg->gws_stride_words = (words + 3) / 4 * 4;
  cfg->pws_stride_words = pair_slab_words(maxnp);
  const int64_t per_cta = (cfg->gws_stride_words + cfg->pws_stride_words) * 4;
  size_t free_b = 0, total_b = 0;
  GX_CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
  const int64_t budget = (int64_t)(free_b + h->d_gws.cap + h->d_pws.cap) * 8 / 10;
  if (per_cta > budget) { gx_set_error("%s: a task needs %lld MB of device workspace, %lld MB are free", who, (long long)(per_cta >> 20), (long long)(budget >> 20)); return GX_ERR_CUDA; }
  cfg->grid = (int)std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>((int64_t)ids.size(), max_ctas), budget / per_cta));
  GX_CUDA_CHECK(h->d_gws.reserve((size_t)cfg->grid * cfg->gws_stride_words * 4));
  cfg->gws = h->d_gws.as<float>();
  return GX_OK;
}

// Words of task T's slab in explain_var.cu (graph mode has no Laplacian term, so no per-pair lapg)
inline int64_t var_slab_words(const gx_handle* h, int graph_mode, const GxTask& T) {
  return gx_make_var_layout(T.n, T.n2, T.e1, graph_mode ? 0 : T.npairs_in, h->m.d, h->m.L, gx_var_row_stride(h->m.hid, h->m.emb), h->m.att,
                            T.e_d, h->m.d >= GX_VAR_WIDE_MIN).total_words;
}

// One persistent launch of explain_var.cu over the whole plan (d_order, work-queue counter 0), each CTA with a task slab and a pair
// slab: at most 4 CTAs per SM in node mode, as many as are co-resident in graph mode.  Records ev_t0 before the launch.
int launch_var_batch(gx_handle* h, const char* who, int graph_mode, const GxHparamsDev& hd, const IoDev& D);

// Runs the n launch classes of an explain call.  h->class_order[c] holds class c's tasks and d_order holds them class by class; the
// caller fills cfg[c] with the class's grid, threads, shared memory, cluster / gang size and task slabs, and slabs[c] with its number
// of pair slabs.  Class c gets its slice of d_order, work-queue counter c and its own pair slabs, and runs on h->side[c], forked from
// h->stream; the highest index is launched first, so that the most expensive class starts at t = 0 and the cheaper ones fill in
// around it.  launch(c, cfg, stream) launches class c's kernel and returns its cudaError_t; overlap() queues the work that runs on
// h->stream beside the classes and returns a GX_ status.  The classes are joined back into h->stream.
template <typename Launch, typename Overlap>
int launch_classes(gx_handle* h, int n, GxExplainLaunch* cfg, const int* slabs, Launch launch, Overlap overlap) {
  int64_t order_off = 0;
  for (int c = 0; c < n; ++c) {
    cfg[c].ntasks = (int32_t)h->class_order[c].size();
    int maxnp = 0;
    for (int32_t t : h->class_order[c]) maxnp = std::max(maxnp, h->tasks[t].npairs_in);
    cfg[c].pws_stride_words = pair_slab_words(maxnp);
    cfg[c].order = h->d_order.as<int32_t>() + order_off;
    cfg[c].counter = h->d_counters.as<int32_t>() + c;
    order_off += cfg[c].ntasks;
  }
  int rc = place_pair_slabs(h, cfg, slabs, n);
  if (rc == GX_OK) rc = begin_timing(h);
  if (rc != GX_OK) return rc;
  GX_CUDA_CHECK(cudaEventRecord(h->ev_fork, h->stream));
  for (int c = n - 1; c >= 0; --c) {
    if (cfg[c].ntasks == 0) continue;
    GX_CUDA_CHECK(cudaStreamWaitEvent(h->side[c], h->ev_fork, 0));
    GX_CUDA_CHECK(cudaEventRecord(h->ev_begin[c], h->side[c]));
    GX_CUDA_CHECK(launch(c, cfg[c], h->side[c]));
    h->launches += 1;
    GX_CUDA_CHECK(cudaEventRecord(h->ev_join[c], h->side[c]));
    h->class_used[c] = true;
  }
  rc = overlap();
  if (rc != GX_OK) return rc;
  for (int c = 0; c < n; ++c)
    if (h->class_used[c]) GX_CUDA_CHECK(cudaStreamWaitEvent(h->stream, h->ev_join[c], 0));
  return GX_OK;
}
