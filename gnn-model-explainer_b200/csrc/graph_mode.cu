// graph_mode.cu -- graph classification on the host side of libgnnx.so: the padded graph batch, gx_plan_graphs (one task per graph,
// sorted into launch classes by shared-memory footprint), gx_explain_graphs, and the graph-list helpers of a sharded run: gx_count_graphs
// and gx_densify_graphs (its kernel: densify_graphs.cu); gx_grad_graphs, the gradient baseline, on the same launch classes.
#include <string.h>

#include <algorithm>
#include <vector>

#include "host.cuh"

namespace {

// Launch classes by footprint: a batch padded to 100 nodes mostly holds 20-40-node molecules; one launch sized for the largest graph
// left 3 CTAs per SM where 5-11 fit (~12 KB of every footprint are the weights).  Classes <= 18 / 27 / 36 / 44 / 80 / 226 KB ->
// 11 / 8 / 6 / 5 / 2 / 1 CTAs per SM (each launch requests its class's largest footprint), most expensive first inside a class.
constexpr int kGraphCap[] = {18 * 1024, 27 * 1024, 36 * 1024, 44 * 1024, 80 * 1024, 226 * 1024};
constexpr int kNumGraphClasses = sizeof(kGraphCap) / sizeof(kGraphCap[0]);
constexpr int kGraphThreads = 128;

// Rows of graph g that have an edge, and its directed edges: the task size of gx_plan_graphs and of gx_count_graphs.
void graph_counts(const gx_handle* h, int g, int* active, int32_t* edges) {
  const int nf = h->gb.max_nodes;
  const int32_t* rp = h->gb_h_rowptr.data() + (int64_t)g * nf;
  int na = 0;
  for (int i = 0; i < nf; ++i) na += rp[i + 1] > rp[i] ? 1 : 0;
  *active = na;
  *edges = rp[nf] - rp[0];
}

// The ids of a graph list: GX_OK when every id names a graph of the uploaded batch.
int check_graph_list(const gx_handle* h, const char* who, const int32_t* graph_ids, int32_t count) {
  for (int t = 0; t < count; ++t)
    if (graph_ids[t] < 0 || graph_ids[t] >= h->gb.num_graphs) { gx_set_error("%s: graph %d out of range", who, graph_ids[t]); return GX_ERR_INVALID; }
  return GX_OK;
}

}  // namespace

extern "C" {

int gx_set_graph_batch_csr(gx_handle* h, int32_t G, int32_t max_nodes, const int32_t* rowptr, const int32_t* col,
                           const float* feat, int32_t d, const int32_t* label) {
  if (!h || !rowptr || !col || !feat || !label) { gx_set_error("gx_set_graph_batch_csr: NULL argument"); return GX_ERR_INVALID; }
  if (G < 1 || max_nodes < 1 || max_nodes > 4096) { gx_set_error("gx_set_graph_batch_csr: num_graphs/max_nodes out of range (max_nodes <= 4096)"); return GX_ERR_INVALID; }
  const int64_t R = (int64_t)G * max_nodes;
  if (rowptr[0] != 0) { gx_set_error("gx_set_graph_batch_csr: rowptr[0] != 0"); return GX_ERR_INVALID; }
  for (int64_t r = 0; r < R; ++r) {
    if (rowptr[r + 1] < rowptr[r]) { gx_set_error("gx_set_graph_batch_csr: rowptr not monotone"); return GX_ERR_INVALID; }
    const int64_t g0 = r / max_nodes * max_nodes;
    const int32_t i = (int32_t)(r - g0);
    for (int64_t e = rowptr[r]; e < rowptr[r + 1]; ++e) {
      const int32_t j = col[e];
      if (j < 0 || j >= max_nodes) { gx_set_error("gx_set_graph_batch_csr: col out of range"); return GX_ERR_INVALID; }
      if (e > rowptr[r] && col[e] <= col[e - 1]) { gx_set_error("gx_set_graph_batch_csr: columns not strictly ascending"); return GX_ERR_INVALID; }
      if (j == i) { gx_set_error("gx_set_graph_batch_csr: self loops are not supported in graph mode"); return GX_ERR_UNSUPPORTED; }
      if (!std::binary_search(col + rowptr[g0 + j], col + rowptr[g0 + j + 1], i)) { gx_set_error("gx_set_graph_batch_csr: adjacency not symmetric"); return GX_ERR_UNSUPPORTED; }
    }
  }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  const int64_t nnz = rowptr[R];
  GX_CUDA_CHECK(h->gb_rowptr.reserve((size_t)(R + 1) * 4));
  GX_CUDA_CHECK(h->gb_col.reserve((size_t)std::max<int64_t>(nnz, 1) * 4));
  GX_CUDA_CHECK(h->gb_feat.reserve((size_t)R * d * 4));
  GX_CUDA_CHECK(h->gb_label.reserve((size_t)G * 4));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->gb_rowptr.p, rowptr, (size_t)(R + 1) * 4, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->gb_col.p, col, (size_t)nnz * 4, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->gb_feat.p, feat, (size_t)R * d * 4, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->gb_label.p, label, (size_t)G * 4, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  h->gb_h_rowptr.assign(rowptr, rowptr + R + 1);
  h->gb_h_label.assign(label, label + G);
  h->gb.num_graphs = G; h->gb.max_nodes = max_nodes; h->gb.d = d;
  h->gb.rowptr = h->gb_rowptr.as<int32_t>(); h->gb.col = h->gb_col.as<int32_t>();
  h->gb.feat = h->gb_feat.as<float>(); h->gb.label = h->gb_label.as<int32_t>();
  h->has_batch = true; h->has_gplan = false;
  return GX_OK;
}

int gx_plan_graphs(gx_handle* h, const int32_t* graph_ids, int32_t count, int64_t* edge_off, int64_t* total_edges) {
  if (!h || !graph_ids) { gx_set_error("gx_plan_graphs: NULL argument"); return GX_ERR_INVALID; }
  if (!h->has_batch || !h->has_model) { gx_set_error("gx_plan_graphs: call gx_set_model and gx_set_graph_batch_csr first"); return GX_ERR_INVALID; }
  if (h->gb.d != h->m.d) { gx_set_error("gx_plan_graphs: feat_dim %d != model input_dim %d", h->gb.d, h->m.d); return GX_ERR_INVALID; }
  if (count <= 0) { gx_set_error("gx_plan_graphs: count <= 0"); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  h->has_gplan = false; h->has_plan = false;
  const int nf = h->gb.max_nodes;
  h->tasks.assign(count, GxTask());
  int64_t tn = 0, te = 0, tp = 0;
  for (int t = 0; t < count; ++t) {
    const int g = graph_ids[t];
    if (g < 0 || g >= h->gb.num_graphs) { gx_set_error("gx_plan_graphs: graph %d out of range", g); return GX_ERR_INVALID; }
    GxTask& T = h->tasks[t];
    memset(&T, 0, sizeof(T));
    int na = 0;
    graph_counts(h, g, &na, &T.e_d);
    T.node = g; T.n = na; T.n1 = na; T.n2 = na;
    T.e1 = T.e_d; T.npairs = T.e_d / 2; T.npairs_in = T.npairs;
    T.gt_label = h->gb_h_label[g]; T.n_norm = nf; T.flags = na < nf ? 1 : 0;
    T.node_off = tn; T.rp_off = tn + t; T.edge_off = te; T.pair_off = tp;
    if (!h->m.variant) {   // the tuned kernel (explain_graph.cu) keeps a graph in shared memory with 16-bit indices
      if (na >= 65535 || T.e_d >= 65535) { gx_set_error("gx_plan_graphs: graph %d too large for the shared-memory kernel", g); return GX_ERR_UNSUPPORTED; }
      const GxLayoutG L = gx_make_layout_graph(na, T.e_d, T.npairs, h->m.d, h->m.hid, h->m.emb, h->m.C, kGraphThreads / 32);
      T.smem_bytes = L.total_words * 4;
      if (T.smem_bytes > kGraphCap[kNumGraphClasses - 1]) { gx_set_error("gx_plan_graphs: graph %d needs %d bytes of shared memory", g, T.smem_bytes); return GX_ERR_UNSUPPORTED; }
    }   // model variants: explain_var.cu keeps a graph in a global slab (smem_bytes 0: one launch class), bounded by max_nodes <= 4096
    tn += na; te += T.e_d; tp += T.npairs;
  }
  for (auto& v : h->class_order) v.clear();
  for (int t = 0; t < count; ++t) {
    int c = 0;
    while (c < kNumGraphClasses - 1 && h->tasks[t].smem_bytes > kGraphCap[c]) ++c;
    h->class_order[c].push_back(t);
  }
  std::vector<int32_t> order;
  order.reserve(count);
  for (int c = 0; c < kNumGraphClasses; ++c) {
    auto& v = h->class_order[c];
    std::stable_sort(v.begin(), v.end(), [&](int32_t x, int32_t y) { return h->tasks[x].e_d + 4 * h->tasks[x].n > h->tasks[y].e_d + 4 * h->tasks[y].n; });
    order.insert(order.end(), v.begin(), v.end());
  }
  GX_CUDA_CHECK(h->d_tasks.reserve((size_t)count * sizeof(GxTask)));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->d_tasks.p, h->tasks.data(), (size_t)count * sizeof(GxTask), cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(h->d_order.reserve((size_t)count * 4));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->d_order.p, order.data(), (size_t)count * 4, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(h->d_counters.reserve(kNumClasses * 4));
  GX_CUDA_CHECK(h->d_lo2gid.reserve((size_t)std::max<int64_t>(tn, 1) * 4));
  GX_CUDA_CHECK(h->d_irp.reserve((size_t)(tn + count) * 4));
  GX_CUDA_CHECK(h->d_icol.reserve((size_t)std::max<int64_t>(te, 1) * 4));
  GX_CUDA_CHECK(h->d_pairs.reserve((size_t)std::max<int64_t>(tp, 1) * 4 * 6));
  h->plan = GxPlanArrays();
  h->plan.tasks = h->d_tasks.as<GxTask>();
  h->plan.lo2gid = h->d_lo2gid.as<int32_t>();
  h->plan.irowptr = h->d_irp.as<int32_t>();
  h->plan.icol = h->d_icol.as<int32_t>();
  int32_t* pb = h->d_pairs.as<int32_t>();
  h->plan.pair_i = pb; h->plan.pair_j = pb + tp; h->plan.pair_pij = pb + 2 * tp;
  h->plan.pair_pji = pb + 3 * tp; h->plan.pair_oij = pb + 4 * tp; h->plan.pair_oji = pb + 5 * tp;
  GX_CUDA_CHECK(gx_launch_graph_plan(h->gb, count, h->plan, h->stream));
  h->launches += 1;
  GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  h->count = count; h->total_e = te;
  h->has_gplan = true;
  if (edge_off) { for (int t = 0; t < count; ++t) edge_off[t] = h->tasks[t].edge_off; edge_off[count] = te; }
  if (total_edges) *total_edges = te;
  return GX_OK;
}

}  // extern "C"

// mode 0: Explainer.explain's optimisation loop; mode 1: its model="grad" baseline (one forward/backward, explain.py:125-133,717-738)
// at grad_label (host, one label per planned graph in [-1, C)).
static int explain_graphs_impl(gx_handle* h, const gx_hparams* hp, int mode, gx_memspace space, const gx_explain_io* io,
                               const int32_t* grad_label = nullptr) {
  const char* who = mode ? "gx_grad_graphs" : "gx_explain_graphs";
  if (!h || !hp) { gx_set_error("%s: NULL argument", who); return GX_ERR_INVALID; }
  if (!h->has_gplan) { gx_set_error("%s: no plan (call gx_plan_graphs)", who); return GX_ERR_INVALID; }
  if (h->gb.d != h->m.d) { gx_set_error("%s: feat_dim %d != model input_dim %d", who, h->gb.d, h->m.d); return GX_ERR_INVALID; }
  const bool var = h->m.variant || hp->opt != GX_OPT_ADAM;   // the whole batch through explain_var.cu
  int rc = check_explain_hparams(who, hp, mode, var, io, true);
  if (rc != GX_OK) return rc;
  const int count = h->count;
  if (mode == 1) {
    if (!grad_label) { gx_set_error("%s: pred_label is NULL", who); return GX_ERR_INVALID; }
    for (int t = 0; t < count; ++t)
      if (grad_label[t] < -1 || grad_label[t] >= h->m.C) {
        gx_set_error("%s: pred_label[%d] = %d outside [-1,%d)", who, t, grad_label[t], h->m.C);
        return GX_ERR_INVALID;
      }
  }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  const int64_t te = h->total_e;
  IoDev D;
  rc = io_prepare(h, who, hp, mode, space, io, count, te, h->m.d, h->m.C, &D);
  if (rc != GX_OK) return rc;
  D.x.tr_outer = nullptr;   // graph mode has no outer pairs
  const int32_t* d_label = nullptr;
  if (mode == 1) {
    GX_CUDA_CHECK(h->d_glabel.reserve((size_t)count * 4));
    // pageable source: the copy is staged before the call returns
    GX_CUDA_CHECK(cudaMemcpyAsync(h->d_glabel.p, grad_label, (size_t)count * 4, cudaMemcpyHostToDevice, h->stream));
    d_label = h->d_glabel.as<int32_t>();
  }
  GxHparamsDev hd;
  fill_hparams(h, hp, mode, D.x.trace != nullptr, &hd);
  hd.c_lap = 0.f;           // lap_loss = 0 in graph mode (explain.py:787-788)
  rc = upload_adam_table(h, hp, hd.iters, mode == 0 ? hp->start_step : 0);
  if (rc != GX_OK) return rc;
  hd.adam_tab = h->d_adam.as<float2>();
  GX_CUDA_CHECK(cudaMemsetAsync(h->d_counters.p, 0, kNumClasses * 4, h->stream));
  if (var) {
    rc = launch_var_batch(h, who, 1, hd, D);
    if (rc != GX_OK) return rc;
  } else {
    // one persistent launch per footprint class, each requesting its largest footprint, as many CTAs per SM as fit
    GxExplainLaunch cfg[kNumGraphClasses] = {};
    int slabs[kNumGraphClasses];
    for (int c = 0; c < kNumGraphClasses; ++c) {
      int need = 1024;
      for (int32_t t : h->class_order[c]) need = std::max(need, h->tasks[t].smem_bytes);
      const int per_sm = std::max(1, std::min(16, (227 * 1024) / (need + 1024)));
      cfg[c].smem_bytes = need;
      cfg[c].threads = kGraphThreads;
      cfg[c].grid = std::min<int>((int)h->class_order[c].size(), h->num_sms * per_sm);
      cfg[c].x = D.x;
      slabs[c] = cfg[c].grid;
    }
    auto launch = [&](int, const GxExplainLaunch& k, cudaStream_t s) {
      return gx_launch_explain_graphs(k, h->gb, h->m, hd, h->plan, D.m0, D.out, D.feat, d_label, s);
    };
    rc = launch_classes(h, kNumGraphClasses, cfg, slabs, launch, [] { return (int)GX_OK; });
    if (rc != GX_OK) return rc;
  }
  if (D.x.trace) {
    GX_CUDA_CHECK(gx_launch_trace_finalize(hd, h->plan, count, D.x, h->stream));
    h->launches += 1;
  }
  GX_CUDA_CHECK(cudaEventRecord(h->ev_t1, h->stream));
  h->timed = true;
  return io_finish(h, hp, space, io, count, te, h->m.d, h->m.C, D);
}

extern "C" {

int gx_explain_graphs(gx_handle* h, const gx_hparams* hp, gx_memspace space, const float* m0_edges,
                      float* edge_mask, float* feat_mask) {
  gx_explain_io io;
  memset(&io, 0, sizeof(io));
  io.m0_edges = m0_edges; io.edge_mask = edge_mask; io.feat_mask = feat_mask;
  return explain_graphs_impl(h, hp, 0, space, &io);
}

int gx_explain_graphs_ex(gx_handle* h, const gx_hparams* hp, gx_memspace space, const gx_explain_io* io) {
  return explain_graphs_impl(h, hp, 0, space, io);
}

int gx_grad_graphs(gx_handle* h, gx_memspace space, const int32_t* pred_label, float* edge_mask) {
  gx_hparams hp;
  gx_default_hparams(&hp);
  gx_explain_io io;
  memset(&io, 0, sizeof(io));
  io.edge_mask = edge_mask;
  return explain_graphs_impl(h, &hp, 1, space, &io, pred_label);
}

int gx_count_graphs(gx_handle* h, const int32_t* graph_ids, int32_t count, int32_t* n_out, int32_t* e_out) {
  if (!h || (count > 0 && (!graph_ids || !n_out || !e_out))) { gx_set_error("gx_count_graphs: NULL argument"); return GX_ERR_INVALID; }
  if (!h->has_batch) { gx_set_error("gx_count_graphs: call gx_set_graph_batch_csr first"); return GX_ERR_INVALID; }
  if (count < 0) { gx_set_error("gx_count_graphs: count < 0"); return GX_ERR_INVALID; }
  const int rc = check_graph_list(h, "gx_count_graphs", graph_ids, count);
  if (rc != GX_OK) return rc;
  for (int t = 0; t < count; ++t) graph_counts(h, graph_ids[t], &n_out[t], &e_out[t]);
  return GX_OK;
}

int gx_densify_graphs(gx_handle* h, gx_memspace space, const int32_t* graph_ids, int32_t count, const float* values, double* out) {
  if (!h || (count > 0 && (!graph_ids || !out))) { gx_set_error("gx_densify_graphs: NULL argument"); return GX_ERR_INVALID; }
  if (!h->has_batch) { gx_set_error("gx_densify_graphs: call gx_set_graph_batch_csr first"); return GX_ERR_INVALID; }
  if (count < 0) { gx_set_error("gx_densify_graphs: count < 0"); return GX_ERR_INVALID; }
  int rc = check_graph_list(h, "gx_densify_graphs", graph_ids, count);
  if (rc != GX_OK || count == 0) return rc;
  std::vector<int64_t> val_off(count + 1, 0);
  for (int t = 0; t < count; ++t) {
    int na;
    int32_t ed;
    graph_counts(h, graph_ids[t], &na, &ed);
    val_off[t + 1] = val_off[t] + ed;
  }
  const int64_t total = val_off[count];
  if (total > 0 && !values) { gx_set_error("gx_densify_graphs: NULL values"); return GX_ERR_INVALID; }
  const size_t dense = (size_t)count * h->gb.max_nodes * h->gb.max_nodes;
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  const size_t b64 = (size_t)count * 8;
  GX_CUDA_CHECK(h->d_dgraph.reserve(b64 + (size_t)count * 4));
  char* b = h->d_dgraph.as<char>();
  GX_CUDA_CHECK(cudaMemcpyAsync(b, val_off.data(), b64, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(cudaMemcpyAsync(b + b64, graph_ids, (size_t)count * 4, cudaMemcpyHostToDevice, h->stream));
  const float* v = values;
  double* o = out;
  if (space == GX_HOST) {
    GX_CUDA_CHECK(stage_in(h, h->d_out, values, (size_t)total, &v));
    GX_CUDA_CHECK(stage_out(h->d_dense, out, dense, &o));
  }
  GX_CUDA_CHECK(gx_launch_densify_graphs(h->gb, (const int32_t*)(b + b64), count, (const int64_t*)b, v, o, h->stream));
  h->launches += 1;
  if (space == GX_HOST) {
    GX_CUDA_CHECK(stage_back(h, out, (const double*)o, dense));
    GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  }
  return GX_OK;
}

}  // extern "C"
