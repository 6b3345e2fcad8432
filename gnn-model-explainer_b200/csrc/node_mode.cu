// node_mode.cu -- node classification on the host side of libgnnx.so: k-hop extraction (gx_plan_nodes and the counting entry points),
// the launch-class policy that sorts a plan's tasks into classes, and gx_explain_nodes.  Every algorithmic step is a kernel in
// khop.cu / explain_*.cu.
#include <string.h>

#include <algorithm>
#include <vector>

#include "host.cuh"

namespace {

int ensure_slot_ws(gx_handle* h) {
  const int64_t N = h->g.N;
  const int W = (int)((N + 31) / 32);
  int slots = h->num_sms * 8;
  const size_t per_slot = (size_t)W * 4 + (size_t)(W + 1) * 4 + (size_t)N + (size_t)(N + 1) * 4 * 2 + (size_t)N * 4 * 2 + 64;
  const size_t budget = (size_t)4 << 30;
  while (slots > 1 && per_slot * slots > budget) slots /= 2;
  if (h->ws.slots == slots && h->ws.W == W && h->ws_buf.p) return GX_OK;
  // carve (each array 16B aligned)
  auto al = [](size_t x) { return (x + 15) / 16 * 16; };
  size_t o = 0;
  const size_t o_bm = o; o += al((size_t)slots * W * 4);
  const size_t o_wp = o; o += al((size_t)slots * (W + 1) * 4);
  const size_t o_q = o; o += al((size_t)slots * (N + 1) * 4);
  const size_t o_loc = o; o += al((size_t)slots * N * 4);
  const size_t o_cof = o; o += al((size_t)slots * N * 4);
  const size_t o_pb = o; o += al((size_t)slots * (N + 1) * 4);
  const size_t o_dist = o; o += al((size_t)slots * N);
  GX_CUDA_CHECK(h->ws_buf.reserve(o));
  char* b = h->ws_buf.as<char>();
  h->ws.bm = (uint32_t*)(b + o_bm);
  h->ws.wpref = (int32_t*)(b + o_wp);
  h->ws.q = (int32_t*)(b + o_q);
  h->ws.loc = (int32_t*)(b + o_loc);
  h->ws.cof = (int32_t*)(b + o_cof);
  h->ws.pbase = (int32_t*)(b + o_pb);
  h->ws.dist = (uint8_t*)(b + o_dist);
  h->ws.W = W;
  h->ws.slots = slots;
  GX_CUDA_CHECK(cudaMemsetAsync(h->ws.bm, 0, (size_t)slots * W * 4, h->stream));
  return GX_OK;
}

int task_smem_class(const gx_handle* h, const GxTask& T, int* bytes_out) {
  // shared-memory classes always use 16-bit indices: a task with n or e1 >= 65535 cannot fit 227 KB anyway
  const GxModelDev& m = h->m;
  const bool small_idx = !h->force_stream && T.n < 65535 && T.e1 < 65535;
  for (int c = 0; small_idx && c < kStreamClass; ++c) {
    const int nwarps = h->classes[c].threads / 32;
    const GxLayout L = gx_make_layout(T.n, T.n1, T.n2, T.e1, m.d, m.hid, m.emb, m.C, nwarps, 2);
    const int64_t bytes = (int64_t)L.total_words * 4;
    if (bytes <= h->classes[c].cap_bytes) {
      *bytes_out = (int)bytes;
      return c;
    }
  }
  *bytes_out = 0;  // streaming class (explain_stream.cu): state in a global slab, sized by gx_make_stream_layout
  return kStreamClass;
}

// the kernel a node-mode launch class runs in one explain call
enum class NodeKernel { smem, cluster, gang, stream1, variant };

}  // namespace

extern "C" {

int gx_plan_class_counts(gx_handle* h, int32_t counts[7], int32_t smem_bytes[7], int32_t* cluster_size) {
  if (!h || !counts || !h->has_plan) { gx_set_error("gx_plan_class_counts: no plan (call gx_plan_nodes)"); return GX_ERR_INVALID; }
  for (int c = 0; c < kNumClasses; ++c) {
    counts[c] = (int32_t)h->class_order[c].size();
    if (smem_bytes) {
      smem_bytes[c] = 0;
      for (int32_t t : h->class_order[c]) smem_bytes[c] = std::max(smem_bytes[c], h->tasks[t].smem_bytes);
    }
  }
  if (cluster_size) *cluster_size = h->plan_cluster;
  return GX_OK;
}

int gx_neighborhood_rows(gx_handle* h, const int32_t* nodes, int32_t count, int32_t n_hops, uint8_t* out_rows) {
  if (!h || !nodes || !out_rows) { gx_set_error("gx_neighborhood_rows: NULL argument"); return GX_ERR_INVALID; }
  if (!h->has_graph) { gx_set_error("gx_neighborhood_rows: call gx_set_graph_csr first"); return GX_ERR_INVALID; }
  int rc = check_node_list(h, "gx_neighborhood_rows", nodes, count, n_hops, 1);
  if (rc != GX_OK || count <= 0) return rc;
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  rc = ensure_slot_ws(h);
  if (rc != GX_OK) return rc;
  const size_t bytes = (size_t)count * h->g.N;
  GX_CUDA_CHECK(h->d_nodes.reserve((size_t)count * 4));
  GX_CUDA_CHECK(h->d_rows.reserve(bytes));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->d_nodes.p, nodes, (size_t)count * 4, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(cudaMemsetAsync(h->d_rows.p, 0, bytes, h->stream));
  GX_CUDA_CHECK(gx_launch_hop_rows(h->g, h->d_nodes.as<int32_t>(), count, n_hops, h->ws, h->d_rows.as<uint8_t>(), h->stream));
  h->launches += 1;
  GX_CUDA_CHECK(cudaMemcpyAsync(out_rows, h->d_rows.p, bytes, cudaMemcpyDeviceToHost, h->stream));
  GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  return GX_OK;
}

int gx_count_nodes(gx_handle* h, const int32_t* nodes, int32_t count, int32_t n_hops, int32_t* n_out, int32_t* e_out) {
  if (!h || !nodes) { gx_set_error("gx_count_nodes: NULL argument"); return GX_ERR_INVALID; }
  if (!h->has_graph) { gx_set_error("gx_count_nodes: call gx_set_graph_csr first"); return GX_ERR_INVALID; }
  int rc = check_node_list(h, "gx_count_nodes", nodes, count, n_hops, 1);
  if (rc != GX_OK || count <= 0) return rc;
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  rc = ensure_slot_ws(h);
  if (rc != GX_OK) return rc;
  h->has_plan = false;     // the task buffer is shared with both plans
  h->has_gplan = false;
  GX_CUDA_CHECK(h->d_nodes.reserve((size_t)count * 4));
  GX_CUDA_CHECK(h->d_tasks.reserve((size_t)count * sizeof(GxTask)));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->d_nodes.p, nodes, (size_t)count * 4, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(gx_launch_khop_count(h->g, h->d_nodes.as<int32_t>(), count, n_hops, h->has_model ? h->m.L - 1 : 2, h->ws, h->d_tasks.as<GxTask>(), h->stream));
  h->launches += 1;
  std::vector<GxTask> tk(count);
  GX_CUDA_CHECK(cudaMemcpyAsync(tk.data(), h->d_tasks.p, (size_t)count * sizeof(GxTask), cudaMemcpyDeviceToHost, h->stream));
  GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  for (int t = 0; t < count; ++t) { if (n_out) n_out[t] = tk[t].n; if (e_out) e_out[t] = tk[t].e_d; }
  return GX_OK;
}

int gx_plan_nodes(gx_handle* h, const int32_t* nodes, int32_t count, int32_t n_hops,
                  int64_t* total_nodes, int64_t* total_edges) {
  if (!h || !nodes) { gx_set_error("gx_plan_nodes: NULL argument"); return GX_ERR_INVALID; }
  if (!h->has_graph || !h->has_model) { gx_set_error("gx_plan_nodes: call gx_set_model and gx_set_graph_csr first"); return GX_ERR_INVALID; }
  if (h->g.d != h->m.d) { gx_set_error("gx_plan_nodes: graph feat_dim %d != model input_dim %d", h->g.d, h->m.d); return GX_ERR_INVALID; }
  int rc = check_node_list(h, "gx_plan_nodes", nodes, count, n_hops, 2);
  if (rc != GX_OK) return rc;
  if (count <= 0) { gx_set_error("gx_plan_nodes: count <= 0"); return GX_ERR_INVALID; }
  // the reference indexes pred[gt_label] / a float pred_label vector (explain.py:750-753,789): a label outside [0,C) is an IndexError there
  if (h->has_label && (h->label_min < 0 || h->label_max >= h->m.C)) { gx_set_error("gx_plan_nodes: label values span [%d,%d], model has %d classes", h->label_min, h->label_max, h->m.C); return GX_ERR_INVALID; }
  if (h->pred_min < 0 || h->pred_max >= h->m.C) { gx_set_error("gx_plan_nodes: pred_label values span [%d,%d], model has %d classes", h->pred_min, h->pred_max, h->m.C); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  const double t0 = h->host_timing ? now_us() : 0.0;
  h->has_plan = false;
  h->has_gplan = false;
  rc = ensure_slot_ws(h);
  if (rc != GX_OK) return rc;
  GX_CUDA_CHECK(h->d_nodes.reserve((size_t)count * 4));
  GX_CUDA_CHECK(h->d_tasks.reserve((size_t)count * sizeof(GxTask)));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->d_nodes.p, nodes, (size_t)count * 4, cudaMemcpyHostToDevice, h->stream));
  const int row_lvl = h->m.L - 1;
  GX_CUDA_CHECK(gx_launch_khop_count(h->g, h->d_nodes.as<int32_t>(), count, n_hops, row_lvl, h->ws, h->d_tasks.as<GxTask>(), h->stream));
  h->launches += 1;
  h->tasks.resize(count);
  GX_CUDA_CHECK(cudaMemcpyAsync(h->tasks.data(), h->d_tasks.p, (size_t)count * sizeof(GxTask), cudaMemcpyDeviceToHost, h->stream));
  GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  const double t1 = h->host_timing ? now_us() : 0.0;
  // host, step 1: status checks and the offsets the fill kernel needs
  int64_t tn = 0, te = 0, tp = 0;
  for (int t = 0; t < count; ++t) {
    GxTask& T = h->tasks[t];
    if (T.status != 0) {
      gx_set_error("gx_plan_nodes: node %d is not inside its own %d-hop neighbourhood (isolated node?)", T.node, n_hops);
      return GX_ERR_NODE;
    }
    if (T.e_d % 2 != 0) { gx_set_error("gx_plan_nodes: induced sub-adjacency of node %d is not symmetric", T.node); return GX_ERR_INVALID; }
    T.node_off = tn; T.rp_off = tn + t; T.edge_off = te; T.pair_off = tp;
    tn += T.n; te += T.e_d; tp += T.npairs;
  }
  h->count = count; h->n_hops = n_hops; h->total_n = tn; h->total_e = te;
  GX_CUDA_CHECK(cudaMemcpyAsync(h->d_tasks.p, h->tasks.data(), (size_t)count * sizeof(GxTask), cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(h->d_counters.reserve(kNumClasses * 4));
  GX_CUDA_CHECK(h->d_nbrs.reserve((size_t)std::max<int64_t>(tn, 1) * 4));
  GX_CUDA_CHECK(h->d_lo2gid.reserve((size_t)std::max<int64_t>(tn, 1) * 4));
  GX_CUDA_CHECK(h->d_srp.reserve((size_t)(tn + count) * 4));
  GX_CUDA_CHECK(h->d_irp.reserve((size_t)(tn + count) * 4));
  GX_CUDA_CHECK(h->d_scol.reserve((size_t)std::max<int64_t>(te, 1) * 4));
  GX_CUDA_CHECK(h->d_icol.reserve((size_t)std::max<int64_t>(te, 1) * 4 * 3));
  GX_CUDA_CHECK(h->d_pairs.reserve((size_t)std::max<int64_t>(tp, 1) * 4 * 6));
  h->plan.tasks = h->d_tasks.as<GxTask>();
  h->plan.nbrs = h->d_nbrs.as<int32_t>();
  h->plan.lo2gid = h->d_lo2gid.as<int32_t>();
  h->plan.sub_rowptr = h->d_srp.as<int32_t>();
  h->plan.irowptr = h->d_irp.as<int32_t>();
  h->plan.sub_col = h->d_scol.as<int32_t>();
  h->plan.icol = h->d_icol.as<int32_t>();
  h->plan.cs2is = h->plan.icol + te;
  h->plan.is2cs = h->plan.icol + 2 * te;
  int32_t* pb = h->d_pairs.as<int32_t>();
  h->plan.pair_i = pb; h->plan.pair_j = pb + tp; h->plan.pair_pij = pb + 2 * tp;
  h->plan.pair_pji = pb + 3 * tp; h->plan.pair_oij = pb + 4 * tp; h->plan.pair_oji = pb + 5 * tp;
  const double t2 = h->host_timing ? now_us() : 0.0;
  GX_CUDA_CHECK(gx_launch_khop_fill(h->g, count, n_hops, h->ws, h->plan, h->stream));
  h->launches += 1;
  // host, step 2 (while the fill kernel runs): launch classes and work order.  Nothing here is read by the device: T.smem_bytes and the
  // class lists stay on the host, only the order array is uploaded.
  const LaunchClass& cluster_cls = h->classes[kClusterClass];
  for (int c = 0; c < kNumClasses; ++c) h->class_order[c].clear();
  auto cost = [&](int32_t t) { const GxTask& T = h->tasks[t]; return (int64_t)T.e1 * (h->m.d + 2 * h->m.hid) + (int64_t)T.n2 * 600 + (int64_t)T.npairs * 60; };
  const int g_cluster_size = h->cluster_size > 1 ? h->cluster_size : 1;
  const int64_t g_cluster_cost = h->cluster_cost;
  h->plan_cluster = g_cluster_size;
  for (int t = 0; t < count; ++t) {
    GxTask& T = h->tasks[t];
    int bytes = 0;
    int cls = h->m.variant ? kStreamClass : task_smem_class(h, T, &bytes);
    if (cls < kStreamClass && g_cluster_size > 1 && cost(t) > g_cluster_cost) {
      // expensive task: one thread-block cluster (explain_node.cu, CS CTAs share the rows and pairs); decided by the task alone
      const GxLayout L = gx_make_layout(T.n, T.n1, T.n2, T.e1, h->m.d, h->m.hid, h->m.emb, h->m.C, cluster_cls.threads / 32, 2, g_cluster_size);
      if ((int64_t)L.total_words * 4 <= cluster_cls.cap_bytes) { cls = kClusterClass; bytes = L.total_words * 4; }
    }
    T.smem_bytes = bytes;
    h->class_order[cls].push_back(t);
  }
  if (h->cluster_size == 0 && !h->m.variant && !h->force_stream && h->class_order[kStreamClass].empty()) {
    // Latency mode (cluster_size 0): a batch that leaves SMs idle (one explain() call, a shard of a strong-scaled list) is bounded by the
    // latency of its most expensive tasks, so those run on thread-block clusters of the spare SMs.  A full batch (700 syn1 nodes on one
    // GPU needs ~180 SM-slots) has no spare SM and stays as it is.  A cluster sums the per-warp dL/dsF partials of its 32 / 64 warps in
    // another order than one CTA's 16 warps: the masks agree with the single-CTA run to round-off, not bit for bit -- which is why
    // this mode is opt-in.
    // Latency model (rough estimates, not calibrated on the H100): a fixed time per cost unit on one CTA; a cluster divides that by
    // its size and adds a fixed cluster-barrier time per 100 epochs (ovh below, in ms).
    double demand = 0;
    for (int c = 0; c < kStreamClass; ++c) demand += (double)h->class_order[c].size() / h->classes[c].ctas_per_sm;
    const int spare = h->num_sms - (int)(demand + 0.999);
    std::vector<int32_t> cand;
    for (int c : {kTwoClass, kOneClass}) for (int32_t t : h->class_order[c]) cand.push_back(t);
    std::stable_sort(cand.begin(), cand.end(), [&](int32_t x, int32_t y) { return cost(x) > cost(y); });
    auto lat = [&](int32_t t) { return 6e-6 * (double)cost(t); };
    int best_cs = 1, best_k = 0;
    if (!cand.empty() && spare >= 2) {
      double best = lat(cand[0]);
      for (int cs : {2, 4}) {
        const double ovh = cs == 2 ? 0.55 : 0.8;
        // the k most expensive tasks on clusters: every one of them must gain, and all of them must fit the class and the spare SMs
        int k = 0;
        while (k < (int)cand.size() && (k + 1) * cs <= spare && lat(cand[k]) / cs + ovh < lat(cand[k])) {
          const GxTask& T = h->tasks[cand[k]];
          const GxLayout L = gx_make_layout(T.n, T.n1, T.n2, T.e1, h->m.d, h->m.hid, h->m.emb, h->m.C, cluster_cls.threads / 32, 2, cs);
          if ((int64_t)L.total_words * 4 > cluster_cls.cap_bytes) break;
          ++k;
        }
        if (k == 0) continue;
        const double span = std::max(lat(cand[0]) / cs + ovh, k < (int)cand.size() ? lat(cand[k]) : 0.0);
        if (span < best * 0.95) { best = span; best_cs = cs; best_k = k; }
      }
    }
    if (best_cs > 1) {
      h->plan_cluster = best_cs;
      for (int i = 0; i < best_k; ++i) {
        const int32_t t = cand[i];
        GxTask& T = h->tasks[t];
        const GxLayout L = gx_make_layout(T.n, T.n1, T.n2, T.e1, h->m.d, h->m.hid, h->m.emb, h->m.C, cluster_cls.threads / 32, 2, best_cs);
        T.smem_bytes = L.total_words * 4;
        for (int c : {kTwoClass, kOneClass}) {
          auto& v = h->class_order[c];
          v.erase(std::remove(v.begin(), v.end(), t), v.end());
        }
        h->class_order[kClusterClass].push_back(t);
      }
    }
  }
  std::vector<int32_t> order_all;
  for (int c = 0; c < kNumClasses; ++c) {
    auto& v = h->class_order[c];
    std::stable_sort(v.begin(), v.end(), [&](int32_t x, int32_t y) { return cost(x) > cost(y); });
  }
  {
    // The batch makespan is the latency of its most expensive tasks (one wave; a 512-thread task is slower
    // when it shares the SM with a second one).  The top-K tasks of the 2-per-SM
    // class therefore run alone on an SM (moved to the 1-per-SM class, which requests the whole shared memory).
    auto& two = h->class_order[kTwoClass];
    auto& one = h->class_order[kOneClass];
    // only when the 2-per-SM class really pairs up tasks, and the exclusive SMs still leave everything in one wave
    int k = 0;
    if ((int)two.size() > h->num_sms) {
      k = h->exclusive_topk;
      while (k > 0 && (int)one.size() + k + ((int)two.size() - k + 1) / 2 > (h->num_sms * 17) / 20) --k;
    }
    if (k > 0 && (int)two.size() > k) {
      one.insert(one.end(), two.begin(), two.begin() + k);
      two.erase(two.begin(), two.begin() + k);
      std::stable_sort(one.begin(), one.end(), [&](int32_t x, int32_t y) { return cost(x) > cost(y); });
    }
  }
  for (int c = 0; c < kNumClasses; ++c) {
    auto& v = h->class_order[c];
    order_all.insert(order_all.end(), v.begin(), v.end());
  }
  GX_CUDA_CHECK(h->d_order.reserve((size_t)count * 4));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->d_order.p, order_all.data(), (size_t)count * 4, cudaMemcpyHostToDevice, h->stream));
  // idx_new (the canonical description's position of the node) is copied back by gx_plan_fetch on demand.  The host still waits for the
  // fill kernel: explainer launches queued BEHIND it all become runnable at the same instant and the block scheduler interleaves the
  // launch classes arbitrarily, which lengthens the batch; issued one by
  // one onto an idle GPU the most expensive class is placed first.
  GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  h->tasks_fetched = false;
  h->has_plan = true;
  if (h->host_timing) {
    const double t3 = now_us();
    fprintf(stderr, "[gnnx] gx_plan_nodes(%d): count kernel + copy %.0f us, offsets + uploads %.0f us, fill kernel (host classes / order underneath) %.0f us\n", count, t1 - t0, t2 - t1, t3 - t2);
  }
  if (total_nodes) *total_nodes = tn;
  if (total_edges) *total_edges = te;
  return GX_OK;
}

int gx_plan_fetch(gx_handle* h, int64_t* node_off, int64_t* edge_off, int32_t* neighbors,
                  int32_t* node_idx_new, int32_t* sub_rowptr, int32_t* sub_col) {
  if (!h || !h->has_plan) { gx_set_error("gx_plan_fetch: no plan (call gx_plan_nodes)"); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  const int count = h->count;
  if (node_off) { for (int t = 0; t < count; ++t) node_off[t] = h->tasks[t].node_off; node_off[count] = h->total_n; }
  if (edge_off) { for (int t = 0; t < count; ++t) edge_off[t] = h->tasks[t].edge_off; edge_off[count] = h->total_e; }
  if (node_idx_new) {
    if (!h->tasks_fetched) {   // only idx_new comes from the device copy (the host copy carries the launch classes)
      std::vector<GxTask> dev(count);
      GX_CUDA_CHECK(cudaMemcpyAsync(dev.data(), h->d_tasks.p, (size_t)count * sizeof(GxTask), cudaMemcpyDeviceToHost, h->stream));
      GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
      for (int t = 0; t < count; ++t) h->tasks[t].idx_new = dev[t].idx_new;
      h->tasks_fetched = true;
    }
    for (int t = 0; t < count; ++t) node_idx_new[t] = h->tasks[t].idx_new;
  }
  if (neighbors) GX_CUDA_CHECK(cudaMemcpyAsync(neighbors, h->d_nbrs.p, (size_t)h->total_n * 4, cudaMemcpyDeviceToHost, h->stream));
  if (sub_rowptr) GX_CUDA_CHECK(cudaMemcpyAsync(sub_rowptr, h->d_srp.p, (size_t)(h->total_n + count) * 4, cudaMemcpyDeviceToHost, h->stream));
  if (sub_col) GX_CUDA_CHECK(cudaMemcpyAsync(sub_col, h->d_scol.p, (size_t)h->total_e * 4, cudaMemcpyDeviceToHost, h->stream));
  GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  return GX_OK;
}

}  // extern "C"

// mode 0: Explainer.explain's optimisation loop; mode 1: its model="grad" baseline (one forward/backward, explain.py:125-133,717-738)
static int explain_nodes_impl(gx_handle* h, const gx_hparams* hp, int mode, gx_memspace space, const gx_explain_io* io) {
  const char* who = "gx_explain_nodes";
  if (!h || !hp) { gx_set_error("gx_explain_nodes: NULL argument"); return GX_ERR_INVALID; }
  if (!h->has_plan) { gx_set_error("gx_explain_nodes: no plan (call gx_plan_nodes)"); return GX_ERR_INVALID; }
  const double t_entry = h->host_timing ? now_us() : 0.0;
  const bool all_var = h->m.variant || hp->opt != GX_OPT_ADAM;   // every task through explain_var.cu
  int rc = check_explain_hparams(who, hp, mode, all_var, io, false);
  if (rc != GX_OK) return rc;
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  const int count = h->count;
  const int64_t te = h->total_e;
  IoDev D;
  rc = io_prepare(h, who, hp, mode, space, io, count, te, h->m.d, h->m.C, &D);
  if (rc != GX_OK) return rc;
  GxHparamsDev hd;
  fill_hparams(h, hp, mode, D.x.trace != nullptr, &hd);
  rc = upload_adam_table(h, hp, hd.iters, mode == 0 ? hp->start_step : 0);
  if (rc != GX_OK) return rc;
  hd.adam_tab = h->d_adam.as<float2>();   // (the buffer may have been (re)allocated by the upload)
  GX_CUDA_CHECK(cudaMemsetAsync(h->d_counters.p, 0, kNumClasses * 4, h->stream));
  auto outer_pairs = [&]() -> int {
    // pairs between two outermost nodes: independent scalar recurrences, whole batch in one launch
    GX_CUDA_CHECK(gx_launch_outer_pairs(hd, h->g, h->plan, count, D.m0, D.out, D.x, h->stream));
    h->launches += 1;
    return GX_OK;
  };
  if (all_var && !h->m.variant) {
    // default model, optimiser other than Adam: the whole batch in one launch of the variant kernel (+ the outer-pair recurrences)
    rc = launch_var_batch(h, who, 0, hd, D);
    if (rc == GX_OK) rc = outer_pairs();
    if (rc != GX_OK) return rc;
  } else {
    // per launch class: its kernel, grid, block and shared memory (the largest footprint of its tasks) and its number of pair slabs
    GxExplainLaunch cfg[kNumClasses] = {};
    int slabs[kNumClasses] = {};
    NodeKernel kernel[kNumClasses] = {};
    for (int c = 0; c < kNumClasses; ++c) {
      const LaunchClass& K = h->classes[c];
      const int nt = (int)h->class_order[c].size();
      int need = 0;
      for (int32_t t : h->class_order[c]) need = std::max(need, h->tasks[t].smem_bytes);
      cfg[c].threads = K.threads;
      cfg[c].dbg = h->dbg;
      cfg[c].x = D.x;
      if (c == kClusterClass) {
        // CTAs, CS per task, one pair slab per cluster; the class requests the whole SM (see the 1-per-SM class)
        kernel[c] = NodeKernel::cluster;
        cfg[c].cluster = h->plan_cluster;
        cfg[c].grid = std::min<int>(nt, h->num_sms / h->plan_cluster) * h->plan_cluster;
        cfg[c].smem_bytes = std::max(need, K.cap_bytes - 2048);
        slabs[c] = cfg[c].grid / h->plan_cluster;
      } else if (K.cap_bytes > 0) {
        // the dynamic shared memory request shrinks to what the class needs (more CTAs can co-reside).  The 1-per-SM class requests
        // the whole SM: a CTA of another class next to it would take the room the scheduler's breadth-first placement needs for the
        // small classes launched last (2 KB short of the class limit: kernels with a trace carry 1.2 KB of static shared memory)
        kernel[c] = NodeKernel::smem;
        cfg[c].grid = std::min<int>(nt, h->num_sms * K.ctas_per_sm);
        cfg[c].smem_bytes = c == kOneClass ? std::max(need, K.cap_bytes - 2048) : std::max(need, 1024);
        slabs[c] = cfg[c].grid;
      } else if (nt > 0) {
        // slab class: as many tasks in flight as the device memory holds, up to one per SM (CTAs of explain_stream.cu / explain_var.cu,
        // gangs of explain_gang.cu)
        int max_slabs = h->num_sms, gang = 0;   // gang > 0: explain_gang.cu with this many CTAs per task
        if (!h->m.variant && h->gang_override >= 0 && h->m.d <= 128 && gx_gang_smem_bytes(h->m.d, h->m.hid, h->m.C) <= gx_explain_max_smem()) {
          // explain_gang.cu: G co-resident CTAs per task.  As many tasks in flight as keep their randomly accessed state
          // (a, gE: 8 B per directed edge; P, dP, dY1: 240 B per node) inside 5/8 of the L2 (31 MB of an H100's 50 MB), the SMs
          // divided evenly among them.
          int64_t ws = 1;
          for (int32_t t : h->class_order[c]) ws = std::max<int64_t>(ws, (int64_t)h->tasks[t].e_d * 8 + (int64_t)h->tasks[t].n * 240);
          const int64_t l2_budget = h->l2_bytes * 5 / 8;
          int ngangs = (int)std::max<int64_t>(1, std::min<int64_t>(std::min(nt, h->num_sms), l2_budget / ws));
          gang = std::max(1, std::min(h->num_sms / ngangs, GX_MAX_GANG));
          if (h->gang_override > 0) gang = std::min(std::min(h->gang_override, h->num_sms), GX_MAX_GANG);
          max_slabs = std::max(1, std::min(ngangs, h->num_sms / gang));
        }
        kernel[c] = h->m.variant ? NodeKernel::variant : gang > 0 ? NodeKernel::gang : NodeKernel::stream1;
        auto stream_words = [&](const GxTask& T) { return gx_make_stream_layout(T.n, T.n1, T.n2, T.e_d, T.npairs_in, h->m.d, h->m.hid, GX_STREAM_THREADS / 32).total_words; };
        rc = h->m.variant ? size_slab_launch(h, who, h->class_order[c], [&](const GxTask& T) { return var_slab_words(h, 0, T); }, max_slabs, &cfg[c])
                          : size_slab_launch(h, who, h->class_order[c], stream_words, max_slabs, &cfg[c]);
        if (rc != GX_OK) return rc;
        slabs[c] = cfg[c].grid;
        if (gang > 0) {
          cfg[c].gang = gang;
          cfg[c].grid = slabs[c] * gang;
          GX_CUDA_CHECK(h->d_gang.reserve((size_t)slabs[c] * 16));
          cfg[c].gang_bars = h->d_gang.as<unsigned long long>();
          cfg[c].gang_mail = reinterpret_cast<int32_t*>(h->d_gang.as<char>() + (size_t)slabs[c] * 8);
        }
      }
    }
    auto launch = [&](int c, const GxExplainLaunch& k, cudaStream_t s) -> cudaError_t {
      switch (kernel[c]) {
        case NodeKernel::smem:
        case NodeKernel::cluster: return gx_launch_explain(k, h->g, h->m, hd, h->plan, D.m0, D.out, D.feat, s);
        case NodeKernel::variant: return gx_launch_explain_var(k, 0, h->g, h->gb, h->m, h->head, hd, h->plan, D.m0, D.out, D.feat, s);
        case NodeKernel::stream1: return gx_launch_explain_stream(k, h->g, h->m, hd, h->plan, D.m0, D.out, D.feat, s);
        case NodeKernel::gang: {
          const cudaError_t e = cudaMemsetAsync(k.gang_bars, 0, (size_t)(k.grid / k.gang) * 16, s);
          return e != cudaSuccess ? e : gx_launch_explain_gang(k, h->g, h->m, hd, h->plan, D.m0, D.out, D.feat, s);
        }
      }
      return cudaErrorInvalidValue;
    };
    rc = launch_classes(h, kNumClasses, cfg, slabs, launch, outer_pairs);
    if (rc != GX_OK) return rc;
  }
  if (D.x.trace) {
    GX_CUDA_CHECK(gx_launch_trace_finalize(hd, h->plan, count, D.x, h->stream));
    h->launches += 1;
  }
  GX_CUDA_CHECK(cudaEventRecord(h->ev_t1, h->stream));
  h->timed = true;
  if (h->host_timing) fprintf(stderr, "[gnnx] gx_explain_nodes: host %.0f us from entry to the last launch\n", now_us() - t_entry);
  return io_finish(h, hp, space, io, count, te, h->m.d, h->m.C, D);
}

extern "C" {

int gx_explain_nodes(gx_handle* h, const gx_hparams* hp, gx_memspace space, const float* m0_edges,
                     float* edge_mask, float* feat_mask) {
  gx_explain_io io;
  memset(&io, 0, sizeof(io));
  io.m0_edges = m0_edges; io.edge_mask = edge_mask; io.feat_mask = feat_mask;
  return explain_nodes_impl(h, hp, 0, space, &io);
}

int gx_explain_nodes_ex(gx_handle* h, const gx_hparams* hp, gx_memspace space, const gx_explain_io* io) {
  return explain_nodes_impl(h, hp, 0, space, io);
}

int gx_grad_nodes(gx_handle* h, gx_memspace space, float* edge_mask) {
  if (h && h->has_plan) {
    // The reference differentiates its raw sub_adj, diagonal included: a self loop adds a term to the forward and backward and a
    // diagonal entry sigmoid(2|g_ii|) to the result.  The kernels work on the edge list without the diagonal, so refuse.
    for (int t = 0; t < h->count; ++t) {
      if (h->tasks[t].loops > 0) {
        gx_set_error("gx_grad_nodes: the neighbourhood of node %d has %d self loop(s); the gradient baseline is not built for self loops",
                     h->tasks[t].node, h->tasks[t].loops);
        return GX_ERR_UNSUPPORTED;
      }
    }
  }
  gx_hparams hp;
  gx_default_hparams(&hp);
  gx_explain_io io;
  memset(&io, 0, sizeof(io));
  io.edge_mask = edge_mask;
  return explain_nodes_impl(h, &hp, 1, space, &io);
}

}  // extern "C"
