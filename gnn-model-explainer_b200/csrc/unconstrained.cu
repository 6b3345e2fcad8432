// unconstrained.cu -- host side of Explainer.explain(..., unconstrained=True) for the planned nodes (gx_plan_nodes) or graphs
// (gx_plan_graphs): checks, staging and one persistent launch of explain_dense.cu over the whole batch, largest task first.
#include <string.h>

#include <algorithm>
#include <numeric>
#include <vector>

#include "host.cuh"

static int explain_unconstrained_impl(gx_handle* h, bool graph, const gx_hparams* hp, gx_memspace space, const float* m0_dense,
                                      float* edge_mask, float* mask_dense, float* trace, float* trace_pred) {
  const char* who = graph ? "gx_explain_graphs_unconstrained" : "gx_explain_nodes_unconstrained";
  if (!h || !hp || !edge_mask) { gx_set_error("%s: NULL argument", who); return GX_ERR_INVALID; }
  if (graph ? !h->has_gplan : !h->has_plan) { gx_set_error("%s: no plan (call %s)", who, graph ? "gx_plan_graphs" : "gx_plan_nodes"); return GX_ERR_INVALID; }
  if (graph && h->gb.d != h->m.d) { gx_set_error("%s: feat_dim %d != model input_dim %d", who, h->gb.d, h->m.d); return GX_ERR_INVALID; }
  int rc = check_explain_hparams(who, hp, 0, false, nullptr, graph);
  if (rc != GX_OK) return rc;
  if (h->has_model && h->m.att) {
    gx_set_error("%s: attention models (GX_MODEL_ATT) are not built for the unconstrained mask (the kernel sums its per-layer pair products in one product)", who);
    return GX_ERR_UNSUPPORTED;
  }
  if (h->has_model && h->m.d >= GX_VAR_WIDE_MIN) {
    gx_set_error("%s: inputs wider than 128 (input_dim=%d) are not built for the unconstrained mask", who, h->m.d);
    return GX_ERR_UNSUPPORTED;
  }
  if (h->has_model && (h->m.hid > 128 || h->m.emb > 128)) {
    gx_set_error("%s: hidden / output widths above 128 (hidden_dim=%d output_dim=%d) are not built for the unconstrained mask", who, h->m.hid, h->m.emb);
    return GX_ERR_UNSUPPORTED;
  }
  if (hp->init == GX_INIT_STATE) { gx_set_error("%s: GX_INIT_STATE is not built for the unconstrained mask", who); return GX_ERR_UNSUPPORTED; }
  if (hp->init == GX_INIT_M0 && !m0_dense) { gx_set_error("%s: GX_INIT_M0 needs m0_dense", who); return GX_ERR_INVALID; }
  if (trace_pred && !trace) { gx_set_error("%s: trace_pred needs trace", who); return GX_ERR_INVALID; }
  if (hp->start_step != 0) { gx_set_error("%s: start_step != 0 without GX_INIT_STATE", who); return GX_ERR_INVALID; }
  const int count = h->count;
  // n of every task's dense problem: the k-hop set in node mode, the padded size in graph mode
  std::vector<int64_t> doff(count + 1, 0);
  for (int t = 0; t < count; ++t) {
    const int n = graph ? h->gb.max_nodes : h->tasks[t].n;
    if (n > GX_DENSE_MAX_N) { gx_set_error("%s: task %d has n = %d > %d (the dense mask has n^2 parameters)", who, t, n, GX_DENSE_MAX_N); return GX_ERR_UNSUPPORTED; }
    doff[t + 1] = doff[t] + (int64_t)n * n;
  }
  const int bytes = gx_dense_smem_bytes(h->m.d, h->m.L, h->m.hid, h->m.emb, h->m.C, h->head);
  if (bytes > gx_explain_max_smem()) { gx_set_error("%s: model does not fit the unconstrained kernel (%d bytes of shared memory)", who, bytes); return GX_ERR_UNSUPPORTED; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  const int per_sm = gx_dense_ctas_per_sm(h->m, h->head);
  if (per_sm < 1) { gx_set_error("%s: the unconstrained kernel cannot be resident (%d bytes of shared memory)", who, bytes); return GX_ERR_UNSUPPORTED; }
  const int64_t dense = doff[count], te = h->total_e;
  GX_CUDA_CHECK(h->d_dense_off.reserve((size_t)(count + 1) * 8));
  // pageable source: the copy is staged before the call returns, the vector may go out of scope
  GX_CUDA_CHECK(cudaMemcpyAsync(h->d_dense_off.p, doff.data(), (size_t)(count + 1) * 8, cudaMemcpyHostToDevice, h->stream));
  GxDenseIo io{};
  io.dense_off = h->d_dense_off.as<int64_t>();
  io.epochs = hp->num_epochs;
  const float* m0 = hp->init == GX_INIT_M0 ? m0_dense : nullptr;
  if (space == GX_DEVICE) {
    io.m0 = m0; io.out_mask = edge_mask; io.out_dense = mask_dense; io.trace = trace; io.trace_pred = trace_pred;
  } else {
    GX_CUDA_CHECK(stage_in(h, h->d_m0dense, m0, (size_t)dense, &io.m0));
    GX_CUDA_CHECK(stage_out(h->d_out, edge_mask, (size_t)std::max<int64_t>(te, 1), &io.out_mask));
    GX_CUDA_CHECK(stage_out(h->d_mdense, mask_dense, (size_t)dense, &io.out_dense));
    GX_CUDA_CHECK(stage_out(h->d_trace, trace, (size_t)count * hp->num_epochs * GX_TRACE_COLS, &io.trace));
    GX_CUDA_CHECK(stage_out(h->d_trpred, trace_pred, (size_t)count * hp->num_epochs * h->m.C, &io.trace_pred));
  }
  GxHparamsDev hd;
  fill_hparams(h, hp, 0, trace != nullptr, &hd);
  if (graph) hd.c_lap = 0.f;   // lap_loss = 0 in graph mode (explain.py:787-788)
  rc = upload_adam_table(h, hp, hd.iters, 0);
  if (rc != GX_OK) return rc;
  hd.adam_tab = h->d_adam.as<float2>();
  // the work queue: largest task first
  std::vector<int32_t> order(count);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int32_t x, int32_t y) { return doff[x + 1] - doff[x] > doff[y + 1] - doff[y]; });
  GX_CUDA_CHECK(h->d_uorder.reserve((size_t)count * 4));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->d_uorder.p, order.data(), (size_t)count * 4, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(h->d_counters.reserve(kNumClasses * 4));
  GX_CUDA_CHECK(cudaMemsetAsync(h->d_counters.p, 0, 4, h->stream));
  const int vw = gx_var_row_stride(h->m.hid, h->m.emb);
  GxExplainLaunch cfg{};
  cfg.order = h->d_uorder.as<int32_t>(); cfg.ntasks = count; cfg.counter = h->d_counters.as<int32_t>();
  rc = size_slab_launch(h, who, order, [&](const GxTask& T) {
    return gx_make_dense_layout(graph ? h->gb.max_nodes : T.n, h->m.d, h->m.L, vw).total_words; }, h->num_sms * per_sm, &cfg);
  if (rc == GX_OK) rc = begin_timing(h);
  if (rc != GX_OK) return rc;
  GX_CUDA_CHECK(gx_launch_explain_dense(cfg, graph ? 1 : 0, h->g, h->gb, h->m, h->head, hd, h->plan, io, h->stream));
  h->launches += 1;
  GX_CUDA_CHECK(cudaEventRecord(h->ev_t1, h->stream));
  h->timed = true;
  if (space == GX_HOST) {
    GX_CUDA_CHECK(stage_back(h, edge_mask, (const float*)io.out_mask, (size_t)te));
    GX_CUDA_CHECK(stage_back(h, mask_dense, (const float*)io.out_dense, (size_t)dense));
    GX_CUDA_CHECK(stage_back(h, trace, (const float*)io.trace, (size_t)count * hp->num_epochs * GX_TRACE_COLS));
    GX_CUDA_CHECK(stage_back(h, trace_pred, (const float*)io.trace_pred, (size_t)count * hp->num_epochs * h->m.C));
    GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  }
  return GX_OK;
}

extern "C" {

int gx_explain_nodes_unconstrained(gx_handle* h, const gx_hparams* hp, gx_memspace space, const float* m0_dense,
                                   float* edge_mask, float* mask_dense, float* trace, float* trace_pred) {
  return explain_unconstrained_impl(h, false, hp, space, m0_dense, edge_mask, mask_dense, trace, trace_pred);
}

int gx_explain_graphs_unconstrained(gx_handle* h, const gx_hparams* hp, gx_memspace space, const float* m0_dense,
                                    float* edge_mask, float* mask_dense, float* trace, float* trace_pred) {
  return explain_unconstrained_impl(h, true, hp, space, m0_dense, edge_mask, mask_dense, trace, trace_pred);
}

}  // extern "C"
