// api.cu -- C-ABI host side of libgnnx.so (see include/gnnx.h for the contract and the reference call sites each entry point
// replaces): the handle, model and graph upload, timing and test knobs, the steps node and graph mode share (argument checks, I/O
// staging, optimiser tables, pair slabs), and the post-processing, comm and forward entry points.  Node mode lives in node_mode.cu,
// graph mode in graph_mode.cu.  No CPU compute path exists here: every algorithmic step is a kernel.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <iterator>
#include <memory>
#include <numeric>
#include <vector>

#include "host.cuh"

static thread_local char g_err[1024] = "";

void gx_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_node_list(const gx_handle* h, const char* who, const int32_t* nodes, int32_t count, int32_t n_hops, int min_hops) {
  if (n_hops < 1 || n_hops >= GX_MAX_LEVELS) { gx_set_error("%s: n_hops=%d outside [1,%d]", who, n_hops, GX_MAX_LEVELS - 1); return GX_ERR_INVALID; }
  if (n_hops < min_hops) { gx_set_error("%s: n_hops=%d never contains the node itself without a self loop", who, n_hops); return GX_ERR_UNSUPPORTED; }
  for (int t = 0; t < count; ++t)
    if (nodes[t] < 0 || nodes[t] >= h->g.N) { gx_set_error("%s: node %d out of range [0,%lld)", who, nodes[t], (long long)h->g.N); return GX_ERR_INVALID; }
  return GX_OK;
}

int check_optimiser(const char* who, const gx_hparams* hp) {
  if (hp->opt < GX_OPT_ADAM || hp->opt > GX_OPT_ADAGRAD) { gx_set_error("%s: unknown optimiser %d", who, hp->opt); return GX_ERR_INVALID; }
  if (hp->opt_scheduler < GX_SCHED_NONE || hp->opt_scheduler > GX_SCHED_COS) { gx_set_error("%s: unknown scheduler %d", who, hp->opt_scheduler); return GX_ERR_INVALID; }
  if (hp->opt_scheduler == GX_SCHED_STEP && hp->opt_decay_step < 1) { gx_set_error("%s: step scheduler needs opt_decay_step >= 1", who); return GX_ERR_INVALID; }
  if (hp->opt_scheduler == GX_SCHED_COS && hp->opt_restart < 1) { gx_set_error("%s: cos scheduler needs opt_restart >= 1", who); return GX_ERR_INVALID; }
  return GX_OK;
}

// var: the call runs on the variant kernels (model variant or an optimiser other than Adam), which build the mask optimisation only.
// init_first: graph mode has always checked the initialisation before the optimiser, node mode after the variant-path refusal; a call
// with two faults gets the status of the first.
int check_explain_hparams(const char* who, const gx_hparams* hp, int mode, bool var, const gx_explain_io* io, bool init_first) {
  // mask_act "ReLU": the reference's entropy term takes log(1 - relu(M)) with M ~ N(1, 2/n) -> NaN masks from step 1 (explain.py:755-770;
  // pinned by tests/test_oracle.py): nothing to reproduce.  mask_bias: the bias parameter starts at 0 where ReLU6'(0) = 0, so Adam never
  // moves it and the result equals the default run bit for bit (explain.py:657-660,673-676; same test): accepted, no extra state.
  if (hp->mask_act != 0) { gx_set_error("%s: mask_act != sigmoid is not built (the reference's ReLU variant returns NaN masks)", who); return GX_ERR_UNSUPPORTED; }
  if (hp->num_epochs < 1) { gx_set_error("%s: num_epochs < 1", who); return GX_ERR_INVALID; }
  const bool init_known = hp->init == GX_INIT_M0 || hp->init == GX_INIT_PHILOX || hp->init == GX_INIT_STATE;
  if (init_first && !init_known) { gx_set_error("%s: unknown init %d", who, hp->init); return GX_ERR_INVALID; }
  const int rc = check_optimiser(who, hp);
  if (rc != GX_OK) return rc;
  if (var && (mode != 0 || hp->init == GX_INIT_STATE || (io && (io->trace || io->trace_pred || io->adam_m_out || io->adam_v_out || io->mask_param_out || io->feat_state_out)))) {
    gx_set_error("%s: model variants (num_layers != 3 / --bn / widths > 32) and optimisers other than Adam build the mask optimisation only (no trace, optimiser state or gradient baseline)", who);
    return GX_ERR_UNSUPPORTED;
  }
  if (!init_known) { gx_set_error("%s: unknown init %d", who, hp->init); return GX_ERR_INVALID; }
  return GX_OK;
}

// Validates the optional buffers, stages them (GX_HOST) and fills the kernels' GxExtra.  epochs = num_epochs of the call.
int io_prepare(gx_handle* h, const char* who, const gx_hparams* hp, int mode, gx_memspace space, const gx_explain_io* io, int count,
               int64_t te, int d, int C, IoDev* D) {
  if (!io || !io->edge_mask) { gx_set_error("%s: io->edge_mask is NULL", who); return GX_ERR_INVALID; }
  const bool state = mode == 0 && hp->init == GX_INIT_STATE;
  if (mode == 0 && hp->init != GX_INIT_PHILOX && !io->m0_edges) { gx_set_error("%s: init %d needs m0_edges", who, hp->init); return GX_ERR_INVALID; }
  if (state && (!io->adam_m_in || !io->adam_v_in)) { gx_set_error("%s: GX_INIT_STATE needs adam_m_in and adam_v_in", who); return GX_ERR_INVALID; }
  if (state && hp->start_step < 0) { gx_set_error("%s: start_step < 0", who); return GX_ERR_INVALID; }
  if (!state && hp->start_step != 0) { gx_set_error("%s: start_step != 0 without GX_INIT_STATE", who); return GX_ERR_INVALID; }
  if (io->trace_pred && !io->trace) { gx_set_error("%s: trace_pred needs trace", who); return GX_ERR_INVALID; }
  if (io->trace && mode != 0) { gx_set_error("%s: no trace for the gradient baseline", who); return GX_ERR_INVALID; }
  if (io->trace && hp->num_epochs > 1536) { gx_set_error("%s: a trace supports at most 1536 epochs per call", who); return GX_ERR_UNSUPPORTED; }
  const size_t ne = (size_t)std::max<int64_t>(te, 1), nf = (size_t)count * d, nfs = (size_t)count * 3 * d;
  const size_t ntr = (size_t)count * hp->num_epochs * GX_TRACE_COLS, ntp = (size_t)count * hp->num_epochs * C;
  GxExtra& x = D->x;
  x.epochs = hp->num_epochs;
  if (space == GX_DEVICE) {
    D->m0 = io->m0_edges; D->out = io->edge_mask; D->feat = io->feat_mask;
    x.trace = io->trace; x.trace_pred = io->trace_pred;
    x.adam_m_in = io->adam_m_in; x.adam_v_in = io->adam_v_in; x.feat_state_in = io->feat_state_in;
    x.mask_param_out = io->mask_param_out; x.adam_m_out = io->adam_m_out; x.adam_v_out = io->adam_v_out; x.feat_state_out = io->feat_state_out;
  } else {
    const bool need_m0 = mode == 0 && hp->init != GX_INIT_PHILOX;
    GX_CUDA_CHECK(stage_in(h, h->d_m0, need_m0 ? io->m0_edges : nullptr, (size_t)te, &D->m0));
    GX_CUDA_CHECK(stage_out(h->d_out, io->edge_mask, ne, &D->out));
    GX_CUDA_CHECK(stage_out(h->d_feat, io->feat_mask, nf, &D->feat));
    GX_CUDA_CHECK(stage_out(h->d_trace, io->trace, ntr, &x.trace));
    GX_CUDA_CHECK(stage_out(h->d_trpred, io->trace_pred, ntp, &x.trace_pred));
    GX_CUDA_CHECK(stage_in(h, h->d_min, state ? io->adam_m_in : nullptr, (size_t)te, &x.adam_m_in));
    GX_CUDA_CHECK(stage_in(h, h->d_vin, state ? io->adam_v_in : nullptr, (size_t)te, &x.adam_v_in));
    GX_CUDA_CHECK(stage_in(h, h->d_fsin, state ? io->feat_state_in : nullptr, nfs, &x.feat_state_in));
    GX_CUDA_CHECK(stage_out(h->d_Mout, io->mask_param_out, ne, &x.mask_param_out));
    GX_CUDA_CHECK(stage_out(h->d_mout, io->adam_m_out, ne, &x.adam_m_out));
    GX_CUDA_CHECK(stage_out(h->d_vout, io->adam_v_out, ne, &x.adam_v_out));
    GX_CUDA_CHECK(stage_out(h->d_fsout, io->feat_state_out, nfs, &x.feat_state_out));
  }
  if (!state) { x.adam_m_in = nullptr; x.adam_v_in = nullptr; x.feat_state_in = nullptr; }
  if (x.trace) {
    GX_CUDA_CHECK(h->d_trouter.reserve((size_t)count * hp->num_epochs * 4 * sizeof(double)));
    GX_CUDA_CHECK(cudaMemsetAsync(h->d_trouter.p, 0, (size_t)count * hp->num_epochs * 4 * sizeof(double), h->stream));
    x.tr_outer = h->d_trouter.as<double>();
  }
  return GX_OK;
}

// copies the staged outputs back (GX_HOST) and synchronises
int io_finish(gx_handle* h, const gx_hparams* hp, gx_memspace space, const gx_explain_io* io, int count, int64_t te, int d, int C, const IoDev& D) {
  if (space != GX_HOST) return GX_OK;
  GX_CUDA_CHECK(stage_back(h, io->edge_mask, D.out, (size_t)te));
  GX_CUDA_CHECK(stage_back(h, io->feat_mask, D.feat, (size_t)count * d));
  GX_CUDA_CHECK(stage_back(h, io->trace, D.x.trace, (size_t)count * hp->num_epochs * GX_TRACE_COLS));
  GX_CUDA_CHECK(stage_back(h, io->trace_pred, D.x.trace_pred, (size_t)count * hp->num_epochs * C));
  GX_CUDA_CHECK(stage_back(h, io->mask_param_out, D.x.mask_param_out, (size_t)te));
  GX_CUDA_CHECK(stage_back(h, io->adam_m_out, D.x.adam_m_out, (size_t)te));
  GX_CUDA_CHECK(stage_back(h, io->adam_v_out, D.x.adam_v_out, (size_t)te));
  GX_CUDA_CHECK(stage_back(h, io->feat_state_out, D.x.feat_state_out, (size_t)count * 3 * d));
  GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  return GX_OK;
}

// Per-step table for steps start+1 .. start+iters, in double like torch's python scalars: the epoch's learning rate under the
// scheduler (StepLR / CosineAnnealingLR are stepped once per epoch AFTER the optimiser, explain.py:144-146, so step t runs with the
// rate after t-1 scheduler steps) and, for Adam, the bias corrections (torch/optim/adam.py): (lr_t / (1-b1^t), sqrt(1-b2^t)).
int upload_adam_table(gx_handle* h, const gx_hparams* hp, int iters, int start) {
  // the table on the device is reused while the optimiser settings do not change (one explain call per step in a serving loop)
  AdamKey key{hp->lr, hp->beta1, hp->beta2, hp->opt_decay_rate, hp->opt, hp->opt_scheduler, hp->opt_decay_step, hp->opt_restart, iters, start};
  if (h->adam_valid && memcmp(&key, &h->adam_key, sizeof(key)) == 0 && h->d_adam.p) return GX_OK;
  std::vector<float2> tab(std::max(iters, 1));
  for (int k = 1; k <= iters; ++k) {
    const double t = (double)(start + k);
    const double e = t - 1.0;   // scheduler steps taken so far
    double lr = (double)hp->lr;
    if (hp->opt_scheduler == GX_SCHED_STEP) lr *= std::pow((double)hp->opt_decay_rate, std::floor(e / (double)hp->opt_decay_step));
    else if (hp->opt_scheduler == GX_SCHED_COS) lr *= 0.5 * (1.0 + std::cos(3.14159265358979323846 * e / (double)hp->opt_restart));
    if (hp->opt == GX_OPT_ADAM) {
      const double bc1 = 1.0 - std::pow((double)hp->beta1, t);
      const double bc2 = 1.0 - std::pow((double)hp->beta2, t);
      tab[k - 1].x = (float)(lr / bc1);
      tab[k - 1].y = (float)std::sqrt(bc2);
    } else {
      tab[k - 1].x = (float)lr;
      tab[k - 1].y = 1.0f;
    }
  }
  GX_CUDA_CHECK(h->d_adam.reserve(tab.size() * sizeof(float2)));
  // pageable source: the copy is staged before the call returns, the vector may go out of scope
  GX_CUDA_CHECK(cudaMemcpyAsync(h->d_adam.p, tab.data(), tab.size() * sizeof(float2), cudaMemcpyHostToDevice, h->stream));
  h->adam_key = key; h->adam_valid = true;
  return GX_OK;
}

void fill_hparams(const gx_handle* h, const gx_hparams* hp, int mode, bool trace, GxHparamsDev* hd) {
  hd->out_iter = mode == 1 ? 1 : hp->num_epochs - 1;
  hd->iters = (trace && mode == 0) ? hp->num_epochs : hd->out_iter;   // a trace also needs the last epoch's loss and the density after its step
  hd->one_minus_b1 = 1.0f - hp->beta1;
  hd->b2 = hp->beta2;
  hd->one_minus_b2 = 1.0f - hp->beta2;
  hd->eps = hp->eps;
  hd->c_size = hp->coef_size; hd->c_feat_size = hp->coef_feat_size; hd->c_ent = hp->coef_ent; hd->c_lap = hp->coef_lap;
  hd->adam_tab = h->d_adam.as<float2>();
  hd->init = hp->init;
  hd->flags = (h->ieee_edge ? GX_HP_IEEE_EDGE : 0) | (h->node_generic ? GX_HP_NODE_GENERIC : 0);
  hd->mode = mode;
  hd->opt = hp->opt;
  hd->seed = hp->seed;
}

// Offsets of the plan's dense n x n blocks, one per task, uploaded to d_dense_off; *total = the number of dense entries.
int upload_dense_offsets(gx_handle* h, int64_t* total) {
  const int count = h->count;
  std::vector<int64_t> doff(count + 1);
  int64_t acc = 0;
  for (int t = 0; t < count; ++t) { doff[t] = acc; acc += (int64_t)h->tasks[t].n * h->tasks[t].n; }
  doff[count] = acc;
  GX_CUDA_CHECK(h->d_dense_off.reserve((size_t)(count + 1) * 8));
  // pageable source: the copy is staged before the call returns, the vector may go out of scope
  GX_CUDA_CHECK(cudaMemcpyAsync(h->d_dense_off.p, doff.data(), (size_t)(count + 1) * 8, cudaMemcpyHostToDevice, h->stream));
  *total = acc;
  return GX_OK;
}

// The start of an explain call's device work (ev_t0, gx_last_explain_ms); gx_last_class_ms forgets the classes of the previous call.
int begin_timing(gx_handle* h) {
  std::fill(std::begin(h->class_used), std::end(h->class_used), false);
  GX_CUDA_CHECK(cudaEventRecord(h->ev_t0, h->stream));
  return GX_OK;
}

int place_pair_slabs(gx_handle* h, GxExplainLaunch* cfg, const int* slabs, int n) {
  int64_t words = 0;
  for (int c = 0; c < n; ++c) words += cfg[c].pws_stride_words * std::max(slabs[c], 0);
  GX_CUDA_CHECK(h->d_pws.reserve((size_t)std::max<int64_t>(words, 4) * 4));
  words = 0;
  for (int c = 0; c < n; ++c) {
    cfg[c].pws = h->d_pws.as<float>() + words;
    words += cfg[c].pws_stride_words * std::max(slabs[c], 0);
  }
  return GX_OK;
}

int launch_var_batch(gx_handle* h, const char* who, int graph_mode, const GxHparamsDev& hd, const IoDev& D) {
  const int bytes = gx_var_smem_bytes(graph_mode, h->m.d, h->m.L, h->m.hid, h->m.emb, h->m.C, h->m.att, h->head);
  if (bytes > gx_explain_max_smem()) { gx_set_error("%s: model does not fit the variant kernel", who); return GX_ERR_UNSUPPORTED; }
  int max_ctas = h->num_sms * 4;
  if (graph_mode) {   // graph mode: as many CTAs as are co-resident
    const int per_sm = gx_var_ctas_per_sm(graph_mode, h->m, h->head);
    if (per_sm < 1) { gx_set_error("%s: the variant kernel cannot be resident (%d bytes of shared memory)", who, bytes); return GX_ERR_UNSUPPORTED; }
    max_ctas = h->num_sms * per_sm;
  }
  std::vector<int32_t> all(h->count);
  std::iota(all.begin(), all.end(), 0);
  GxExplainLaunch cfg{};
  cfg.order = h->d_order.as<int32_t>(); cfg.ntasks = h->count; cfg.counter = h->d_counters.as<int32_t>(); cfg.x = D.x;
  int rc = size_slab_launch(h, who, all, [&](const GxTask& T) { return var_slab_words(h, graph_mode, T); }, max_ctas, &cfg);
  if (rc == GX_OK) rc = place_pair_slabs(h, &cfg, &cfg.grid, 1);
  if (rc == GX_OK) rc = begin_timing(h);
  if (rc != GX_OK) return rc;
  GX_CUDA_CHECK(gx_launch_explain_var(cfg, graph_mode, h->g, h->gb, h->m, h->head, hd, h->plan, D.m0, D.out, D.feat, h->stream));
  h->launches += 1;
  return GX_OK;
}

// Model variant (num_gc_layers 2 / 4 .. 7, --bn, widths 33..256, attention, inputs wider than 128): explain_var.cu, true widths (a zero-padded column would enter
// the bn statistics).  att_w != nullptr: an attention model, each layer's (in, in) attention weights right after its conv weights
// (gx_att_weight).  head.k > 0: an MLP prediction head, whose Linears replace pred_w / pred_b (head_w / head_b: head.k + 1 pointers each),
// its block after the conv layers (GxHeadDev).  The widths were checked by the caller.
static int set_variant_model(gx_handle* h, const char* who, const gx_model_dims* dims, const float* const* conv_w, const float* const* conv_b,
                             const float* const* att_w, const float* pred_w, const float* pred_b, GxHeadDev head = GxHeadDev{},
                             const float* const* head_w = nullptr, const float* const* head_b = nullptr) {
  const int L = dims->num_layers, d = dims->input_dim, hid0 = dims->hidden_dim, emb0 = dims->embed_dim, C = dims->num_classes;
  const int att = att_w != nullptr ? 1 : 0;
  if (gx_var_smem_bytes(0, d, L, hid0, emb0, C, att, head) > gx_explain_max_smem()) {
    gx_set_error("%s: model variant does not fit shared memory", who);
    return GX_ERR_UNSUPPORTED;
  }
  std::vector<float> host;
  size_t offW[GX_MAX_LAYERS], offb[GX_MAX_LAYERS];
  auto al4 = [&]() { while (host.size() % 4) host.push_back(0.f); };
  for (int l = 0; l < L; ++l) {
    if (!conv_w[l]) { gx_set_error("%s: conv_w[%d] is NULL", who, l); return GX_ERR_INVALID; }
    if (att && !att_w[l]) { gx_set_error("%s: att_w[%d] is NULL", who, l); return GX_ERR_INVALID; }
    const int win = l == 0 ? d : hid0, wout = l == L - 1 ? emb0 : hid0;
    al4(); offW[l] = host.size();
    host.insert(host.end(), conv_w[l], conv_w[l] + (size_t)win * wout);
    if (att) host.insert(host.end(), att_w[l], att_w[l] + (size_t)win * win);
    al4(); offb[l] = host.size();
    for (int c = 0; c < wout; ++c) host.push_back((conv_b && conv_b[l]) ? conv_b[l][c] : 0.f);
  }
  const int PD0 = hid0 * (L - 1) + emb0;
  al4();
  size_t offWp = host.size(), offbp;
  if (head.k == 0) {
    host.insert(host.end(), pred_w, pred_w + (size_t)C * PD0);
    al4(); offbp = host.size();
    host.insert(host.end(), pred_b, pred_b + C);
  } else {   // Linear j: weight then bias, back to back (gx_head_off); Wp / bp point at the last one
    for (int j = 0; j <= head.k; ++j) {
      const int in = gx_head_in(head, PD0, j), out = gx_head_out(head, C, j);
      if (!head_w[j] || !head_b[j]) { gx_set_error("%s: head_w[%d] or head_b[%d] is NULL", who, j, j); return GX_ERR_INVALID; }
      offWp = host.size();
      host.insert(host.end(), head_w[j], head_w[j] + (size_t)out * in);
      offbp = host.size();
      host.insert(host.end(), head_b[j], head_b[j] + out);
    }
  }
  const size_t offHead = host.size() - gx_head_words(head, PD0, C);
  GX_CUDA_CHECK(h->m_buf.reserve(host.size() * 4));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->m_buf.p, host.data(), host.size() * 4, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  float* b = h->m_buf.as<float>();
  h->m = GxModelDev{};
  h->m.d = d; h->m.hid = hid0; h->m.emb = emb0; h->m.C = C; h->m.L = L;
  h->m.bn = (dims->flags & GX_MODEL_BN) ? 1 : 0; h->m.variant = 1; h->m.att = att;
  for (int l = 0; l < L; ++l) { h->m.W[l] = b + offW[l]; h->m.Wt[l] = nullptr; h->m.b[l] = b + offb[l]; }
  h->m.Wp = b + offWp; h->m.bp = b + offbp;
  h->head = head;
  h->head.W = head.k > 0 ? b + offHead : nullptr;
  h->has_model = true; h->has_plan = false; h->has_gplan = false;   // both plans were laid out for the previous model
  return GX_OK;
}

// The dimension checks of gx_set_model / gx_set_model_att
static int check_model_dims(const char* who, const gx_model_dims* dims) {
  if (dims->num_layers < 2 || dims->num_layers > GX_MAX_LAYERS) {
    gx_set_error("%s: num_layers=%d outside [2,%d] (the k-hop planner's limit: n_hops = num_layers <= %d)", who, dims->num_layers, GX_MAX_LAYERS,
                 GX_MAX_LEVELS - 1);
    return GX_ERR_UNSUPPORTED;
  }
  if (dims->hidden_dim < 1 || dims->embed_dim < 1 || dims->hidden_dim > GX_MAX_WIDTH || dims->embed_dim > GX_MAX_WIDTH) {
    gx_set_error("%s: hidden_dim=%d output_dim=%d; this build supports widths up to GX_MAX_WIDTH = %d (tuned kernels up to 32, the variant kernel beyond)",
                 who, dims->hidden_dim, dims->embed_dim, GX_MAX_WIDTH);
    return GX_ERR_UNSUPPORTED;
  }
  if (dims->input_dim < 1 || dims->input_dim > GX_VAR_WIDE_MAX) {
    gx_set_error("%s: input_dim=%d outside [1,%d] (inputs wider than 128 run the variant kernel's wide path)", who, dims->input_dim, GX_VAR_WIDE_MAX);
    return GX_ERR_UNSUPPORTED;
  }
  if (dims->num_classes < 1) { gx_set_error("%s: num_classes < 1", who); return GX_ERR_INVALID; }
  return GX_OK;
}

// gx_offedge_regularisers (graph = false, after gx_plan_nodes: one n_t x n_t block per node) and gx_offedge_regularisers_graphs
// (graph = true, after gx_plan_graphs: one max_nodes x max_nodes block per graph).
static int offedge_impl(gx_handle* h, bool graph, const gx_hparams* hp, gx_memspace space, const float* m0_dense, double* out) {
  const char* who = graph ? "gx_offedge_regularisers_graphs" : "gx_offedge_regularisers";
  if (!h || !hp || !m0_dense || !out) { gx_set_error("%s: NULL argument", who); return GX_ERR_INVALID; }
  if (graph ? !h->has_gplan : !h->has_plan) { gx_set_error("%s: no plan (call %s)", who, graph ? "gx_plan_graphs" : "gx_plan_nodes"); return GX_ERR_INVALID; }
  if (hp->num_epochs < 1 || hp->num_epochs > 3072) { gx_set_error("%s: num_epochs outside [1,3072]", who); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  const int count = h->count, E = hp->num_epochs;
  int64_t dense = (int64_t)count * h->gb.max_nodes * h->gb.max_nodes;
  int rc = graph ? GX_OK : upload_dense_offsets(h, &dense);
  if (rc != GX_OK) return rc;
  GxHparamsDev hd;
  fill_hparams(h, hp, 0, false, &hd);
  if (hp->opt != GX_OPT_ADAM) { gx_set_error("%s: the off-edge trajectories are built for Adam only", who); return GX_ERR_UNSUPPORTED; }
  rc = check_optimiser(who, hp);
  if (rc != GX_OK) return rc;
  rc = upload_adam_table(h, hp, E, 0);
  if (rc != GX_OK) return rc;
  hd.adam_tab = h->d_adam.as<float2>();
  const float* m0d = m0_dense;
  double* od = out;
  const size_t nout = (size_t)count * E * 2;
  if (space == GX_HOST) {
    GX_CUDA_CHECK(stage_in(h, h->d_m0dense, m0_dense, (size_t)dense, &m0d));
    GX_CUDA_CHECK(stage_out(h->d_offedge, out, nout, &od));
  }
  GX_CUDA_CHECK(cudaMemsetAsync(od, 0, nout * 8, h->stream));
  if (graph) GX_CUDA_CHECK(gx_launch_offedge_graphs(hd, h->plan, h->gb, count, E, m0d, od, h->stream));
  else GX_CUDA_CHECK(gx_launch_offedge(hd, h->plan, count, E, h->d_dense_off.as<int64_t>(), m0d, od, h->stream));
  h->launches += 1;
  if (space == GX_HOST) GX_CUDA_CHECK(stage_back(h, out, (const double*)od, nout));
  GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  return GX_OK;
}

extern "C" {

const char* gx_last_error(void) { return g_err; }
int gx_version(void) { return GX_VERSION; }

void gx_default_hparams(gx_hparams* hp) {
  if (!hp) return;
  hp->num_epochs = 100;
  hp->lr = 0.1f;
  hp->beta1 = 0.9f;
  hp->beta2 = 0.999f;
  hp->eps = 1e-8f;
  hp->coef_size = 0.005f;
  hp->coef_feat_size = 1.0f;
  hp->coef_ent = 1.0f;
  hp->coef_lap = 1.0f;
  hp->mask_act = 0;
  hp->mask_bias = 0;
  hp->init = GX_INIT_M0;
  hp->seed = 0;
  hp->start_step = 0;
  hp->opt = GX_OPT_ADAM;
  hp->opt_scheduler = GX_SCHED_NONE;
  hp->opt_decay_step = 0;
  hp->opt_decay_rate = 1.0f;
  hp->opt_restart = 0;
}

int gx_create(int device, gx_handle** out) {
  if (!out) { gx_set_error("gx_create: out is NULL"); return GX_ERR_INVALID; }
  *out = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    gx_set_error("gx_create: no CUDA device (%s); libgnnx has no CPU fallback",
                 e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    return GX_ERR_CUDA;
  }
  if (device < 0 || device >= ndev) { gx_set_error("gx_create: device %d out of range [0,%d)", device, ndev); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(device));
  cudaDeviceProp prop;
  GX_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {   // sm_90a code loads on compute capability 9.0 only
    gx_set_error("gx_create: device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
    return GX_ERR_CUDA;
  }
  auto h = std::make_unique<gx_handle>();
  h->device = device;
  h->num_sms = prop.multiProcessorCount;
  h->l2_bytes = prop.l2CacheSize;
  std::copy(std::begin(kNodeClasses), std::end(kNodeClasses), h->classes);
  if (const char* env = getenv("GNNX_CLASS_THREADS")) {   // tuning knob: threads per launch class, comma separated
    int v[kNumClasses], k = 0;
    const char* p = env;
    while (*p && k < kNumClasses) { v[k++] = atoi(p); while (*p && *p != ',') ++p; if (*p == ',') ++p; }
    // (a class runs the 256-thread kernel with up to 256 threads or the 512-thread kernel with exactly 512)
    for (int c = 0; c < k; ++c) if (v[c] >= 32 && v[c] % 32 == 0 && (v[c] <= 256 || v[c] == 512)) h->classes[c].threads = v[c];
  }
  if (const char* env = getenv("GNNX_EXCLUSIVE_TOPK")) h->exclusive_topk = atoi(env);
  if (const char* env = getenv("GNNX_HOST_TIMING")) h->host_timing = env[0] == '1';
  if (const char* env = getenv("GNNX_FORCE_STREAM")) h->force_stream = atoi(env) != 0;
  if (const char* env = getenv("GNNX_GANG")) h->gang_override = atoi(env);
  if (const char* env = getenv("GNNX_CLUSTER_SIZE")) { const int v = atoi(env); if (v == 0 || v == 1 || v == 2 || v == 4) h->cluster_size = v; }
  if (const char* env = getenv("GNNX_CLUSTER_COST")) { const long long v = atoll(env); if (v > 0) h->cluster_cost = v; }
  if (const char* env = getenv("GNNX_IEEE_EDGE")) h->ieee_edge = atoi(env) != 0;
  if (const char* env = getenv("GNNX_NODE_GENERIC")) h->node_generic = atoi(env) != 0;
  for (int i = 0; i < kNumClasses; ++i) {
    GX_CUDA_CHECK(cudaStreamCreateWithFlags(&h->side[i], cudaStreamNonBlocking));
    GX_CUDA_CHECK(cudaEventCreate(&h->ev_join[i]));
    GX_CUDA_CHECK(cudaEventCreate(&h->ev_begin[i]));
  }
  GX_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
  GX_CUDA_CHECK(cudaEventCreate(&h->ev_t0));
  GX_CUDA_CHECK(cudaEventCreate(&h->ev_t1));
  *out = h.release();
  return GX_OK;
}

int gx_destroy(gx_handle* h) {
  if (!h) return GX_OK;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  delete h;
  return GX_OK;
}

int gx_set_stream(gx_handle* h, void* cuda_stream) {
  if (!h) { gx_set_error("gx_set_stream: NULL handle"); return GX_ERR_INVALID; }
  h->stream = (cudaStream_t)cuda_stream;
  return GX_OK;
}

int gx_sync(gx_handle* h) {
  if (!h) { gx_set_error("gx_sync: NULL handle"); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  return GX_OK;
}

int64_t gx_launch_count(gx_handle* h) { return h ? h->launches : 0; }

/* debug only (not in gnnx.h): device buffer receiving the shared-memory slab of the first task of each class */
int gx_debug_set_dump(gx_handle* h, float* dev_buf) { if (!h) return GX_ERR_INVALID; h->dbg = dev_buf; return GX_OK; }

/* debug only: IEEE exp/div/sqrt in the edge phase instead of the hardware approximations (parity measurements) */
int gx_debug_ieee_edge(gx_handle* h, int on) { if (!h) return GX_ERR_INVALID; h->ieee_edge = on != 0; return GX_OK; }

int gx_model_forward(gx_handle* h, gx_memspace space, float* pred) {
  if (!h || !pred) { gx_set_error("gx_model_forward: NULL argument"); return GX_ERR_INVALID; }
  if (!h->has_graph || !h->has_model) { gx_set_error("gx_model_forward: call gx_set_model and gx_set_graph_csr first"); return GX_ERR_INVALID; }
  if (h->g.d != h->m.d) { gx_set_error("gx_model_forward: graph feat_dim %d != model input_dim %d", h->g.d, h->m.d); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  const size_t np_ = (size_t)h->g.N * h->m.C;
  const size_t nh = (size_t)h->m.L * h->g.N * gx_var_row_stride(h->m.hid, h->m.emb);   // every layer's rows, 32 / 64 / 128 / 256 floats each
  const size_t npw = h->m.att ? (size_t)h->g.N * gx_round_up(std::max(h->m.d, h->m.hid), 4) : 0;   // attention models: P
  const size_t ne = h->head.k > 0 ? (size_t)h->g.N * (h->m.hid * (h->m.L - 1) + h->m.emb) : 0;   // MLP head: the concatenated rows
  GX_CUDA_CHECK(h->d_fwd.reserve((nh + np_ + npw + ne) * 4));
  float* H = h->d_fwd.as<float>();
  float* pd = space == GX_DEVICE ? pred : H + nh;
  float* P = h->m.att ? H + nh + np_ : nullptr;
  float* E = h->head.k > 0 ? H + nh + np_ + npw : nullptr;
  GX_CUDA_CHECK(gx_launch_model_forward(h->g, h->m, h->head, H, pd, E, P, h->stream));
  h->launches += h->m.L * (h->m.att ? 2 : 1) + 1 + (h->head.k > 0 ? 1 : 0);
  if (space != GX_DEVICE) {
    GX_CUDA_CHECK(cudaMemcpyAsync(pred, pd, np_ * 4, cudaMemcpyDeviceToHost, h->stream));
    GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  }
  return GX_OK;
}
int gx_debug_set_gang(gx_handle* h, int ctas_per_task) { if (!h) return GX_ERR_INVALID; h->gang_override = ctas_per_task; return GX_OK; }
int gx_debug_set_cluster(gx_handle* h, int cluster_size, int64_t min_cost) {
  if (!h || !(cluster_size == 0 || cluster_size == 1 || cluster_size == 2 || cluster_size == 4)) return GX_ERR_INVALID;
  h->cluster_size = cluster_size; h->cluster_cost = min_cost; h->has_plan = false;
  return GX_OK;
}
/* debug only: plan every task into the streaming class (explain_stream.cu) regardless of its size */
int gx_debug_force_stream(gx_handle* h, int on) { if (!h) return GX_ERR_INVALID; h->force_stream = on != 0; h->has_plan = false; return GX_OK; }

int gx_last_explain_ms(gx_handle* h, float* ms) {
  if (!h || !ms) { gx_set_error("gx_last_explain_ms: NULL argument"); return GX_ERR_INVALID; }
  if (!h->timed) { gx_set_error("gx_last_explain_ms: no explain call yet"); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  GX_CUDA_CHECK(cudaEventSynchronize(h->ev_t1));
  GX_CUDA_CHECK(cudaEventElapsedTime(ms, h->ev_t0, h->ev_t1));
  return GX_OK;
}

int gx_last_class_ms(gx_handle* h, float begin_ms[7], float end_ms[7]) {
  if (!h || !begin_ms || !end_ms) { gx_set_error("gx_last_class_ms: NULL argument"); return GX_ERR_INVALID; }
  if (!h->timed) { gx_set_error("gx_last_class_ms: no explain call yet"); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  GX_CUDA_CHECK(cudaEventSynchronize(h->ev_t1));
  for (int c = 0; c < kNumClasses; ++c) {
    begin_ms[c] = end_ms[c] = -1.f;
    if (!h->class_used[c]) continue;
    GX_CUDA_CHECK(cudaEventElapsedTime(&begin_ms[c], h->ev_t0, h->ev_begin[c]));
    GX_CUDA_CHECK(cudaEventElapsedTime(&end_ms[c], h->ev_t0, h->ev_join[c]));
  }
  return GX_OK;
}

int gx_set_model(gx_handle* h, const gx_model_dims* dims, const float* const* conv_w,
                 const float* const* conv_b, const float* pred_w, const float* pred_b) {
  if (!h || !dims || !conv_w || !pred_w || !pred_b) { gx_set_error("gx_set_model: NULL argument"); return GX_ERR_INVALID; }
  const int rc = check_model_dims("gx_set_model", dims);
  if (rc != GX_OK) return rc;
  if (dims->flags & GX_MODEL_ATT) { gx_set_error("gx_set_model: GX_MODEL_ATT models are set with gx_set_model_att (it takes the attention weights)"); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  if (dims->num_layers != 3 || (dims->flags & GX_MODEL_BN) || dims->hidden_dim > 32 || dims->embed_dim > 32 || dims->input_dim >= GX_VAR_WIDE_MIN)
    return set_variant_model(h, "gx_set_model", dims, conv_w, conv_b, nullptr, pred_w, pred_b);
  // The kernels are instantiated for the reference default 20/20 and for 32/32; any other width <= 32 is
  // zero-padded to 32.  Padding is exact: a padded output column is 0*W + 0 = 0, contributes nothing to the
  // row norm, stays 0 through normalise/ReLU, and its pred_model column is 0 (forward and backward).
  const int d = dims->input_dim, hid0 = dims->hidden_dim, emb0 = dims->embed_dim, C = dims->num_classes;
  const bool native = hid0 == 20 && emb0 == 20;
  const int hid = native ? 20 : 32, emb = native ? 20 : 32;
  const int in0[3] = {d, hid0, hid0}, out0[3] = {hid0, hid0, emb0};
  const int in_dim[3] = {d, hid, hid}, out_dim[3] = {hid, hid, emb};
  const int PD0 = 2 * hid0 + emb0, PD = 2 * hid + emb;
  std::vector<float> host;
  size_t offW[3], offWt[3], offb[3], offWp, offbp;
  auto al4 = [&]() { while (host.size() % 4) host.push_back(0.f); };
  for (int l = 0; l < 3; ++l) {
    if (!conv_w[l]) { gx_set_error("gx_set_model: conv_w[%d] is NULL", l); return GX_ERR_INVALID; }
    auto Wat = [&](int f, int c) -> float { return (f < in0[l] && c < out0[l]) ? conv_w[l][(size_t)f * out0[l] + c] : 0.f; };
    al4(); offW[l] = host.size();
    for (int f = 0; f < in_dim[l]; ++f) for (int c = 0; c < out_dim[l]; ++c) host.push_back(Wat(f, c));
    al4(); offWt[l] = host.size();
    for (int c = 0; c < out_dim[l]; ++c) for (int f = 0; f < in_dim[l]; ++f) host.push_back(Wat(f, c));
    al4(); offb[l] = host.size();
    for (int c = 0; c < out_dim[l]; ++c) host.push_back((conv_b && conv_b[l] && c < out0[l]) ? conv_b[l][c] : 0.f);
  }
  al4(); offWp = host.size();
  for (int c = 0; c < C; ++c)
    for (int k = 0; k < PD; ++k) {
      const int part = k / hid >= 2 ? 2 : k / hid, within = k - part * hid;     // padded column -> (layer, feature)
      const int w0 = part == 2 ? emb0 : hid0;
      host.push_back(within < w0 ? pred_w[(size_t)c * PD0 + part * hid0 + within] : 0.f);
    }
  al4(); offbp = host.size();
  host.insert(host.end(), pred_b, pred_b + C);
  GX_CUDA_CHECK(h->m_buf.reserve(host.size() * 4));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->m_buf.p, host.data(), host.size() * 4, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  float* b = h->m_buf.as<float>();
  h->m = GxModelDev{};
  h->m.d = d; h->m.hid = hid; h->m.emb = emb; h->m.C = C; h->m.L = 3;
  for (int l = 0; l < 3; ++l) { h->m.W[l] = b + offW[l]; h->m.Wt[l] = b + offWt[l]; h->m.b[l] = b + offb[l]; }
  h->m.Wp = b + offWp;
  h->m.bp = b + offbp;
  h->head = GxHeadDev{};
  h->has_model = true;
  h->has_plan = false;
  h->has_gplan = false;   // a graph plan's shared-memory footprints were computed for the previous model
  return GX_OK;
}

int gx_set_model_att(gx_handle* h, const gx_model_dims* dims, const float* const* conv_w, const float* const* conv_b,
                     const float* const* att_w, const float* pred_w, const float* pred_b) {
  if (!h || !dims || !conv_w || !att_w || !pred_w || !pred_b) { gx_set_error("gx_set_model_att: NULL argument"); return GX_ERR_INVALID; }
  const int rc = check_model_dims("gx_set_model_att", dims);
  if (rc != GX_OK) return rc;
  if (dims->input_dim >= GX_VAR_WIDE_MIN) {
    gx_set_error("gx_set_model_att: input_dim=%d; attention models are built for inputs up to 128 wide (layer 1's attention matrix is input_dim x input_dim)", dims->input_dim);
    return GX_ERR_UNSUPPORTED;
  }
  if (dims->hidden_dim > 128 || dims->embed_dim > 128) {
    gx_set_error("gx_set_model_att: hidden_dim=%d output_dim=%d; attention models are built for widths up to 128 (widths above 128 run the "
                 "variant kernel's row-block path, which has no attention layers)", dims->hidden_dim, dims->embed_dim);
    return GX_ERR_UNSUPPORTED;
  }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  return set_variant_model(h, "gx_set_model_att", dims, conv_w, conv_b, att_w, pred_w, pred_b);
}

int gx_set_model_head(gx_handle* h, const gx_model_dims* dims, const float* const* conv_w, const float* const* conv_b,
                      const float* const* att_w, int32_t head_layers, const int32_t* head_widths, const float* const* head_w,
                      const float* const* head_b) {
  const char* who = "gx_set_model_head";
  if (!h || !dims || !conv_w || !head_widths || !head_w || !head_b) { gx_set_error("%s: NULL argument", who); return GX_ERR_INVALID; }
  const int rc = check_model_dims(who, dims);
  if (rc != GX_OK) return rc;
  if (head_layers < 1 || head_layers > GX_MAX_HEAD_LAYERS) {
    gx_set_error("%s: head_layers=%d outside [1,%d] (GX_MAX_HEAD_LAYERS; a model without hidden head layers is set with gx_set_model)", who,
                 head_layers, GX_MAX_HEAD_LAYERS);
    return GX_ERR_UNSUPPORTED;
  }
  GxHeadDev head{};
  head.k = head_layers;
  for (int j = 0; j < head_layers; ++j) {
    if (head_widths[j] < 1 || head_widths[j] > GX_MAX_WIDTH) {
      gx_set_error("%s: head_widths[%d]=%d outside [1,%d] (GX_MAX_WIDTH)", who, j, head_widths[j], GX_MAX_WIDTH);
      return GX_ERR_UNSUPPORTED;
    }
    head.w[j] = head_widths[j];
  }
  const bool att = att_w != nullptr;
  if ((dims->flags & GX_MODEL_ATT) && !att) { gx_set_error("%s: GX_MODEL_ATT without att_w", who); return GX_ERR_INVALID; }
  if (att && (dims->input_dim >= GX_VAR_WIDE_MIN || dims->hidden_dim > 128 || dims->embed_dim > 128)) {
    gx_set_error("%s: input_dim=%d hidden_dim=%d output_dim=%d; attention models are built for inputs and widths up to 128", who, dims->input_dim,
                 dims->hidden_dim, dims->embed_dim);
    return GX_ERR_UNSUPPORTED;
  }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  return set_variant_model(h, who, dims, conv_w, conv_b, att_w, nullptr, nullptr, head, head_w, head_b);
}

int gx_set_graph_csr(gx_handle* h, int64_t N, const int32_t* rowptr, const int32_t* col,
                     const float* feat, int32_t d, const int32_t* label, const int32_t* pred_label) {
  if (!h || !rowptr || !col || !feat || !pred_label) { gx_set_error("gx_set_graph_csr: NULL argument"); return GX_ERR_INVALID; }
  if (N < 1 || N > 0x7fffffff - 64) { gx_set_error("gx_set_graph_csr: num_nodes out of range"); return GX_ERR_INVALID; }
  if (rowptr[0] != 0) { gx_set_error("gx_set_graph_csr: rowptr[0] != 0"); return GX_ERR_INVALID; }
  const int64_t nnz = rowptr[N];
  for (int64_t i = 0; i < N; ++i) {
    if (rowptr[i + 1] < rowptr[i]) { gx_set_error("gx_set_graph_csr: rowptr not monotone at %lld", (long long)i); return GX_ERR_INVALID; }
    for (int64_t e = rowptr[i]; e < rowptr[i + 1]; ++e) {
      if (col[e] < 0 || col[e] >= N) { gx_set_error("gx_set_graph_csr: col out of range in row %lld", (long long)i); return GX_ERR_INVALID; }
      if (e > rowptr[i] && col[e] <= col[e - 1]) { gx_set_error("gx_set_graph_csr: row %lld columns not strictly ascending", (long long)i); return GX_ERR_INVALID; }
    }
  }
  // symmetric pattern (the reference's datasets are undirected 0/1 adjacency)
  for (int64_t i = 0; i < N; ++i)
    for (int64_t e = rowptr[i]; e < rowptr[i + 1]; ++e) {
      const int32_t j = col[e];
      if (!std::binary_search(col + rowptr[j], col + rowptr[j + 1], (int32_t)i)) {
        gx_set_error("gx_set_graph_csr: adjacency not symmetric: (%lld,%d) present, (%d,%lld) absent", (long long)i, j, j, (long long)i);
        return GX_ERR_UNSUPPORTED;
      }
    }
  h->has_label = label != nullptr;
  h->label_min = h->label_max = label ? label[0] : 0;
  h->pred_min = h->pred_max = pred_label[0];
  for (int64_t i = 0; i < N; ++i) {
    if (label) { h->label_min = std::min(h->label_min, label[i]); h->label_max = std::max(h->label_max, label[i]); }
    h->pred_min = std::min(h->pred_min, pred_label[i]); h->pred_max = std::max(h->pred_max, pred_label[i]);
  }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  GX_CUDA_CHECK(h->g_rowptr.reserve((size_t)(N + 1) * 4));
  GX_CUDA_CHECK(h->g_col.reserve((size_t)std::max<int64_t>(nnz, 1) * 4));
  GX_CUDA_CHECK(h->g_feat.reserve((size_t)N * d * 4));
  GX_CUDA_CHECK(h->g_label.reserve((size_t)N * 4));
  GX_CUDA_CHECK(h->g_pred.reserve((size_t)N * 4));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->g_rowptr.p, rowptr, (size_t)(N + 1) * 4, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->g_col.p, col, (size_t)nnz * 4, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->g_feat.p, feat, (size_t)N * d * 4, cudaMemcpyHostToDevice, h->stream));
  if (label) GX_CUDA_CHECK(cudaMemcpyAsync(h->g_label.p, label, (size_t)N * 4, cudaMemcpyHostToDevice, h->stream));
  else GX_CUDA_CHECK(cudaMemsetAsync(h->g_label.p, 0, (size_t)N * 4, h->stream));
  GX_CUDA_CHECK(cudaMemcpyAsync(h->g_pred.p, pred_label, (size_t)N * 4, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  h->g.N = N; h->g.nnz = (int32_t)nnz;
  h->g.rowptr = h->g_rowptr.as<int32_t>(); h->g.col = h->g_col.as<int32_t>();
  h->g.feat = h->g_feat.as<float>(); h->g.d = d;
  h->g.label = h->g_label.as<int32_t>(); h->g.pred_label = h->g_pred.as<int32_t>();
  h->has_graph = true;
  h->has_plan = false;
  h->ws.slots = 0;
  return GX_OK;
}

int gx_offedge_regularisers(gx_handle* h, const gx_hparams* hp, gx_memspace space, const float* m0_dense, double* out) {
  return offedge_impl(h, false, hp, space, m0_dense, out);
}

int gx_offedge_regularisers_graphs(gx_handle* h, const gx_hparams* hp, gx_memspace space, const float* m0_dense, double* out) {
  return offedge_impl(h, true, hp, space, m0_dense, out);
}

int gx_comm_unique_id(char id[128]) {
  if (!id) { gx_set_error("gx_comm_unique_id: NULL argument"); return GX_ERR_INVALID; }
  return gx_comm_impl_unique_id(id);
}

int gx_comm_init(gx_handle* h, int32_t world, int32_t rank, const char id[128]) {
  if (!h || !id) { gx_set_error("gx_comm_init: NULL argument"); return GX_ERR_INVALID; }
  if (world < 1 || rank < 0 || rank >= world) { gx_set_error("gx_comm_init: rank %d outside [0,%d)", rank, world); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  gx_comm_impl_destroy(h->comm);
  h->comm = nullptr;
  return gx_comm_impl_init(&h->comm, world, rank, id);
}

int gx_comm_destroy(gx_handle* h) {
  if (!h) return GX_OK;
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream);
  gx_comm_impl_destroy(h->comm);
  h->comm = nullptr;
  return GX_OK;
}

int gx_allgather_masks(gx_handle* h, const float* local_dev, int64_t local_floats, int64_t slot_floats, float* gathered_dev) {
  if (!h || !gathered_dev || (local_floats > 0 && !local_dev)) { gx_set_error("gx_allgather_masks: NULL argument"); return GX_ERR_INVALID; }
  if (!h->comm) { gx_set_error("gx_allgather_masks: no communicator (call gx_comm_init)"); return GX_ERR_INVALID; }
  if (local_floats < 0 || slot_floats < local_floats || slot_floats < 1) { gx_set_error("gx_allgather_masks: need 0 <= local_floats <= slot_floats"); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  // the send slot: this rank's values, zero padded to the common slot size (in place inside the receive buffer: NCCL's in-place all-gather)
  float* mine = gathered_dev + (int64_t)gx_comm_impl_rank(h->comm) * slot_floats;
  if (local_floats > 0 && mine != local_dev)
    GX_CUDA_CHECK(cudaMemcpyAsync(mine, local_dev, (size_t)local_floats * 4, cudaMemcpyDeviceToDevice, h->stream));
  if (slot_floats > local_floats)
    GX_CUDA_CHECK(cudaMemsetAsync(mine + local_floats, 0, (size_t)(slot_floats - local_floats) * 4, h->stream));
  return gx_comm_impl_allgather(h->comm, mine, gathered_dev, (size_t)slot_floats, h->stream);
}

int gx_unshard_masks(gx_handle* h, const float* gathered_dev, int32_t items, const int64_t* src_off, const int64_t* dst_off,
                     const int32_t* sizes, float* out_dev) {
  if (!h || !gathered_dev || !src_off || !dst_off || !sizes || !out_dev) { gx_set_error("gx_unshard_masks: NULL argument"); return GX_ERR_INVALID; }
  if (items <= 0) return GX_OK;
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  const size_t b64 = (size_t)items * 8, b32 = (size_t)items * 4;
  GX_CUDA_CHECK(h->d_us.reserve(2 * b64 + b32));
  char* b = h->d_us.as<char>();
  GX_CUDA_CHECK(cudaMemcpyAsync(b, src_off, b64, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(cudaMemcpyAsync(b + b64, dst_off, b64, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(cudaMemcpyAsync(b + 2 * b64, sizes, b32, cudaMemcpyHostToDevice, h->stream));
  GX_CUDA_CHECK(gx_launch_unshard(gathered_dev, items, (const int64_t*)b, (const int64_t*)(b + b64), (const int32_t*)(b + 2 * b64), out_dev, h->stream));
  h->launches += 1;
  return GX_OK;
}

int gx_denoise_topk(gx_handle* h, gx_memspace space, const float* edge_mask, int32_t threshold_num, int32_t cap,
                    float* out_threshold, int32_t* out_count, int32_t* out_slots, float* out_vals) {
  if (!h || !edge_mask || !out_threshold || !out_count || !out_slots) { gx_set_error("gx_denoise_topk: NULL argument"); return GX_ERR_INVALID; }
  if (!h->has_plan) { gx_set_error("gx_denoise_topk: no plan (call gx_plan_nodes)"); return GX_ERR_INVALID; }
  if (threshold_num < 1 || cap < 1) { gx_set_error("gx_denoise_topk: threshold_num and cap must be >= 1"); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  const size_t count = (size_t)h->count, nslots = count * cap;
  const float* em = edge_mask;
  float* thr = out_threshold; int32_t* cnt = out_count; int32_t* slots = out_slots; float* vals = out_vals;
  if (space == GX_HOST) {
    GX_CUDA_CHECK(stage_in(h, h->d_out, edge_mask, (size_t)h->total_e, &em));
    GX_CUDA_CHECK(stage_out(h->d_dn_thr, out_threshold, count, &thr));
    GX_CUDA_CHECK(stage_out(h->d_dn_cnt, out_count, count, &cnt));
    GX_CUDA_CHECK(stage_out(h->d_dn_slots, out_slots, nslots, &slots));
    GX_CUDA_CHECK(stage_out(h->d_dn_vals, out_vals, nslots, &vals));
  }
  GX_CUDA_CHECK(cudaMemsetAsync(slots, 0xFF, nslots * 4, h->stream));   // unused entries read as -1
  if (vals) GX_CUDA_CHECK(cudaMemsetAsync(vals, 0, nslots * 4, h->stream));   // and their values as 0, not a reused buffer's contents
  GX_CUDA_CHECK(gx_launch_denoise_topk(h->plan, (int)count, em, 2 * threshold_num, cap, thr, cnt, slots, vals, h->stream));
  h->launches += 1;
  if (space == GX_HOST) {
    GX_CUDA_CHECK(stage_back(h, out_threshold, (const float*)thr, count));
    GX_CUDA_CHECK(stage_back(h, out_count, (const int32_t*)cnt, count));
    GX_CUDA_CHECK(stage_back(h, out_slots, (const int32_t*)slots, nslots));
    GX_CUDA_CHECK(stage_back(h, out_vals, (const float*)vals, nslots));
    GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  }
  return GX_OK;
}

int gx_denoise_topk_edges(gx_handle* h, gx_memspace space, const float* edge_mask, int32_t threshold_num, int32_t cap,
                          float* out_threshold, int32_t* out_count, int32_t* out_uv, float* out_vals) {
  if (!h || !edge_mask || !out_threshold || !out_count || !out_uv) { gx_set_error("gx_denoise_topk_edges: NULL argument"); return GX_ERR_INVALID; }
  if (!h->has_plan) { gx_set_error("gx_denoise_topk_edges: no plan (call gx_plan_nodes)"); return GX_ERR_INVALID; }
  if (threshold_num < 1 || cap < 1) { gx_set_error("gx_denoise_topk_edges: threshold_num and cap must be >= 1"); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  const size_t count = (size_t)h->count, nslots = count * cap;
  const float* em = edge_mask;
  float* thr = out_threshold; int32_t* cnt = out_count; int32_t* uv = out_uv; float* vals = out_vals;
  if (space == GX_HOST) {
    GX_CUDA_CHECK(stage_in(h, h->d_out, edge_mask, (size_t)h->total_e, &em));
    GX_CUDA_CHECK(stage_out(h->d_dn_thr, out_threshold, count, &thr));
    GX_CUDA_CHECK(stage_out(h->d_dn_cnt, out_count, count, &cnt));
    GX_CUDA_CHECK(stage_out(h->d_dn_slots, out_uv, 2 * nslots, &uv));
    GX_CUDA_CHECK(stage_out(h->d_dn_vals, out_vals, nslots, &vals));
  }
  GX_CUDA_CHECK(cudaMemsetAsync(uv, 0xFF, 2 * nslots * 4, h->stream));   // unused pairs read as (-1, -1)
  if (vals) GX_CUDA_CHECK(cudaMemsetAsync(vals, 0, nslots * 4, h->stream));
  GX_CUDA_CHECK(gx_launch_denoise_topk_edges(h->plan, (int)count, em, 2 * threshold_num, cap, thr, cnt, uv, vals, h->stream));
  h->launches += 1;
  if (space == GX_HOST) {
    GX_CUDA_CHECK(stage_back(h, out_threshold, (const float*)thr, count));
    GX_CUDA_CHECK(stage_back(h, out_count, (const int32_t*)cnt, count));
    GX_CUDA_CHECK(stage_back(h, out_uv, (const int32_t*)uv, 2 * nslots));
    GX_CUDA_CHECK(stage_back(h, out_vals, (const float*)vals, nslots));
    GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  }
  return GX_OK;
}

int gx_densify(gx_handle* h, gx_memspace space, const float* edge_mask, double* out) {
  if (!h || !edge_mask || !out) { gx_set_error("gx_densify: NULL argument"); return GX_ERR_INVALID; }
  if (!h->has_plan) { gx_set_error("gx_densify: no plan"); return GX_ERR_INVALID; }
  GX_CUDA_CHECK(cudaSetDevice(h->device));
  int64_t dense = 0;
  const int rc = upload_dense_offsets(h, &dense);
  if (rc != GX_OK) return rc;
  const float* em = edge_mask;
  double* o = out;
  if (space == GX_HOST) {
    GX_CUDA_CHECK(stage_in(h, h->d_out, edge_mask, (size_t)h->total_e, &em));
    GX_CUDA_CHECK(stage_out(h->d_dense, out, (size_t)dense, &o));
  }
  GX_CUDA_CHECK(gx_launch_densify(h->plan, h->count, h->d_dense_off.as<int64_t>(), em, o, h->stream));
  h->launches += 1;
  if (space == GX_HOST) {
    GX_CUDA_CHECK(stage_back(h, out, (const double*)o, (size_t)dense));
    GX_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  }
  return GX_OK;
}

}  // extern "C"
