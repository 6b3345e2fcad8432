"""bench_graph_trace.py -- what print_training costs in graph-classification mode.

    python tools/bench_graph_trace.py [--steps K] [--warmup W]

Workload: bench.py's configs[3] stand-in (4337 padded molecule-like graphs, max_nodes 100, d = 14, 100 epochs), the default model on
the tuned kernel, M0 drawn like the reference (torch's CPU generator, one (max_nodes, max_nodes) draw per graph).  Three configurations,
all buffers on the device:
  plain           gx_explain_graphs;
  trace           gx_explain_graphs_ex with the per-epoch trace and softmax rows;
  trace_offedge   the same plus gx_offedge_regularisers_graphs over the dense M0 (G * max_nodes^2 floats, ~173 MB): the printed loss.
Prints one JSON line: per configuration the device time (CUDA events around the calls, plan outside, L2 flushed between steps), with the
GPU's name and power limit.  Writes nothing.
"""
import argparse
import ctypes as C
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import NUM_EPOCHS, gpu_ctx, make_graph_batch, timed  # noqa: E402
from bench_graph_variants import _gpu_name_power  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    a.gpus = 1
    c = gpu_ctx(a)
    import torch
    import gnnx
    from gnnx import _abi
    adj, feat, label, W = make_graph_batch()
    G, n = adj.shape[0], adj.shape[1]
    eng = gnnx.Engine(c.local_rank)
    eng.set_stream(c.stream.cuda_stream)
    eng.set_model(W)
    eng.set_graph_batch(adj, feat, label)
    gids = np.arange(G, dtype=np.int32)
    edge_off = eng.plan_graphs(gids)
    te = int(edge_off[-1])
    torch.manual_seed(0)
    std = torch.nn.init.calculate_gain("relu") * math.sqrt(2.0 / (n + n))
    dense = torch.empty(G, n, n, dtype=torch.float32)
    m0 = np.empty(te, np.float32)
    for g in range(G):
        dense[g].normal_(1.0, std)
        r, cc = eng.graph_rows_cols(g)
        m0[edge_off[g]:edge_off[g + 1]] = dense[g].numpy()[r, cc]
    dense_dev = dense.reshape(-1).to(c.dev)
    m0_dev = torch.from_numpy(m0).to(c.dev)
    out_dev = torch.empty(te, dtype=torch.float32, device=c.dev)
    trace_dev = torch.empty(G * NUM_EPOCHS * _abi.GX_TRACE_COLS, dtype=torch.float32, device=c.dev)
    pred_dev = torch.empty(G * NUM_EPOCHS * W["Wp"].shape[0], dtype=torch.float32, device=c.dev)
    off_dev = torch.empty(G * NUM_EPOCHS * 2, dtype=torch.float64, device=c.dev)
    hp = eng.make_hparams(num_epochs=NUM_EPOCHS)
    lib = _abi.lib()
    io = _abi.GxExplainIo()
    io.m0_edges = m0_dev.data_ptr(); io.edge_mask = out_dev.data_ptr(); io.trace = trace_dev.data_ptr(); io.trace_pred = pred_dev.data_ptr()
    p = lambda t: C.c_void_p(t.data_ptr())

    def plain():
        _abi.check(lib.gx_explain_graphs(eng._h, C.byref(hp), _abi.GX_DEVICE, p(m0_dev), p(out_dev), None))

    def trace():
        _abi.check(lib.gx_explain_graphs_ex(eng._h, C.byref(hp), _abi.GX_DEVICE, C.byref(io)))

    def trace_offedge():
        trace()
        _abi.check(lib.gx_offedge_regularisers_graphs(eng._h, C.byref(hp), _abi.GX_DEVICE, p(dense_dev), p(off_dev)))

    name, power = _gpu_name_power(c.local_rank)
    steps, warmup = max(1, a.steps), max(0, a.warmup)
    res = {}
    for tag, fn in (("plain", plain), ("trace", trace), ("trace_offedge", trace_offedge)):
        ms, _, _, _ = timed(c, fn, steps, warmup)
        res[tag] = {"ms_per_step": ms / steps, "graphs_per_s": G * steps / (ms / 1e3)}
    for tag in ("trace", "trace_offedge"):
        res[tag]["vs_plain"] = res[tag]["ms_per_step"] / res["plain"]["ms_per_step"]
    eng.close()
    print(json.dumps({"metric": "device ms per explain_graphs call, with and without the print_training trace",
                      "config": {"workload": "configs[3] stand-in: %d padded graphs (max_nodes %d, d=14), graph-level mask, %d epochs" % (G, n, NUM_EPOCHS),
                                 "init": "torch (host M0)", "dense_m0_bytes": int(G * n * n * 4), "steps": steps, "warmup": warmup},
                      "gpu": name, "power_limit_w": power,
                      "timing": "CUDA events around the calls (plan outside), L2 flushed between steps", "results": res}), flush=True)


if __name__ == "__main__":
    main()
