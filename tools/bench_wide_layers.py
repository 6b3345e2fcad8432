"""bench_wide_layers.py -- throughput of Explainer.explain on GCNs with hidden / output widths of 256 (csrc/explain_var.cu, row-block path).

    python tools/bench_wide_layers.py [--steps K] [--warmup W]

Workloads, 100 epochs, Philox init, a random 3-layer 256 / 256 model (biases N(0, 0.4)): the syn1 graph, all 700 nodes (node mode,
3 hops), and bench.py's configs[3] stand-in (4337 padded graphs, max_nodes 100, d = 14; graph mode).  Prints one JSON line: per workload
the device time of one gx_explain_nodes / gx_explain_graphs call (CUDA events after warm-up, L2 flushed between steps, plan outside) as
items/s over the windows of tools/bench_wide.py (median, min / max as the spread), the SM clock sampled during the first window, and the
GPU's name and power limit read in the same run.  Writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import NUM_EPOCHS, gpu_ctx, load_syn1, make_graph_batch  # noqa: E402
from bench_deep import _model  # noqa: E402
from bench_graph_variants import _gpu_name_power  # noqa: E402
from bench_wide import _device_rate  # noqa: E402

L, HID = 3, 256


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    a.gpus = 1
    import gnnx
    from gnnx import _abi
    c = gpu_ctx(a)
    name, power = _gpu_name_power(c.local_rank)
    lib = _abi.lib()
    rng = np.random.default_rng(9)
    res = {}
    g = load_syn1()
    nodes = np.arange(g["N"], dtype=np.int32)
    eng = gnnx.Engine(c.local_rank)
    eng.set_stream(c.stream.cuda_stream)
    eng.set_model(_model(rng, g["feat"].shape[1], g["weights"]["Wp"].shape[0], L, HID), num_layers=L)
    eng.set_graph_csr(g["rowptr"], g["col"], g["feat"], g["label"], g["pred_label"])
    plan = eng.plan_nodes(nodes, L)
    r = _device_rate(c, eng, lib.gx_explain_nodes, len(nodes), plan.total_edges, a)
    eng.close()
    r.update(unit="nodes/s", workload="syn1 graph, all %d nodes x %d epochs, %d layers, widths %d / %d" % (len(nodes), NUM_EPOCHS, L, HID, HID))
    res["syn1_nodes"] = r
    adj, feat, label, _ = make_graph_batch()
    G = adj.shape[0]
    eng = gnnx.Engine(c.local_rank)
    eng.set_stream(c.stream.cuda_stream)
    eng.set_model(_model(rng, feat.shape[2], 2, L, HID), num_layers=L)
    eng.set_graph_batch(adj, feat, label)
    te = int(eng.plan_graphs(np.arange(G, dtype=np.int32))[-1])
    r = _device_rate(c, eng, lib.gx_explain_graphs, G, te, a)
    eng.close()
    r.update(unit="graphs/s", workload="configs[3] stand-in: %d padded graphs (max_nodes %d, d=%d) x %d epochs, %d layers, widths %d / %d"
             % (G, adj.shape[1], feat.shape[2], NUM_EPOCHS, L, HID, HID))
    res["graphs"] = r
    print(json.dumps({"metric": "explained items/s, 3-layer GCN with widths 256 / 256, %d epochs, device Philox init" % NUM_EPOCHS,
                      "gpu": name, "power_limit_w": power, "kernel": "explain_var_kernel (row-block path, KW = 8)",
                      "timing": "CUDA events around one gx_explain_nodes / gx_explain_graphs call (plan outside), L2 flushed between steps",
                      "workloads": res}), flush=True)


if __name__ == "__main__":
    main()
