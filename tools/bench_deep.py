"""bench_deep.py -- throughput of Explainer.explain on GCNs with four to seven graph-convolution layers (csrc/explain_var.cu).

    python tools/bench_deep.py [--steps K] [--warmup W]

Workloads, 100 epochs, Philox init, random models (hidden / output 20, biases N(0, 0.4)) with L = 4, 5 and 7 layers: the syn1 graph, all
700 nodes (node mode, n_hops = L), and bench.py's configs[3] stand-in (4337 padded graphs, max_nodes 100, d = 14; graph mode).  Prints
one JSON line: per workload the device time of one gx_explain_nodes / gx_explain_graphs call (CUDA events after warm-up, L2 flushed
between steps, plan outside) as items/s over WINDOWS windows of at least one second each (median, and the min / max as the spread), the
mean k-hop set size of the node workloads, the SM clock sampled during the first window, and the GPU's name and power limit read in the
same run.  Writes nothing.
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
from bench_graph_variants import _gpu_name_power  # noqa: E402
from bench_wide import _device_rate  # noqa: E402

LAYERS = (4, 5, 7)


def _model(rng, d, C_, L, hid=20):
    dims = [d] + [hid] * L
    w = {}
    for l in range(1, L + 1):
        w["W%d" % l] = (rng.normal(size=(dims[l - 1], dims[l])) * 1.5 / np.sqrt(dims[l - 1])).astype(np.float32)
        w["b%d" % l] = (rng.normal(size=dims[l]) * 0.4).astype(np.float32)
    w["Wp"] = (rng.normal(size=(C_, hid * L)) * 0.4).astype(np.float32); w["bp"] = (rng.normal(size=C_) * 0.4).astype(np.float32)
    return w


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
    for L in LAYERS:
        w = _model(rng, g["feat"].shape[1], g["weights"]["Wp"].shape[0], L)
        eng = gnnx.Engine(c.local_rank)
        eng.set_stream(c.stream.cuda_stream)
        eng.set_model(w, num_layers=L)
        eng.set_graph_csr(g["rowptr"], g["col"], g["feat"], g["label"], g["pred_label"])
        plan = eng.plan_nodes(nodes, L)
        mean_n = float(np.mean([plan.n(t) for t in range(plan.count)]))
        r = _device_rate(c, eng, lib.gx_explain_nodes, len(nodes), plan.total_edges, a)
        eng.close()
        r.update(unit="nodes/s", mean_khop_nodes=mean_n,
                 workload="syn1 graph, all %d nodes x %d epochs, %d layers, %d hops" % (len(nodes), NUM_EPOCHS, L, L))
        res["syn1_L%d_nodes" % L] = r
    adj, feat, label, _ = make_graph_batch()
    G = adj.shape[0]
    for L in LAYERS:
        w = _model(rng, feat.shape[2], 2, L)
        eng = gnnx.Engine(c.local_rank)
        eng.set_stream(c.stream.cuda_stream)
        eng.set_model(w, num_layers=L)
        eng.set_graph_batch(adj, feat, label)
        te = int(eng.plan_graphs(np.arange(G, dtype=np.int32))[-1])
        r = _device_rate(c, eng, lib.gx_explain_graphs, G, te, a)
        eng.close()
        r.update(unit="graphs/s", workload="configs[3] stand-in: %d padded graphs (max_nodes %d, d=%d) x %d epochs, %d layers"
                 % (G, adj.shape[1], feat.shape[2], NUM_EPOCHS, L))
        res["graphs_L%d" % L] = r
    print(json.dumps({"metric": "explained items/s, GCNs with 4 to 7 layers, %d epochs, device Philox init" % NUM_EPOCHS,
                      "gpu": name, "power_limit_w": power, "kernel": "explain_var_kernel (L = 4, 5, 7)",
                      "timing": "CUDA events around one gx_explain_nodes / gx_explain_graphs call (plan outside), L2 flushed between steps",
                      "workloads": res}), flush=True)


if __name__ == "__main__":
    main()
