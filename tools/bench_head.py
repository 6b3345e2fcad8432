"""bench_head.py -- throughput of Explainer.explain on GCNs with an MLP prediction head (pred_hidden_dims, csrc/explain_var.cu).

    python tools/bench_head.py [--steps K] [--warmup W]

Workloads, 100 epochs, Philox init, random models: a 3-layer --bn 20 / 20 model without and with pred_hidden_dims=[50] (the head's
cost on top of the same variant kernel), and a 7-layer 256 / 256 model with pred_hidden_dims=[256] (the largest first head product,
1792 x 256); each on the syn1 graph, all 700 nodes (node mode, n_hops = L), and on bench.py's configs[3] stand-in (4337 padded graphs,
max_nodes 100, d = 14; graph mode).  Prints a JSON line per finished workload (the 7-layer model takes minutes), then one with the device time of one explain call per workload (bench_wide's
_device_rate: CUDA events after warm-up, L2 flushed between steps, plan outside, median and min / max over its windows) and the GPU's
name and power limit read in the same run.  Writes nothing.
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

# name: (layers, bn, hidden = output width, head widths)
MODELS = {"L3_bn_h20": (3, True, 20, []), "L3_bn_h20_head50": (3, True, 20, [50]), "L7_h256_head256": (7, False, 256, [256])}


def _model(rng, d, C, L, hid, widths):
    dims = [d] + [hid] * L
    w = {}
    for l in range(1, L + 1):
        w["W%d" % l] = (rng.normal(size=(dims[l - 1], dims[l])) * 1.5 / np.sqrt(dims[l - 1])).astype(np.float32)
        w["b%d" % l] = (rng.normal(size=dims[l]) * 0.4).astype(np.float32)
    fan = hid * L
    head = []
    for h in widths:
        head.append(((rng.normal(size=(h, fan)) * 1.5 / np.sqrt(fan)).astype(np.float32), (rng.normal(size=h) * 0.4).astype(np.float32)))
        fan = h
    w["Wp"] = (rng.normal(size=(C, fan)) * 1.5 / np.sqrt(fan)).astype(np.float32)
    w["bp"] = (rng.normal(size=C) * 0.4).astype(np.float32)
    return w, (head or None)


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
    adj, feat, label, _ = make_graph_batch()
    G = adj.shape[0]
    for key, (L, bn, hid, widths) in MODELS.items():
        w, head = _model(rng, g["feat"].shape[1], g["weights"]["Wp"].shape[0], L, hid, widths)
        eng = gnnx.Engine(c.local_rank)
        eng.set_stream(c.stream.cuda_stream)
        eng.set_model(w, num_layers=L, bn=bn, head=head)
        eng.set_graph_csr(g["rowptr"], g["col"], g["feat"], g["label"], g["pred_label"])
        plan = eng.plan_nodes(nodes, L)
        r = _device_rate(c, eng, lib.gx_explain_nodes, len(nodes), plan.total_edges, a)
        eng.close()
        r.update(unit="nodes/s", workload="syn1 graph, all %d nodes x %d epochs, %s, head %s" % (len(nodes), NUM_EPOCHS, key, widths))
        res["syn1_" + key] = r
        print(json.dumps({"partial": "syn1_" + key, "result": r}), flush=True)
        w, head = _model(rng, feat.shape[2], 2, L, hid, widths)
        eng = gnnx.Engine(c.local_rank)
        eng.set_stream(c.stream.cuda_stream)
        eng.set_model(w, num_layers=L, bn=bn, head=head)
        eng.set_graph_batch(adj, feat, label)
        te = int(eng.plan_graphs(np.arange(G, dtype=np.int32))[-1])
        r = _device_rate(c, eng, lib.gx_explain_graphs, G, te, a)
        eng.close()
        r.update(unit="graphs/s", workload="configs[3] stand-in: %d padded graphs (max_nodes %d, d=%d) x %d epochs, %s, head %s"
                 % (G, adj.shape[1], feat.shape[2], NUM_EPOCHS, key, widths))
        res["graphs_" + key] = r
        print(json.dumps({"partial": key, "gpu": name, "power_limit_w": power, "syn1": res["syn1_" + key], "graphs": r}), flush=True)
    print(json.dumps({"metric": "explained items/s, GCNs with an MLP prediction head, %d epochs, device Philox init" % NUM_EPOCHS,
                      "gpu": name, "power_limit_w": power, "kernel": "explain_var_kernel",
                      "timing": "CUDA events around one gx_explain_nodes / gx_explain_graphs call (plan outside), L2 flushed between steps",
                      "workloads": res}), flush=True)


if __name__ == "__main__":
    main()
