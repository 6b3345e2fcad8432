"""bench_att.py -- throughput of Explainer.explain on attention models (--method att) in the model-variant kernel (csrc/explain_var.cu).

    python tools/bench_att.py [--steps K] [--warmup W]

Workloads, 100 epochs, Philox init, random attention models (3 layers, widths 20, biases N(0, 0.16)): syn1, all 700 nodes (node
mode, 3 hops), and bench.py's configs[3] stand-in (4337 padded molecule-like graphs, max_nodes 100, d = 14; graph mode).  Prints
one JSON line: per workload the device time of one gx_explain_nodes / gx_explain_graphs call (CUDA events after warm-up, L2 flushed
between steps, plan outside) as items/s, and the GPU's name and power limit.  Writes nothing.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import NUM_EPOCHS, gpu_ctx, load_syn1, make_graph_batch, timed  # noqa: E402
from bench_graph_variants import _gpu_name_power  # noqa: E402


def _att_model(rng, d, C_, L=3, hid=20):
    sc = lambda *s_: (rng.normal(size=s_) * 0.4).astype(np.float32)
    w, att = {}, []
    for l in range(1, L + 1):
        win = d if l == 1 else hid
        w["W%d" % l] = sc(win, hid); w["b%d" % l] = sc(hid)
        att.append((rng.normal(size=(win, win)) / np.sqrt(win)).astype(np.float32))
    w["Wp"] = sc(C_, hid * L); w["bp"] = sc(C_)
    return w, att


def _device_rate(c, eng, fn, count, total_edges, a):
    import torch
    from gnnx import _abi
    out_dev = torch.empty(max(total_edges, 1), dtype=torch.float32, device=c.dev)
    hp = eng.make_hparams(num_epochs=NUM_EPOCHS, init=_abi.GX_INIT_PHILOX, seed=7)

    def step():
        _abi.check(fn(eng._h, C.byref(hp), _abi.GX_DEVICE, None, C.c_void_p(out_dev.data_ptr()), None))
    steps, warmup = max(1, a.steps), max(0, a.warmup)
    ms, _, _, _ = timed(c, step, steps, warmup)
    return {"value": count * steps / (ms / 1e3), "ms_per_step": ms / steps, "steps": steps, "warmup": warmup}


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
    rng = np.random.default_rng(5)
    res = {}
    # ---- node mode: syn1-shaped, all nodes
    g = load_syn1()
    w, att = _att_model(rng, g["feat"].shape[1], g["weights"]["Wp"].shape[0])
    eng = gnnx.Engine(c.local_rank)
    eng.set_stream(c.stream.cuda_stream)
    eng.set_model(w, num_layers=3, att=att)
    eng.set_graph_csr(g["rowptr"], g["col"], g["feat"], g["label"], g["pred_label"])
    nodes = np.arange(g["N"], dtype=np.int32)
    plan = eng.plan_nodes(nodes, 3)
    r = _device_rate(c, eng, lib.gx_explain_nodes, len(nodes), plan.total_edges, a)
    eng.close()
    r.update(unit="nodes/s", workload="syn1 graph, all %d nodes x %d epochs, 3 hops, random 3-layer attention model" % (len(nodes), NUM_EPOCHS))
    res["syn1_nodes"] = r
    # ---- graph mode: the configs[3] stand-in
    adj, feat, label, _ = make_graph_batch()
    G, n, d = adj.shape[0], adj.shape[1], feat.shape[2]
    w, att = _att_model(rng, d, 2)
    eng = gnnx.Engine(c.local_rank)
    eng.set_stream(c.stream.cuda_stream)
    eng.set_model(w, num_layers=3, att=att)
    eng.set_graph_batch(adj, feat, label)
    te = int(eng.plan_graphs(np.arange(G, dtype=np.int32))[-1])
    r = _device_rate(c, eng, lib.gx_explain_graphs, G, te, a)
    eng.close()
    r.update(unit="graphs/s", workload="configs[3] stand-in: %d padded graphs (max_nodes %d, d=%d) x %d epochs, random 3-layer attention model"
             % (G, n, d, NUM_EPOCHS))
    res["graphs"] = r
    print(json.dumps({"metric": "explained items/s, attention models (--method att), %d epochs, device Philox init" % NUM_EPOCHS,
                      "gpu": name, "power_limit_w": power, "kernel": "explain_var_kernel<..., kAtt = true>",
                      "timing": "CUDA events around one gx_explain_nodes / gx_explain_graphs call (plan outside), L2 flushed between steps",
                      "workloads": res}), flush=True)


if __name__ == "__main__":
    main()
