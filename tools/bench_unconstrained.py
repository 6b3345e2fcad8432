"""bench_unconstrained.py -- throughput of Explainer.explain(..., unconstrained=True) on the dense kernel (csrc/explain_dense.cu).

    python tools/bench_unconstrained.py [--steps K] [--warmup W] [--cpu-sample S]

Workloads: syn1, all 700 nodes x 100 epochs (node mode, the fixture's model), and bench.py's configs[3] stand-in (4337 padded
molecule-like graphs, max_nodes 100, d = 14, 100 epochs; graph mode).  Philox init.  Prints one JSON line: per workload the device
time of gx_explain_{nodes,graphs}_unconstrained (CUDA events after warm-up, L2 flushed between steps, plan outside) as items/s,
the GPU's name and power limit, and the line-by-line CPU port's rate (gnnx_oracle.explain_dense_torch, unconstrained=True) on S evenly
spaced items.  Also the time of ONE task near the size limit (a 3-hop subgraph of n = 3769 in a Barabasi-Albert graph, 100 epochs): one CTA
per task, so this is the latency of the largest task a batch can hold.  Writes nothing.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench import NUM_EPOCHS, gpu_ctx, load_syn1, make_ba_csr, make_graph_batch, timed  # noqa: E402
from bench_graph_variants import _gpu_name_power  # noqa: E402


def _device_rate(c, eng, fn, count, total_edges, a, steps=None, warmup=None):
    import torch
    from gnnx import _abi
    out_dev = torch.empty(max(total_edges, 1), dtype=torch.float32, device=c.dev)
    hp = eng.make_hparams(num_epochs=NUM_EPOCHS, init=_abi.GX_INIT_PHILOX, seed=7)

    def step():
        _abi.check(fn(eng._h, C.byref(hp), _abi.GX_DEVICE, None, C.c_void_p(out_dev.data_ptr()), None, None, None))
    steps = max(1, a.steps) if steps is None else steps
    warmup = max(0, a.warmup) if warmup is None else warmup
    ms, _, _, _ = timed(c, step, steps, warmup)
    return {"value": count * steps / (ms / 1e3), "ms_per_step": ms / steps, "steps": steps, "warmup": warmup}


def _cpu_rate(items):
    """items: callables running one item through the CPU port; returns items/s of one process."""
    t0 = time.perf_counter()
    for f in items:
        f()
    return len(items) / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cpu-sample", type=int, default=3)
    a = ap.parse_args()
    a.gpus = 1
    import gnnx
    import gnnx_oracle as O
    from gnnx import _abi
    c = gpu_ctx(a)
    name, power = _gpu_name_power(c.local_rank)
    lib = _abi.lib()
    res = {}
    # ---- node mode: syn1, all nodes
    g = load_syn1()
    eng = gnnx.Engine(c.local_rank)
    eng.set_stream(c.stream.cuda_stream)
    eng.set_model(g["weights"])
    eng.set_graph_csr(g["rowptr"], g["col"], g["feat"], g["label"], g["pred_label"])
    nodes = np.arange(g["N"], dtype=np.int32)
    plan = eng.plan_nodes(nodes, 3)
    n_t = np.diff(plan.node_off)
    r = _device_rate(c, eng, lib.gx_explain_nodes_unconstrained, len(nodes), plan.total_edges, a)
    eng.close()

    def node_item(v):
        idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(g["rowptr"], g["col"], g["feat"], g["label"], int(v), 3)
        A = O.dense_from_csr(srp, scol)
        return lambda: O.explain_dense_torch(A, X, int(lab[idx]), g["pred_label"][nbrs], idx, g["weights"],
                                             O.draw_m0(len(nbrs), seed=int(v)),
                                             hp=O.default_hparams(num_epochs=NUM_EPOCHS), unconstrained=True)
    sample = nodes[np.linspace(0, len(nodes) - 1, a.cpu_sample).astype(int)]
    r.update(unit="nodes/s", workload="syn1, all %d nodes x %d epochs, 3 hops" % (len(nodes), NUM_EPOCHS),
             n_mean=float(n_t.mean()), n_max=int(n_t.max()),
             cpu_port_nodes_per_s=_cpu_rate([node_item(v) for v in sample]), cpu_port_sample=[int(v) for v in sample])
    res["syn1_nodes"] = r
    # ---- graph mode: the configs[3] stand-in
    adj, feat, label, _ = make_graph_batch()
    G, n = adj.shape[0], adj.shape[1]
    rng = np.random.default_rng(11)
    sc = lambda *s_: (rng.normal(size=s_) * 0.4).astype(np.float32)
    d = feat.shape[2]
    W = dict(W1=sc(d, 20), b1=sc(20), W2=sc(20, 20), b2=sc(20), W3=sc(20, 20), b3=sc(20), Wp=sc(2, 60), bp=sc(2))
    eng = gnnx.Engine(c.local_rank)
    eng.set_stream(c.stream.cuda_stream)
    eng.set_model(W)
    eng.set_graph_batch(adj, feat, label)
    gids = np.arange(G, dtype=np.int32)
    te = int(eng.plan_graphs(gids)[-1])
    r = _device_rate(c, eng, lib.gx_explain_graphs_unconstrained, G, te, a)
    eng.close()
    gsample = np.linspace(0, G - 1, a.cpu_sample).astype(int)

    def graph_item(k):
        return lambda: O.explain_dense_torch(adj[k].astype(np.float64), feat[k], int(label[k]), None, 0, W, O.draw_m0(n, seed=k),
                                             hp=O.default_hparams(num_epochs=NUM_EPOCHS), graph_mode=True, unconstrained=True)
    r.update(unit="graphs/s", workload="configs[3] stand-in: %d padded graphs (max_nodes %d, d=%d) x %d epochs, random 3-layer model" % (G, n, d, NUM_EPOCHS),
             cpu_port_graphs_per_s=_cpu_rate([graph_item(int(k)) for k in gsample]), cpu_port_sample=[int(k) for k in gsample])
    res["graphs"] = r
    # ---- one task near the n <= 4096 limit
    rowptr, col = make_ba_csr(20000, 2, 0)
    N = len(rowptr) - 1
    rng = np.random.default_rng(3)
    W = dict(W1=sc(16, 20), b1=sc(20), W2=sc(20, 20), b2=sc(20), W3=sc(20, 20), b3=sc(20), Wp=sc(3, 60), bp=sc(3))
    eng = gnnx.Engine(c.local_rank)
    eng.set_stream(c.stream.cuda_stream)
    eng.set_model(W)
    eng.set_graph_csr(rowptr, col, rng.normal(size=(N, 16)).astype(np.float32), rng.integers(0, 3, N).astype(np.int32),
                      rng.integers(0, 3, N).astype(np.int32))
    plan = eng.plan_nodes([17617], 3)
    r = _device_rate(c, eng, lib.gx_explain_nodes_unconstrained, 1, plan.total_edges, a, steps=1, warmup=1)
    eng.close()
    r.update(unit="nodes/s", workload="one node of BA(20000, 2), 3 hops: n = %d, %d epochs" % (plan.n(0), NUM_EPOCHS))
    res["largest_task"] = r
    print(json.dumps({"metric": "explained items/s, unconstrained=True (dense mask), %d epochs, device Philox init" % NUM_EPOCHS,
                      "gpu": name, "power_limit_w": power, "kernel": "explain_dense_kernel",
                      "timing": "CUDA events around one gx_explain_*_unconstrained call (plan outside), L2 flushed between steps; CPU port: "
                                "one process, torch threads as configured",
                      "workloads": res}), flush=True)


if __name__ == "__main__":
    main()
