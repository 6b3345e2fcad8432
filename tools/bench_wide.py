"""bench_wide.py -- throughput of Explainer.explain on inputs wider than 128 features (the wide path of csrc/explain_var.cu).

    python tools/bench_wide.py [--steps K] [--warmup W]

Workloads, 100 epochs, Philox init, random 3-layer models (widths 20, W1 scaled by 1 / sqrt(d)): the syn1 graph with random features
of width d = 256 and d = 1433, all 700 nodes (node mode, 3 hops), and the 12-graph stand-in of tests/golden/graphs_golden.npz with
one-hot features over 190 labels (graph mode).  Prints one JSON line: per workload the device time of one gx_explain_nodes /
gx_explain_graphs call (CUDA events after warm-up, L2 flushed between steps, plan outside) as items/s over WINDOWS windows of at least
one second each (median, and the min / max as the spread), the SM clock sampled during the first window, the CPU port's rate on a few
items of the same workload (gnnx_oracle.explain_dense_torch, fp32 torch, one process), and the GPU's name and power limit.  Writes nothing.
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
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench import NUM_EPOCHS, ClockSampler, gpu_ctx, load_syn1, timed  # noqa: E402
from bench_graph_variants import _gpu_name_power  # noqa: E402


def _model(rng, d, C_, L=3, hid=20):
    w = {}
    for l in range(1, L + 1):
        win = d if l == 1 else hid
        w["W%d" % l] = (rng.normal(size=(win, hid)) * (2.0 / np.sqrt(d) if l == 1 else 0.5)).astype(np.float32)
        w["b%d" % l] = (rng.normal(size=hid) * 0.4).astype(np.float32)
    w["Wp"] = (rng.normal(size=(C_, hid * L)) * 0.4).astype(np.float32); w["bp"] = (rng.normal(size=C_) * 0.4).astype(np.float32)
    return w


WINDOWS = 3


def _device_rate(c, eng, fn, count, total_edges, a):
    import time
    import torch
    from gnnx import _abi
    out_dev = torch.empty(max(total_edges, 1), dtype=torch.float32, device=c.dev)
    hp = eng.make_hparams(num_epochs=NUM_EPOCHS, init=_abi.GX_INIT_PHILOX, seed=7)

    def step():
        _abi.check(fn(eng._h, C.byref(hp), _abi.GX_DEVICE, None, C.c_void_p(out_dev.data_ptr()), None))
    warmup = max(1, a.warmup)
    t0 = time.perf_counter()
    for _ in range(warmup):
        step()
    torch.cuda.synchronize(c.dev)
    est = (time.perf_counter() - t0) / warmup
    steps = max(a.steps, int(np.ceil(1.0 / max(est, 1e-4))))   # at least one second of work per window
    per_step, clocks = [], None
    for w in range(WINDOWS):
        sampler = ClockSampler(c.local_rank) if w == 0 else None
        ms, _, _, cl = timed(c, step, steps, 0, sampler=sampler)
        per_step.append(ms / steps)
        clocks = cl if w == 0 else clocks
    med = float(np.median(per_step))
    return {"value": count / (med / 1e3), "ms_per_step": med, "ms_per_step_min_max": [min(per_step), max(per_step)],
            "steps_per_window": steps, "windows": WINDOWS, "warmup": warmup, "clocks": clocks}


def _port_rate(items):
    """items: callables, one explanation each on the CPU port; -> items/s."""
    import time
    t0 = time.perf_counter()
    for f in items:
        f()
    return len(items) / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--port-items", type=int, default=3, help="items per workload timed on the CPU port (0: skip)")
    a = ap.parse_args()
    a.gpus = 1
    import gnnx
    import gnnx_oracle as O
    from gnnx import _abi
    c = gpu_ctx(a)
    name, power = _gpu_name_power(c.local_rank)
    lib = _abi.lib()
    rng = np.random.default_rng(5)
    res = {}
    g = load_syn1()
    hp = O.default_hparams(num_epochs=NUM_EPOCHS)
    for d in (256, 1433):
        feat = rng.normal(size=(g["N"], d)).astype(np.float32)
        w = _model(rng, d, g["weights"]["Wp"].shape[0])
        eng = gnnx.Engine(c.local_rank)
        eng.set_stream(c.stream.cuda_stream)
        eng.set_model(w, num_layers=3)
        eng.set_graph_csr(g["rowptr"], g["col"], feat, g["label"], g["pred_label"])
        nodes = np.arange(g["N"], dtype=np.int32)
        plan = eng.plan_nodes(nodes, 3)
        r = _device_rate(c, eng, lib.gx_explain_nodes, len(nodes), plan.total_edges, a)
        eng.close()
        r.update(unit="nodes/s", workload="syn1 graph, random features d=%d, all %d nodes x %d epochs, 3 hops" % (d, len(nodes), NUM_EPOCHS))
        items = []
        for node in range(0, g["N"], max(1, g["N"] // max(a.port_items, 1)))[:a.port_items]:
            idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(g["rowptr"], g["col"], feat, g["label"], node, 3)
            A = O.dense_from_csr(srp, scol)
            M0 = O.draw_m0(len(nbrs), seed=node)
            items.append(lambda A=A, sfeat=sfeat, gt=slabel[idx], pl=g["pred_label"][nbrs], idx=idx, M0=M0:
                         O.explain_dense_torch(A, sfeat, gt, pl, idx, w, M0, hp))
        r["cpu_port"] = {"value": _port_rate(items), "unit": "nodes/s", "items": len(items)} if items else None
        res["syn1_d%d_nodes" % d] = r
    gg = np.load(os.path.join(ROOT, "tests", "golden", "graphs_golden.npz"))
    adj = gg["adj"]
    d = 190
    feat = (np.eye(d, dtype=np.float32)[rng.integers(0, d, size=adj.shape[:2])] * (adj.sum(2, keepdims=True) > 0)).astype(np.float32)
    w = _model(rng, d, 2)
    label = np.asarray(gg["label"]) % 2
    eng = gnnx.Engine(c.local_rank)
    eng.set_stream(c.stream.cuda_stream)
    eng.set_model(w, num_layers=3)
    eng.set_graph_batch(adj, feat, label)
    G = adj.shape[0]
    te = int(eng.plan_graphs(np.arange(G, dtype=np.int32))[-1])
    r = _device_rate(c, eng, lib.gx_explain_graphs, G, te, a)
    eng.close()
    r.update(unit="graphs/s", workload="12-graph stand-in (max_nodes %d), one-hot features d=%d, x %d epochs" % (adj.shape[1], d, NUM_EPOCHS))
    items = [lambda gi=gi: O.explain_dense_torch(np.asarray(adj[gi], np.float64), feat[gi], int(label[gi]), None, 0, w,
                                            O.draw_m0(adj.shape[1], seed=gi), hp, graph_mode=True) for gi in range(min(a.port_items, G))]
    r["cpu_port"] = {"value": _port_rate(items), "unit": "graphs/s", "items": len(items)} if items else None
    res["graphs_d190"] = r
    print(json.dumps({"metric": "explained items/s, inputs wider than 128 features, %d epochs, device Philox init" % NUM_EPOCHS,
                      "gpu": name, "power_limit_w": power, "kernel": "explain_var_kernel<..., kWide = true>",
                      "timing": "CUDA events around one gx_explain_nodes / gx_explain_graphs call (plan outside), L2 flushed between steps",
                      "workloads": res}), flush=True)


if __name__ == "__main__":
    main()
