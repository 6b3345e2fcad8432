"""bench_graph_grad.py -- what the gradient baseline costs in graph-classification mode, against the mask optimisation.

    python tools/bench_graph_grad.py [--steps K] [--warmup W]

Workload: bench.py --workload graphs (4337 padded molecule-like graphs, max_nodes 100, d = 14), the default model on the tuned kernel,
all buffers on the device:
  grad      gx_grad_graphs, every graph at the model's own prediction (pred_label = -1): one forward and one backward per graph;
  explain   gx_explain_graphs, GX_INIT_PHILOX, 100 epochs (bench.py's flagship call).
Prints one JSON line: per call the device time (CUDA events around the calls, plan outside, L2 flushed between steps) and graphs/s, the
ratio of the two, with the GPU's name and power limit read in the same run.  Writes nothing.
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
from bench import NUM_EPOCHS, gpu_ctx, make_graph_batch, timed  # noqa: E402
from bench_graph_variants import _gpu_name_power  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
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
    te = int(eng.plan_graphs(np.arange(G, dtype=np.int32))[-1])
    out_dev = torch.empty(te, dtype=torch.float32, device=c.dev)
    labels = np.full(G, -1, np.int32)
    hp = eng.make_hparams(num_epochs=NUM_EPOCHS, init=_abi.GX_INIT_PHILOX, seed=7)
    lib = _abi.lib()
    p = lambda t: C.c_void_p(t.data_ptr())

    def grad():
        _abi.check(lib.gx_grad_graphs(eng._h, _abi.GX_DEVICE, labels.ctypes.data, p(out_dev)))

    def explain():
        _abi.check(lib.gx_explain_graphs(eng._h, C.byref(hp), _abi.GX_DEVICE, None, p(out_dev), None))

    name, power = _gpu_name_power(c.local_rank)
    steps, warmup = max(1, a.steps), max(0, a.warmup)
    res = {}
    for tag, fn in (("grad", grad), ("explain", explain)):
        ms, _, _, _ = timed(c, fn, steps, warmup)
        res[tag] = {"ms_per_step": ms / steps, "graphs_per_s": G * steps / (ms / 1e3)}
    res["grad_over_explain"] = res["grad"]["ms_per_step"] / res["explain"]["ms_per_step"]
    eng.close()
    print(json.dumps({"metric": "device ms per call: gx_grad_graphs vs gx_explain_graphs",
                      "config": {"workload": "bench.py --workload graphs: %d padded graphs (max_nodes %d, d=14)" % (G, n),
                                 "explain": "%d epochs, GX_INIT_PHILOX" % NUM_EPOCHS, "grad": "pred_label = -1", "steps": steps,
                                 "warmup": warmup},
                      "gpu": name, "power_limit_w": power,
                      "timing": "CUDA events around the calls (plan outside), L2 flushed between steps", "results": res}), flush=True)


if __name__ == "__main__":
    main()
