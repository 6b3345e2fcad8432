"""bench_graph_variants.py -- graphs/s of graph-classification mode with model variants (csrc/explain_var.cu, graph mode).

    python tools/bench_graph_variants.py [--steps K] [--warmup W]

Workload: bench.py's configs[3] stand-in (4337 padded molecule-like graphs, max_nodes 100, d = 14, 100 epochs, Philox init),
explained with a 3-layer --bn model and with a 4-layer model (hidden / output 20, random weights).  Prints one JSON line: per
model the device time of gx_explain_graphs (CUDA events, L2 flushed between steps) as graphs/s, with the GPU's name and
power limit.  Writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import NUM_EPOCHS, gpu_ctx, make_graph_batch, timed  # noqa: E402


def _gpu_name_power(index):
    """(name, enforced power limit in W) of the GPU, from a read-only nvidia-smi query; None where it is unavailable."""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        name, lim = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return name, float(lim)
    except Exception:
        import torch
        return torch.cuda.get_device_name(index), None


def bench_graph_variants(a, c, adj, feat, label):
    """The same stand-in explained with model variants (explain_var.cu): a 3-layer --bn model and a 4-layer model (hidden /
    output 20, random weights), Philox init, 100 epochs.  Device time of the explain call (CUDA events), graphs/s."""
    import ctypes as C
    import gnnx
    from gnnx import _abi
    rng = np.random.default_rng(11)
    sc = lambda *s_: (rng.normal(size=s_) * 0.4).astype(np.float32)
    d, Cn, G = feat.shape[2], 2, adj.shape[0]
    name, power = _gpu_name_power(c.local_rank)
    steps, warmup = max(1, a.steps), max(0, a.warmup)
    out = {}
    for tag, L, bn in (("bn_3layer", 3, True), ("plain_4layer", 4, False)):
        dims = [d] + [20] * L
        W = {}
        for l in range(1, L + 1):
            W["W%d" % l] = sc(dims[l - 1], dims[l]); W["b%d" % l] = sc(dims[l])
        W["Wp"], W["bp"] = sc(Cn, 20 * L), sc(Cn)
        eng = gnnx.Engine(c.local_rank)
        eng.set_stream(c.stream.cuda_stream)
        eng.set_model(W, num_layers=L, bn=bn)
        eng.set_graph_batch(adj, feat, label)
        gids = np.arange(G, dtype=np.int32)
        te = int(eng.plan_graphs(gids)[-1])
        import torch
        out_dev = torch.empty(te, dtype=torch.float32, device=c.dev)
        hp = eng.make_hparams(num_epochs=NUM_EPOCHS, init=_abi.GX_INIT_PHILOX, seed=7)
        lib = _abi.lib()

        def step():
            _abi.check(lib.gx_explain_graphs(eng._h, C.byref(hp), _abi.GX_DEVICE, None, C.c_void_p(out_dev.data_ptr()), None))

        eng.plan_graphs(gids)
        ms, _, _, _ = timed(c, step, steps, warmup)
        eng.close()
        out[tag] = {"value": G * steps / (ms / 1e3), "unit": "graphs/s", "ms_per_step": ms / steps, "steps": steps, "warmup": warmup,
                    "num_layers": L, "bn": bn, "hidden_dim": 20, "output_dim": 20, "kernel": "explain_var_kernel",
                    "gpu": name, "power_limit_w": power, "timing": "CUDA events around gx_explain_graphs (plan outside), L2 flushed between steps"}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    a.gpus = 1
    c = gpu_ctx(a)
    adj, feat, label, _ = make_graph_batch()
    print(json.dumps({"metric": "explained-graphs/sec (100 mask-opt epochs each), model variants",
                      "config": {"workload": "configs[3] stand-in: %d padded graphs (max_nodes 100, d=14), graph-level mask, 100 epochs" % adj.shape[0],
                                 "init": "device Philox"},
                      "variants": bench_graph_variants(a, c, adj, feat, label)}), flush=True)


if __name__ == "__main__":
    main()
