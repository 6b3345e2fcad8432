#!/usr/bin/env python
"""BASELINE configs[4] through the public interface, sharded: BA(N = 100 000, m = 32) => average degree 64, d = 128, 3-hop neighbourhoods
of about the whole graph, --nodes explained nodes (default 10 000) dealt across the ranks of a torchrun group, each rank explaining its
share --chunk nodes at a time (default: one per SM) and delivering denoise_graph's top-k edges (threshold_num = 20) in global node ids
(gnnx.dist.explain_nodes_topk_sharded).  The graph is built as bench.py --workload c5 builds it and handed to the Explainer as a
scipy.sparse adjacency; the device init (Philox N(1, 2/n)).

    torchrun --nproc_per_node 1 tools/bench_c5_dist.py --nodes 1320

Prints one JSON line (rank 0): nodes/s (device-timed: the explainer kernels of every chunk; wall: the whole sharded call), the per-rank
time split (count, plan, explain, top-k, the two gathers), gathered bytes against the full-mask bytes, the GPU name and power limit read
in the same run, and a bit-identity check: rank 0 re-runs the first chunk of the list with explain_nodes_topk on one GPU."""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gnn-model-explainer_b200"))
sys.path.insert(0, ROOT)


def gpu_info(index):
    q = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    f = [x.strip() for x in q.stdout.strip().split(",")]
    return {"name": f[0], "power_limit": f[1], "sm_max_clock": f[2]} if len(f) >= 3 else {"error": q.stderr.strip()}


def build_c5(N, m, d=128, C=4):
    """bench.py bench_c5's graph, features, labels, weights and predicted labels (same seeds)."""
    import scipy.sparse as sp
    from bench import make_ba_csr
    rng = np.random.default_rng(0)
    rowptr, col = make_ba_csr(N, m, 0)
    X = rng.normal(size=(N, d)).astype(np.float32)
    label = rng.integers(0, C, N).astype(np.int32)
    sc = lambda *s_: (rng.normal(size=s_) * 0.3).astype(np.float32)
    W = dict(W1=sc(d, 20), b1=sc(20), W2=sc(20, 20), b2=sc(20), W3=sc(20, 20), b3=sc(20), Wp=sc(C, 60), bp=sc(C))
    A = sp.csr_matrix((np.ones(len(col), np.float32), col, rowptr), shape=(N, N))
    nrm = lambda Y: Y / np.maximum(np.linalg.norm(Y, axis=1, keepdims=True), 1e-12)
    H1 = np.maximum(nrm((A @ X) @ W["W1"] + W["b1"]), 0); H2 = np.maximum(nrm((A @ H1) @ W["W2"] + W["b2"]), 0)
    H3 = nrm((A @ H2) @ W["W3"] + W["b3"])
    logits = np.concatenate([H1, H2, H3], 1) @ W["Wp"].T + W["bp"]
    return A, X, label, W, logits.astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10000)
    ap.add_argument("--chunk", type=int, default=None, help="nodes per chunk on a rank (default: the device's SM count)")
    ap.add_argument("--n", type=int, default=100000)
    ap.add_argument("--m", type=int, default=32)
    ap.add_argument("--epochs", type=int, default=100)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    import gnnx
    from gnnx.dist import explain_nodes_topk_sharded, count_nodes_cached
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    world, rank = dist.get_world_size(), dist.get_rank()
    t0 = time.perf_counter()
    A, X, label, W, logits = build_c5(a.n, a.m)
    gen_s = time.perf_counter() - t0
    args = types.SimpleNamespace(num_gc_layers=3, num_epochs=a.epochs, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                 mask_bias=False, gpu=True, bias=True, method="base", dataset="c5", bmname=None, hidden_dim=20,
                                 output_dim=20, name_suffix="", explainer_suffix="", logdir="/tmp", gnnx_init="device", gnnx_seed=99)
    model = gnnx.models.GcnEncoderNode(X.shape[1], 20, 20, 4, 3, bn=False, args=args)
    sd = {"conv_first.weight": W["W1"], "conv_first.bias": W["b1"], "conv_block.0.weight": W["W2"], "conv_block.0.bias": W["b2"],
          "conv_last.weight": W["W3"], "conv_last.bias": W["b3"], "pred_model.weight": W["Wp"], "pred_model.bias": W["bp"]}
    model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    ex = gnnx.Explainer(model=model, adj=A, feat=X[None], label=label[None], pred=logits[None], train_idx=[], args=args, writer=None,
                        print_training=False, graph_idx=-1, device=local)
    nodes = np.random.default_rng(1).permutation(a.n)[:a.nodes].astype(np.int64)
    chunk = a.chunk or torch.cuda.get_device_properties(local).multi_processor_count
    ex.explain_nodes_topk(nodes[:2], chunk_size=2)                  # warm-up: module loads, the streaming kernel's first launch
    dist.barrier()
    torch.cuda.synchronize()
    tw = time.perf_counter()
    timings = {}
    thr, offsets, uv, vals, pos = explain_nodes_topk_sharded(ex, nodes, chunk_size=chunk, timings=timings)
    torch.cuda.synchronize()
    dist.barrier()
    wall = time.perf_counter() - tw
    per_rank = [None] * world
    dist.all_gather_object(per_rank, {"rank": rank, "nodes": int(len(pos)), **{k: float(v) for k, v in timings.items()}})
    if rank != 0:
        dist.destroy_process_group()
        return
    _, e_all = count_nodes_cached(ex, nodes)
    full_bytes = 4 * int(np.sum(e_all))
    gathered = 8 * len(nodes) + 12 * int(offsets[-1])
    # bit identity: the first chunk of the list again, on this GPU alone
    k = min(chunk, len(nodes))
    t1, o1, u1, v1 = ex.explain_nodes_topk(nodes[:k], chunk_size=chunk)
    same = (torch.equal(t1, thr[:k]) and np.array_equal(o1, offsets[:k + 1]) and torch.equal(u1, uv[:offsets[k]])
            and torch.equal(v1, vals[:offsets[k]]))
    dev_s = max(r["explain_device"] for r in per_rank)
    chunks = [int(np.ceil(r["nodes"] / chunk)) for r in per_rank]
    line = {
        "metric": "configs[4] explained nodes/s, top-k delivery (threshold_num 20)", "world": world, "nodes": len(nodes), "chunk": chunk,
        "config": "BA(N=%d, m=%d) d=128 C=4, 3-hop, %d epochs, device init, scipy.sparse adjacency through Explainer" % (a.n, a.m, a.epochs),
        "gpu": gpu_info(local),
        "nodes_per_s_device": len(nodes) / dev_s, "nodes_per_s_wall": len(nodes) / wall, "wall_s": wall,
        "per_rank": per_rank,
        "per_chunk_rank0": {k2: per_rank[0][k2] / max(chunks[0], 1) for k2 in ("plan", "explain", "explain_device", "topk") if k2 in per_rank[0]},
        "gathered_bytes": gathered, "full_mask_bytes": full_bytes, "gathered_over_full": gathered / max(full_bytes, 1),
        "edges_delivered": int(offsets[-1]), "graph_gen_s": gen_s,
        "bit_identical_first_chunk": bool(same),
    }
    s = json.dumps(line)
    print(s, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
