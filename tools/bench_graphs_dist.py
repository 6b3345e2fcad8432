#!/usr/bin/env python
"""Graph-classification mode sharded over GPUs (gnnx.dist.explain_graphs_sharded) on the configs[3] stand-in of bench.py: 4337 padded
graphs (max_nodes 100, d = 14), 100 epochs, one process per GPU:

    torchrun --nproc_per_node N tools/bench_graphs_dist.py [--steps 5 --warmup 2 --out result.json]

Reports, for the device (Philox) init:
  packed  graphs/s of the sharded call with every graph's packed masks on every rank (explain + ONE all-gather + unshard)
  dense   graphs/s of the same call with dense=True: the (4337, 100, 100) float64 arrays explain_graphs returns, built on device
  rank 0's explainer-kernel time per step
and, separately, the host time per rank of the torch-compatible init (every rank draws all 4337 x 100^2 normals, whatever it owns), a
bit-identity check of the dense result against explain_graphs on one GPU (rank 0), and the GPU name and power limit (read-only query)."""
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


def gpu_info(dev):
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:                                   # the query is informative only
        import torch
        return {"name": torch.cuda.get_device_name(dev), "error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file (rank 0)")
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    import gnnx
    from gnnx.dist import explain_graphs_sharded, ensure_comm, shard_layout
    from bench import make_graph_batch, NUM_EPOCHS

    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    if "MASTER_ADDR" not in os.environ:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29533")
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    adj, feat, label, W = make_graph_batch()
    G = adj.shape[0]
    gids = np.arange(G)
    args = types.SimpleNamespace(num_gc_layers=3, num_epochs=NUM_EPOCHS, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                 mask_bias=False, gpu=False, bias=True, method="base", dataset="graphs", bmname=None, hidden_dim=20,
                                 output_dim=20, name_suffix="", explainer_suffix="", logdir="/tmp/gnnx_bench_graphs_dist",
                                 gnnx_init="device", gnnx_seed=7)
    model = gnnx.models.GcnEncoderGraph(feat.shape[2], 20, 20, W["Wp"].shape[0], 3, bn=False, args=args)
    sd = {"conv_first.weight": W["W1"], "conv_first.bias": W["b1"], "conv_block.0.weight": W["W2"], "conv_block.0.bias": W["b2"],
          "conv_last.weight": W["W3"], "conv_last.bias": W["b3"], "pred_model.weight": W["Wp"], "pred_model.bias": W["bp"]}
    model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    ex = gnnx.Explainer(model=model, adj=adj, feat=feat, label=label, pred=None, train_idx=[], args=args, writer=None,
                        print_training=False, graph_mode=True, graph_idx=0, device=local)
    eng = ex.engine
    ensure_comm(eng)

    def timed(step):
        for _ in range(a.warmup):
            step()
        torch.cuda.synchronize()
        dist.barrier()
        kern = []
        t0 = time.perf_counter()
        for _ in range(a.steps):
            step()
            kern.append(eng.last_explain_ms())      # synchronises the engine's stream
        torch.cuda.synchronize()
        dist.barrier()
        ms = (time.perf_counter() - t0) * 1e3 / a.steps
        return {"ms_per_step": ms, "graphs_per_s": G / (ms / 1e3), "rank0_kernel_ms_per_step": float(np.mean(kern))}

    keep = {}
    res = {"packed": timed(lambda: keep.__setitem__("p", explain_graphs_sharded(ex, gids))),
           "dense": timed(lambda: keep.__setitem__("d", explain_graphs_sharded(ex, gids, dense=True)))}
    dense = keep["d"][3]
    # the torch-compatible init: host time per rank of the draw walk (every rank draws all G x max_nodes^2 normals)
    _, e_all = eng.count_graphs(gids)
    pos = shard_layout(e_all, world)[0][rank]
    rcs = [eng.graph_rows_cols(int(g)) for g in pos]
    t_init = []
    for _ in range(2):
        torch.manual_seed(0)
        t0 = time.perf_counter()
        ex._draw_graph_m0_subset(eng.batch_n, G, pos, rcs)
        t_init.append((time.perf_counter() - t0) * 1e3)
    t_all = [None] * world
    dist.all_gather_object(t_all, min(t_init))
    ident = None
    if rank == 0:
        full = ex.explain_graphs(gids.tolist(), save=False)            # the same list on one GPU, the product path
        d = dense.cpu().numpy()
        ident = bool(all(np.array_equal(d[t], full[t]) for t in range(G)))
    line = {"metric": "explained-graphs/sec, graph mode sharded (gnnx.dist.explain_graphs_sharded), device init", "world": world,
            "graphs": G, "epochs": NUM_EPOCHS, "sum_E_d": int(e_all.sum()), "steps": a.steps, "warmup": a.warmup, **res,
            "torch_init_host_ms_per_rank": t_all, "bit_identical": ident, "gpu": gpu_info(local),
            "config": "configs[3] stand-in (bench.make_graph_batch): 4337 padded graphs, max_nodes 100, d=14, 20/20/2 model"}
    if rank == 0:
        print(json.dumps(line))
        if a.out:
            with open(a.out, "w") as f:
                f.write(json.dumps(line) + "\n")
    dist.barrier()
    eng.comm_destroy()
    eng.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
