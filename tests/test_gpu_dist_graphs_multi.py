"""GPU (-m gpu), needs >= 2 devices: Explainer(graph_mode=True) sharded over 2 ranks (one process per GPU) through
gnnx.dist.explain_graphs_sharded with the library's own NCCL communicator must reproduce the single-GPU explain_graphs bit for bit,
packed and dense, with the torch-compatible init (every rank walks the whole list through torch's RNG)."""
import os
import socket
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GIDS = [5, 0, 11, 3, 3, 8, 1, 10, 2, 9, 7]


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import conftest  # noqa: F401
    import torch.distributed as dist
    import util
    import gnnx
    from gnnx.dist import explain_graphs_sharded
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    args = types.SimpleNamespace(num_gc_layers=3, num_epochs=30, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                 mask_bias=False, gpu=False, bias=True, method="base", dataset="graphs", bmname=None, hidden_dim=20,
                                 output_dim=20, name_suffix="", explainer_suffix="", logdir="/tmp/gnnx_dist_graphs_%d" % rank,
                                 gnnx_init="torch")
    model = gnnx.models.GcnEncoderGraph(14, 20, 20, 2, 3, bn=False, args=args)
    sd = {"conv_first.weight": gg["W1"], "conv_first.bias": gg["b1"], "conv_block.0.weight": gg["W2"], "conv_block.0.bias": gg["b2"],
          "conv_last.weight": gg["W3"], "conv_last.bias": gg["b3"], "pred_model.weight": gg["Wp"], "pred_model.bias": gg["bp"]}
    model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    ex = gnnx.Explainer(model=model, adj=torch.tensor(gg["adj"], dtype=torch.float), feat=torch.tensor(gg["feat"]),
                        label=torch.tensor(gg["label"]), pred=None, train_idx=[], args=args, writer=None, print_training=False,
                        graph_mode=True, graph_idx=0, device=rank)
    torch.manual_seed(8)
    values, offsets, (_, pos), dense = explain_graphs_sharded(ex, GIDS, dense=True)     # gx_allgather_masks: the library's communicator
    rng_after = torch.get_rng_state()
    if rank == 0:
        torch.manual_seed(8)
        full = ex.explain_graphs(GIDS, save=False)                                       # the same list on one GPU
        same_rng = torch.equal(torch.get_rng_state(), rng_after)
        packed = np.concatenate([D[ex.engine.graph_rows_cols(g)] for D, g in zip(full, GIDS)]).astype(np.float32)
        want_off = np.concatenate([[0], np.cumsum([len(ex.engine.graph_rows_cols(g)[0]) for g in GIDS])])
        q.put((values.cpu().numpy(), np.asarray(offsets), want_off, dense.cpu().numpy(), np.stack(full), packed, same_rng, len(pos)))
    dist.barrier()
    ex.engine.close()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_graph_mode_matches_single_gpu():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    try:
        values, offsets, want_off, dense, full, packed, same_rng, owned = q.get(timeout=300)
    finally:
        for p in procs:
            p.join(120)
            if p.is_alive():
                p.terminate()
                p.join(10)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    assert 0 < owned < len(GIDS)
    assert np.array_equal(offsets, want_off)
    assert np.array_equal(values, packed), "sharded masks differ from the single-GPU result"
    assert np.array_equal(dense, full), "densified masks differ from explain_graphs"
    assert same_rng, "torch's RNG ends elsewhere than after one process's explain_graphs"
