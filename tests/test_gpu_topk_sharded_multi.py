"""GPU (-m gpu), needs >= 2 devices: Explainer.explain_nodes_topk sharded over 2 ranks (one process per GPU) through
gnnx.dist.explain_nodes_topk_sharded -- the chunk loop on every rank, two all-gathers of the thresholds / counts and of the edge records --
must reproduce explain_nodes_topk on one GPU bit for bit, with the library's communicator and with torch.distributed, both inits."""
import os
import socket
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
NODES = list(range(0, 700, 9)) + [0, 300, 3]


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import conftest  # noqa: F401
    import torch.distributed as dist
    import util
    import gnnx
    import gnnx_oracle as O
    from gnnx.dist import explain_nodes_topk_sharded
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    fx = util.load_fixture("syn1")
    out = {}
    for init in ("torch", "device"):
        args = types.SimpleNamespace(num_gc_layers=3, num_epochs=30, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                     mask_bias=False, gpu=False, bias=True, method="base", dataset="syn1", bmname=None, hidden_dim=20,
                                     output_dim=20, name_suffix="", explainer_suffix="", logdir="/tmp/gnnx_topk_%d" % rank,
                                     gnnx_init=init, gnnx_seed=5)
        model = gnnx.models.GcnEncoderNode(10, 20, 20, 4, 3, bn=False, args=args)
        sd = {"conv_first.weight": fx.weights["W1"], "conv_first.bias": fx.weights["b1"], "conv_block.0.weight": fx.weights["W2"],
              "conv_block.0.bias": fx.weights["b2"], "conv_last.weight": fx.weights["W3"], "conv_last.bias": fx.weights["b3"],
              "pred_model.weight": fx.weights["Wp"], "pred_model.bias": fx.weights["bp"]}
        model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
        A = O.dense_from_csr(fx.rowptr, fx.col)
        ex = gnnx.Explainer(model=model, adj=A[None], feat=fx.feat[None], label=fx.label[None], pred=fx.pred[None],
                            train_idx=[], args=args, writer=None, print_training=False, graph_idx=-1, device=rank)
        res = {}
        for use_engine_comm in (True, False):
            torch.manual_seed(8)
            thr, offsets, uv, vals, pos = explain_nodes_topk_sharded(ex, NODES, chunk_size=7, use_engine_comm=use_engine_comm)
            res[use_engine_comm] = (thr.cpu().numpy(), np.asarray(offsets), uv.cpu().numpy(), vals.cpu().numpy(), torch.get_rng_state(), len(pos))
        if rank == 0:
            torch.manual_seed(8)
            thr, offsets, uv, vals = ex.explain_nodes_topk(NODES)               # the same list on one GPU
            out[init] = (res, (thr.cpu().numpy(), offsets, uv.cpu().numpy(), vals.cpu().numpy(), torch.get_rng_state()))
        dist.barrier()
        ex.engine.close()
    if rank == 0:
        q.put(out)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_topk_matches_single_gpu():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    try:
        out = q.get(timeout=300)
    finally:
        for p in procs:
            p.join(120)
            if p.is_alive():
                p.terminate()
                p.join(10)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    for init, (res, want) in out.items():
        for use_engine_comm, got in res.items():
            assert 0 < got[5] < len(NODES)
            for x, y in zip(got[:4], want[:4]):
                assert x.dtype == y.dtype and np.array_equal(x, y), (init, use_engine_comm)
            assert torch.equal(got[4], want[4]), (init, use_engine_comm)
