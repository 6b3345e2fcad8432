"""CPU: the two all-gathers of gnnx.dist.explain_nodes_topk_sharded (allgather_topk) with gloo at world size 2 on fake per-rank records --
thresholds and counts first, then 3-word edge records in the explanation's shards -- including a rank that owns nothing; and
graph_utils.csr_from_sparse against csr_from_dense."""
import os
import socket

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _item(p):
    """Fake result of list entry p: (threshold, uv [k, 2] int32, vals [k] float32); k = 0 for some entries, ids past 2^23 for others."""
    rng = np.random.default_rng(500 + p)
    k = (p * 5) % 7
    uv = np.sort(rng.integers(0, 1 << 30 if p % 3 == 0 else 1000, (k, 2)), 1).astype(np.int32)
    return np.float32(rng.random()) if k else np.float32(np.inf), uv, rng.random(k).astype(np.float32)


def _costs(num):
    return (np.arange(num) * 37) % 11 + 1


def _worker(rank, world, port, num, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import conftest  # noqa: F401  (sys.path)
    from gnnx.dist import shard_layout, allgather_topk
    costs = _costs(num)
    pos = shard_layout(costs, world, costs)[0][rank]
    items = [_item(int(p)) for p in pos]
    thr = torch.tensor([it[0] for it in items], dtype=torch.float32)
    cnt = np.array([len(it[1]) for it in items], np.int64)
    uv = torch.from_numpy(np.concatenate([it[1] for it in items]).reshape(-1, 2) if items else np.zeros((0, 2), np.int32))
    vals = torch.from_numpy(np.concatenate([it[2] for it in items]) if items else np.zeros(0, np.float32))
    calls = []
    orig = dist.all_gather_into_tensor
    dist.all_gather_into_tensor = lambda *a, **k: (calls.append(1), orig(*a, **k))[1]
    timings = {}
    out = allgather_topk(thr, cnt, uv, vals, costs, timings=timings)
    assert len(calls) == 2, "two collectives: thresholds / counts, then the records"
    q.put((rank, len(pos), [x.numpy() if torch.is_tensor(x) else x for x in out], timings))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("num", [13, 1])
def test_allgather_topk_world2(num):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, num, q)) for r in range(2)]
    [p.start() for p in procs]
    res = [q.get(timeout=120) for _ in range(2)]
    [p.join(60) for p in procs]
    items = [_item(p) for p in range(num)]
    want_thr = np.array([it[0] for it in items], np.float32)
    want_off = np.concatenate([[0], np.cumsum([len(it[1]) for it in items])]).astype(np.int64)
    want_uv = np.concatenate([it[1] for it in items]).reshape(-1, 2)
    want_vals = np.concatenate([it[2] for it in items])
    owned = sorted(r[1] for r in res)
    assert sum(owned) == num and (num > 1 or owned[0] == 0)      # with one item, one rank owns nothing
    for rank, _, (thr, off, uv, vals), timings in res:
        assert np.array_equal(thr, want_thr) and np.array_equal(off, want_off), rank
        assert uv.dtype == np.int32 and np.array_equal(uv, want_uv), rank
        assert np.array_equal(vals, want_vals), rank
        assert timings["gather1_bytes"] == 8 * num and timings["gather2_bytes"] == 12 * int(want_off[-1])


def test_csr_from_sparse_matches_dense():
    from gnnx.graph_utils import csr_from_dense, csr_from_sparse
    rng = np.random.default_rng(3)
    A = (rng.random((60, 60)) < 0.1).astype(np.float32)
    A = np.maximum(A, A.T)
    A[5] = 0; A[:, 5] = 0                              # an isolated row
    A[7, 7] = 1                                        # a self loop
    want = csr_from_dense(A)
    coo = sp.coo_matrix(A)
    dup = sp.coo_matrix((np.r_[coo.data, 0.0], (np.r_[coo.row, 3], np.r_[coo.col, 4])), shape=A.shape)   # an explicit zero
    for M in (sp.csr_matrix(A), sp.csc_matrix(A), coo, dup, sp.csr_array(A)):
        got = csr_from_sparse(M)
        assert got[0].dtype == np.int32 and got[1].dtype == np.int32
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), type(M)
    with pytest.raises(NotImplementedError):
        csr_from_sparse(sp.csr_matrix(A * 0.5))
    with pytest.raises(ValueError):
        csr_from_sparse(sp.csr_matrix(np.ones((3, 4))))
