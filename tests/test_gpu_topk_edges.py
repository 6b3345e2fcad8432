"""GPU (-m gpu), one device: top-k delivery of node masks in global node ids (gx_denoise_topk_edges, Engine.denoise_topk_edges,
Explainer.explain_nodes_topk, gnnx.dist.explain_nodes_topk_sharded) and the sparse node-mode adjacency.

gx_denoise_topk_edges against the reference's own denoise_graph output and against gx_denoise_topk + host mapping; the chunked explain
against explain_nodes_packed + denoise_nodes for every chunk size, both inits, the streaming kernel; rank emulation of the sharded call
for world sizes 1, 2, 3, 4 and 8 (every rank's shard and chunk loop on its own, both gathers put together on the host with shard_layout);
a one-rank group end to end with the library's communicator and with gloo."""
import socket
import types

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.distributed as dist

import gnnx
import gnnx_oracle as O
import util
from gnnx import dist as gdist

pytestmark = pytest.mark.gpu
WORLDS = (1, 2, 3, 4, 8)
NODES = [0, 3, 300, 301, 683, 699, 13, 550, 3, 42, 120, 640, 401, 7, 222, 515, 98, 333]     # hub node 0, a repeated node


@pytest.fixture(scope="module")
def syn1():
    return util.load_fixture("syn1")


def _args(tmp_path, fx, init="torch", epochs=20, **over):
    a = dict(num_gc_layers=3, num_epochs=epochs, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid", mask_bias=False,
             gpu=False, bias=True, method="base", dataset=fx.name, bmname=None, hidden_dim=20, output_dim=20, name_suffix="",
             explainer_suffix="", logdir=str(tmp_path), gnnx_init=init, gnnx_seed=5)
    a.update(over)
    return types.SimpleNamespace(**a)


def _model(fx, args):
    model = gnnx.models.GcnEncoderNode(fx.feat.shape[1], 20, 20, fx.weights["Wp"].shape[0], 3, bn=False, args=args)
    sd = {"conv_first.weight": fx.weights["W1"], "conv_first.bias": fx.weights["b1"], "conv_block.0.weight": fx.weights["W2"],
          "conv_block.0.bias": fx.weights["b2"], "conv_last.weight": fx.weights["W3"], "conv_last.bias": fx.weights["b3"],
          "pred_model.weight": fx.weights["Wp"], "pred_model.bias": fx.weights["bp"]}
    model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    return model


def _explainer(fx, args, sparse=False):
    A = O.dense_from_csr(fx.rowptr, fx.col)
    adj = sp.csr_matrix(A) if sparse else A[None]
    return gnnx.Explainer(model=_model(fx, args), adj=adj, feat=fx.feat[None], label=fx.label[None], pred=fx.pred[None],
                          train_idx=[], args=args, writer=None, print_training=False, graph_idx=-1)


def _host_edges(eng, plan, mask, thr_num):
    """gx_denoise_topk + host mapping: per task (thr, directed count, the row < col kept slots as global (u, v), their values)."""
    eng_thr, cnt, slots, vals = eng.denoise_topk(mask, thr_num, cap=4096)
    out = []
    for t in range(plan.count):
        k = int(cnt[t])
        rows, cols = plan.rows_cols_of(t)
        s = slots[t, :k]
        up = rows[s] < cols[s]
        nb = plan.neighbors_of(t).astype(np.int64)
        out.append((eng_thr[t], k, np.stack([nb[rows[s][up]], nb[cols[s][up]]], 1), vals[t, :k][up]))
    return out


def _flatten(per_task):
    """[(thr, _, uv, vals)] -> (thr, offsets, uv, vals) as explain_nodes_topk returns them (host arrays)."""
    thr = np.array([p[0] for p in per_task], np.float32)
    offsets = np.concatenate([[0], np.cumsum([len(p[2]) for p in per_task])]).astype(np.int64)
    uv = np.concatenate([p[2] for p in per_task]).astype(np.int32).reshape(-1, 2)
    vals = np.concatenate([p[3] for p in per_task]).astype(np.float32)
    return thr, offsets, uv, vals


def _host(res):
    thr, offsets, uv, vals = res[:4]
    return thr.cpu().numpy(), np.asarray(offsets), uv.cpu().numpy(), vals.cpu().numpy()


def _assert_same(a, b, what=""):
    for x, y, name in zip(a, b, ("thr", "offsets", "uv", "vals")):
        assert x.dtype == y.dtype and np.array_equal(x, y), (what, name)


# ------------------------------------------------------------------------------------------------ gx_denoise_topk_edges
@pytest.mark.parametrize("which", ["syn1", "syn4"])
def test_edges_match_reference_denoise_graph(which):
    """The reference's golden masks (so the values are the reference's) against its own denoise_graph(threshold_num=20) edges and weights."""
    fx = util.load_fixture(which)
    dg = np.load(util.GOLDEN + "/denoise_golden.npz")
    nodes = [int(x) for x in dg[which + "_nodes"]]
    eng = util.make_engine(fx)
    plan = eng.plan_nodes(nodes, 3)
    mask = np.concatenate([fx.gold["n%d_mask" % n] for n in nodes]).astype(np.float32)
    for space in ("host", "device"):
        m = mask if space == "host" else torch.from_numpy(mask).cuda()
        thr, cnt, uv, vals = eng.denoise_topk_edges(m, int(dg["threshold_num"]), cap=256)
        if space == "device":
            assert uv.is_cuda and vals.is_cuda and uv.dtype == torch.int32
            thr, cnt, uv, vals = (x.cpu().numpy() for x in (thr, cnt, uv, vals))
        for t, node in enumerate(nodes):
            want = dg["%s_n%d_edges" % (which, node)]
            nb = plan.neighbors_of(t)
            k = int(cnt[t])
            assert np.array_equal(uv[t, :k], nb[want]), (which, node, space)
            assert np.array_equal(vals[t, :k], dg["%s_n%d_weights" % (which, node)]), (which, node, space)
            assert thr[t] == dg["%s_n%d_weights" % (which, node)].min()
            assert (uv[t, k:] == -1).all()
    eng.close()


def test_edges_match_denoise_topk_all_syn1_nodes(syn1):
    """Kernel masks of all 700 syn1 nodes: the thresholds of gx_denoise_topk, half its count, the same values; host and device agree."""
    eng = util.make_engine(syn1)
    nodes = list(range(syn1.N))
    plan = eng.plan_nodes(nodes, 3)
    mask = np.zeros(plan.total_edges, np.float32)
    eng.explain_nodes_host(eng.make_hparams(num_epochs=30, init=1, seed=3), None, mask)
    want = _host_edges(eng, plan, mask, 20)
    h = eng.denoise_topk_edges(mask, 20, cap=128)
    d = [x.cpu().numpy() for x in eng.denoise_topk_edges(torch.from_numpy(mask).cuda(), 20, cap=128)]
    for x, y in zip(h, d):
        assert np.array_equal(x, y)
    thr, cnt, uv, vals = h
    for t in range(plan.count):
        w_thr, w_cnt, w_uv, w_vals = want[t]
        assert thr[t] == w_thr and 2 * cnt[t] == w_cnt and cnt[t] == len(w_uv), t
        assert np.array_equal(uv[t, :cnt[t]], w_uv) and np.array_equal(vals[t, :cnt[t]], w_vals), t
        assert (np.diff(uv[t, :cnt[t], 0].astype(np.int64) * syn1.N + uv[t, :cnt[t], 1]) > 0).all()      # ascending (u, v), u < v
        assert (uv[t, :cnt[t], 0] < uv[t, :cnt[t], 1]).all()
    eng.close()


def test_edges_awkward_inputs(syn1):
    """Asymmetric random values with heavy ties, zeros, a node without a positive value and caps below the number kept, against numpy."""
    eng = util.make_engine(syn1)
    nodes = [0, 3, 300, 683, 13, 699]
    plan = eng.plan_nodes(nodes, 3)
    rng = np.random.default_rng(5)
    v = rng.random(plan.total_edges).astype(np.float32)
    v[rng.random(plan.total_edges) < 0.1] = 0.0
    sl = slice(plan.edge_off[2], plan.edge_off[3])
    v[sl] = np.round(v[sl] * 8) / 8                      # heavy ties
    v[plan.edge_off[4]:plan.edge_off[5]] = 0.0           # no positive entry
    for k, cap in ((20, 64), (5, 3), (3, 4096), (1, 1)):
        for space in ("host", "device"):
            res = eng.denoise_topk_edges(v if space == "host" else torch.from_numpy(v).cuda(), k, cap=cap)
            thr, cnt, uv, vals = res if space == "host" else (x.cpu().numpy() for x in res)
            assert uv.shape == (plan.count, cap, 2) and vals.shape == (plan.count, cap)
            for t in range(plan.count):
                x = v[plan.edge_off[t]:plan.edge_off[t + 1]]
                pos = x[x > 0]
                if len(pos) == 0:
                    assert cnt[t] == 0 and np.isinf(thr[t]) and thr[t] > 0 and (uv[t] == -1).all() and (vals[t] == 0).all()
                    continue
                want_thr = np.sort(pos)[-min(len(pos), 2 * k)]
                assert thr[t] == want_thr
                rows, cols = plan.rows_cols_of(t)
                keep = np.nonzero((x >= want_thr) & (rows < cols))[0]
                assert cnt[t] == len(keep), (k, cap, t)
                m = min(len(keep), cap)
                nb = plan.neighbors_of(t)
                assert np.array_equal(uv[t, :m], np.stack([nb[rows[keep[:m]]], nb[cols[keep[:m]]]], 1))
                assert np.array_equal(vals[t, :m], x[keep[:m]])
                assert (uv[t, m:] == -1).all() and (vals[t, m:] == 0).all()
    eng.close()


# ------------------------------------------------------------------------------------------------ Explainer.explain_nodes_topk
def _packed_then_denoise(ex, nodes, k=20):
    """explain_nodes_packed + denoise_nodes (local numbering), mapped to global ids."""
    plan, mask = ex.explain_nodes_packed(nodes)
    graphs, thr = ex.denoise_nodes(plan, mask, threshold_num=k, max_component=False)
    per = []
    for t in range(plan.count):
        nb = plan.neighbors_of(t)
        e = np.array(sorted((min(u, v), max(u, v)) for u, v in graphs[t].edges()), np.int64).reshape(-1, 2)
        w = np.array([graphs[t][u][v]["weight"] for u, v in e], np.float32)
        per.append((thr[t], None, nb[e], w))
    return _flatten(per)


@pytest.mark.parametrize("init", ["torch", "device"])
def test_chunk_invariance_and_packed_parity(syn1, tmp_path, init):
    ex = _explainer(syn1, _args(tmp_path, syn1, init=init))
    torch.manual_seed(4)
    want = _packed_then_denoise(ex, NODES)
    rng_after = torch.get_rng_state()
    for chunk in (1, 5, 132, len(NODES), None):
        torch.manual_seed(4)
        res = ex.explain_nodes_topk(NODES, threshold_num=20, chunk_size=chunk)
        assert torch.equal(torch.get_rng_state(), rng_after), chunk       # M0 and torch's RNG as explain_nodes leaves them
        thr, offsets, uv, vals = res
        assert thr.is_cuda and uv.is_cuda and vals.is_cuda and uv.dtype == torch.int32 and offsets.dtype == np.int64
        _assert_same(_host(res), want, chunk)
    assert not any(f.suffix == ".npy" for f in tmp_path.iterdir())
    ex.engine.close()


def test_torch_init_rng_matches_explain_nodes(syn1, tmp_path):
    """With the torch init, explain_nodes draws the same M0 as explain_nodes_topk, and leaves torch's RNG in the same place."""
    ex = _explainer(syn1, _args(tmp_path, syn1, init="torch"))
    torch.manual_seed(9)
    ex.explain_nodes(NODES[:6], save=False)
    after = torch.get_rng_state()
    torch.manual_seed(9)
    ex.explain_nodes_topk(NODES[:6], chunk_size=4)
    assert torch.equal(torch.get_rng_state(), after)
    ex.engine.close()


def test_latency_mode_is_off_for_topk(syn1, tmp_path):
    ex = _explainer(syn1, _args(tmp_path, syn1, init="device", gnnx_latency=True))
    ref = _explainer(syn1, _args(tmp_path, syn1, init="device"))
    _assert_same(_host(ex.explain_nodes_topk(NODES, chunk_size=3)), _host(ref.explain_nodes_topk(NODES)))
    ex.engine.close(); ref.engine.close()


def _ba_explainer(tmp_path, N=1500, m=6, d=128, seed=11):
    """BA(N, m), d = 128 through a scipy.sparse adjacency: 3-hop neighbourhoods of most of the graph, beyond shared memory."""
    import networkx as nx
    rng = np.random.default_rng(seed)
    G = nx.barabasi_albert_graph(N, m, seed=seed)
    e = np.array(G.edges(), np.int64)
    A = sp.coo_matrix((np.ones(2 * len(e), np.float32), (np.r_[e[:, 0], e[:, 1]], np.r_[e[:, 1], e[:, 0]])), shape=(N, N))
    fx = types.SimpleNamespace(name="ba", feat=rng.normal(size=(N, d)).astype(np.float32))
    args = _args(tmp_path, fx, init="device", epochs=4)
    torch.manual_seed(seed)
    model = gnnx.models.GcnEncoderNode(d, 20, 20, 4, 3, bn=False, args=args)
    return gnnx.Explainer(model=model, adj=A, feat=fx.feat[None], label=rng.integers(0, 4, (1, N)), pred=None, train_idx=[],
                          args=args, writer=None, print_training=False, graph_idx=-1)


def test_streaming_kernel_chunks(tmp_path):
    ex = _ba_explainer(tmp_path)
    nodes = [0, 700, 1499, 20, 999]
    ex.engine.plan_nodes(nodes, 3, fetch=False)
    assert ex.engine.plan_class_counts()[0][5] >= 3        # the large tasks land in the streaming class by themselves
    whole = _host(ex.explain_nodes_topk(nodes, chunk_size=len(nodes)))
    _assert_same(_host(ex.explain_nodes_topk(nodes, chunk_size=2)), whole)
    assert int(whole[1][-1]) > 0
    _assert_same(whole, _packed_then_denoise(ex, nodes))
    ex.engine.close()


# ------------------------------------------------------------------------------------------------ rank emulation
def _emulate(ex, nodes, world, chunk, seed):
    """Every rank's shard and chunk loop on its own (as explain_nodes_topk_sharded runs them), both gathers assembled with shard_layout."""
    nodes = np.asarray(nodes, np.int64)
    n_all, e_all = gdist.count_nodes_cached(ex, nodes)
    shards = gdist.shard_layout(e_all, world)[0]
    rng_states, parts = [], []
    for rank in range(world):
        torch.manual_seed(seed)
        thr, cnt, uv, vals = ex._topk_chunks(nodes, shards[rank], n_all, 20, chunk)
        rng_states.append(torch.get_rng_state())
        parts.append((thr.cpu().numpy(), cnt, uv.cpu().numpy(), vals.cpu().numpy()))
    num = len(nodes)
    # gather 1: (threshold, count) per node
    sizes1 = np.full(num, 2, np.int64)
    _, slot1, src1, _ = gdist.shard_layout(sizes1, world, e_all)
    buf = np.zeros(world * slot1, np.float32)
    for r, (thr, cnt, _, _) in enumerate(parts):
        head = np.stack([thr, cnt.astype(np.int32).view(np.float32)], 1).reshape(-1)
        buf[r * slot1: r * slot1 + len(head)] = head
    g1 = np.stack([buf[src1[p]: src1[p] + 2] for p in range(num)]) if num else np.zeros((0, 2), np.float32)
    thr_all, cnt_all = g1[:, 0].copy(), g1[:, 1].copy().view(np.int32).astype(np.int64)
    # gather 2: 3 words per edge, the same shards
    sizes2 = 3 * cnt_all
    sh2, slot2, src2, _ = gdist.shard_layout(sizes2, world, e_all)
    assert all(np.array_equal(a, b) for a, b in zip(sh2, shards))
    buf = np.zeros(world * slot2, np.float32)
    for r, (_, _, uv, vals) in enumerate(parts):
        rec = np.concatenate([uv.view(np.float32), vals[:, None]], 1).reshape(-1)
        buf[r * slot2: r * slot2 + len(rec)] = rec
    g2 = np.concatenate([buf[src2[p]: src2[p] + sizes2[p]] for p in range(num)]).reshape(-1, 3)
    offsets = np.concatenate([[0], np.cumsum(cnt_all)]).astype(np.int64)
    return (thr_all, offsets, g2[:, :2].copy().view(np.int32), g2[:, 2].copy()), rng_states


@pytest.mark.parametrize("init", ["torch", "device"])
def test_rank_emulation(syn1, tmp_path, init):
    ex = _explainer(syn1, _args(tmp_path, syn1, init=init))
    torch.manual_seed(6)
    want = _host(ex.explain_nodes_topk(NODES, chunk_size=4))
    rng_after = torch.get_rng_state()
    for world in WORLDS:
        got, states = _emulate(ex, NODES, world, chunk=3, seed=6)
        _assert_same(got, want, world)
        if init == "torch":
            assert all(torch.equal(s, rng_after) for s in states), world
    ex.engine.close()


# ------------------------------------------------------------------------------------------------ end to end, one rank
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def test_explain_nodes_topk_sharded_one_rank(syn1, tmp_path):
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % _free_port(), rank=0, world_size=1)
    try:
        ex = _explainer(syn1, _args(tmp_path, syn1, init="torch"))
        torch.manual_seed(21)
        want = _host(ex.explain_nodes_topk(NODES))
        rng_after = torch.get_rng_state()
        for use_engine_comm in (False, True):         # torch.distributed (gloo), then the library's NCCL communicator
            torch.manual_seed(21)
            timings = {}
            res = gdist.explain_nodes_topk_sharded(ex, NODES, chunk_size=5, use_engine_comm=use_engine_comm, timings=timings)
            assert torch.equal(torch.get_rng_state(), rng_after)
            _assert_same(_host(res), want, use_engine_comm)
            assert np.array_equal(res[4], np.arange(len(NODES)))
            assert timings["gather2_bytes"] == 12 * int(want[1][-1]) and timings["gather1_bytes"] == 8 * len(NODES)
            assert all(timings[k] >= 0 for k in ("count", "plan", "m0", "explain", "topk", "gather1", "gather2", "explain_device"))
        assert not any(f.suffix == ".npy" for f in tmp_path.iterdir())
        ex.engine.close()
    finally:
        dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------ sparse adjacency
def test_sparse_adjacency_matches_dense(syn1, tmp_path):
    args = _args(tmp_path, syn1, init="torch")
    dense = _explainer(syn1, args)
    sparse = _explainer(syn1, args, sparse=True)
    for node in (0, 300, 683):
        a, b = dense.extract_neighborhood(node), sparse.extract_neighborhood(node)
        assert a[0] == b[0] and all(np.array_equal(x, y) for x, y in zip(a[1:], b[1:])), node
        assert b[1].shape == (len(b[4]), len(b[4]))
        torch.manual_seed(node)
        m_d = dense.explain(node)
        torch.manual_seed(node)
        assert np.array_equal(sparse.explain(node), m_d), node
    torch.manual_seed(2)
    want = dense.explain_nodes(NODES, save=False)
    torch.manual_seed(2)
    got = sparse.explain_nodes(NODES, save=False)
    assert all(np.array_equal(x, y) for x, y in zip(got, want))
    torch.manual_seed(2)
    w2 = _host(dense.explain_nodes_topk(NODES))
    torch.manual_seed(2)
    _assert_same(_host(sparse.explain_nodes_topk(NODES)), w2)
    dense.engine.close(); sparse.engine.close()


def test_sparse_adjacency_refusals(syn1, tmp_path):
    args = _args(tmp_path, syn1)
    A = sp.csr_matrix(O.dense_from_csr(syn1.rowptr, syn1.col) * 2.0)
    with pytest.raises(NotImplementedError):
        gnnx.Explainer(model=_model(syn1, args), adj=A, feat=syn1.feat[None], label=syn1.label[None], pred=syn1.pred[None],
                       train_idx=[], args=args, writer=None, print_training=False, graph_idx=-1)
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    model = gnnx.models.GcnEncoderGraph(gg["feat"].shape[2], 20, 20, 2, 3, bn=False, args=args)
    with pytest.raises(ValueError):
        gnnx.Explainer(model=model, adj=sp.csr_matrix(gg["adj"][0]), feat=gg["feat"], label=gg["label"], pred=None, train_idx=[],
                       args=args, writer=None, print_training=False, graph_mode=True, graph_idx=0)
