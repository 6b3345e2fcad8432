"""GPU (-m gpu): GCNs with hidden / output widths of 129 .. 256 on the model-variant kernel's row-block path (explain_var.cu, kBlk) and
the model forward (forward.cu), through the C ABI, the drop-in Explainer and gnnx.dist, node and graph mode: against the masks the
unmodified reference returned (tests/golden/wide_layers_golden.npz), against the torch port (gnnx_oracle.explain_dense_torch) in fp32
and fp64, and against the narrow kernel on a zero-padded model."""
import os
import types

import numpy as np
import pytest
import torch

import gnnx
import gnnx_oracle as O
import pool_oracle as PO
import util
from gnnx import _abi
from test_gpu_deep import GG, GX_ERR_UNSUPPORTED, _args, _check, _graph_setup, _hp, _m0, _node_setup, _ohp, _state_dict, _sub, random_model
from test_oracle_pool_ties import NEAR_TIES
from test_oracle_wide_layers import GOLDEN, case_weights, golden_cases

pytestmark = pytest.mark.gpu

# seed, L, bn, hid, emb, d, C, opt, scheduler.  Every width pair of the row-block path, 2 / 3 / 5 / 7 layers, d = 10 / 128 and the wide
# input path (d = 300); the 256-wide conv weights go through L2, the (129, 129) and (20, 256) ones at L = 2 fit shared memory.
CASES = [
    (1, 3, False, 256, 256, 10, 4, "adam", "none"),
    (2, 2, True, 129, 129, 128, 3, "sgd", "step"),
    (3, 5, False, 160, 136, 12, 4, "rmsprop", "cos"),
    (4, 7, True, 256, 20, 16, 3, "adagrad", "none"),
    (5, 3, True, 20, 256, 300, 3, "adam", "step"),
    (6, 2, False, 256, 256, 300, 4, "adagrad", "cos"),
    (7, 5, True, 256, 256, 10, 3, "adam", "none"),
    (8, 7, False, 129, 129, 128, 5, "sgd", "cos"),
    (9, 2, False, 20, 256, 10, 3, "rmsprop", "step"),
]


def _case_id(c):
    return "s%d_L%d%s_h%d_e%d_d%d_%s_%s" % (c[0], c[1], "_bn" if c[2] else "", c[3], c[4], c[5], c[7], c[8])


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_wide_layers_nodes_match_port(case):
    seed, L, bn, hid, emb, d, C, opt, sched = case
    s = _node_setup(seed, L, bn, False, hid, emb, d, C)
    nodes = [0, 7, 23, 47]
    plan = s.eng.plan_nodes(nodes, L)
    m0, dense = _m0(plan, 500 * seed)
    E = 20
    out = np.zeros(plan.total_edges, np.float32)
    fm = np.zeros((plan.count, d), np.float32)
    s.eng.explain_nodes_host(_hp(s.eng, E, opt, sched), m0, out, fm)
    s.eng.close()
    for t, node in enumerate(nodes):
        A, X, gt, pl, idx = _sub(s, node)
        _check(plan.dense_of(t, out), fm[t], s.w, (A, X, gt, pl, idx, s.w, dense[t]), dict(hp=_ohp(E, opt, sched), bn=bn))


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_wide_layers_graphs_match_port(case):
    seed, L, bn, hid, emb, d, C, opt, sched = case
    adj, feat, label, w, eng = _graph_setup(seed + 20, L, bn, False, hid, emb, d, C)
    gids = [0, 3, 5, 9, 11]
    n = adj.shape[1]
    dense = {g: O.draw_m0(n, seed=300 * seed + g) for g in gids}
    rc = {g: eng.graph_rows_cols(g) for g in gids}
    edge_off = eng.plan_graphs(gids)
    out = np.zeros(int(edge_off[-1]), np.float32)
    fm = np.zeros((len(gids), d), np.float32)
    E = 20
    eng.explain_graphs_host(_hp(eng, E, opt, sched), np.concatenate([dense[g][rc[g]] for g in gids]).astype(np.float32), out, fm)
    eng.close()
    for t, g in enumerate(gids):
        Dm = np.zeros((n, n))
        Dm[rc[g]] = out[edge_off[t]:edge_off[t + 1]]
        _check(Dm, fm[t], w, (np.asarray(adj[g], np.float64), feat[g], int(label[g]), None, 0, w, dense[g]),
               dict(hp=_ohp(E, opt, sched), bn=bn, graph_mode=True))


@pytest.mark.parametrize("case", [(31, 3, True, 256, 256, 16), (32, 5, False, 160, 136, 10), (33, 2, False, 256, 20, 300)],
                         ids=lambda c: "L%d%s_h%d_e%d_d%d" % (c[1], "_bn" if c[2] else "", c[3], c[4], c[5]))
def test_wide_layers_one_update_matches_fp64_port(case):
    """num_epochs = 2: one update; edge and feature masks within 1e-5 of the fp64 port (or 3 x the fp32 port's distance from it),
    node and graph mode."""
    seed, L, bn, hid, emb, d = case
    s = _node_setup(seed, L, bn, False, hid, emb, d, 4)
    nodes = list(range(0, 48, 5))
    plan = s.eng.plan_nodes(nodes, L)
    m0, dense = _m0(plan, 70)
    out = np.zeros(plan.total_edges, np.float32)
    fm = np.zeros((plan.count, d), np.float32)
    s.eng.explain_nodes_host(s.eng.make_hparams(num_epochs=2), m0, out, fm)
    s.eng.close()
    for t, node in enumerate(nodes):
        A, X, gt, pl, idx = _sub(s, node)
        ref, f1 = O.explain_dense_torch(A, X, gt, pl, idx, s.w, dense[t], O.default_hparams(num_epochs=2), bn=bn, dtype=torch.float64,
                                        return_feat=True)
        p32, f32 = O.explain_dense_torch(A, X, gt, pl, idx, s.w, dense[t], O.default_hparams(num_epochs=2), bn=bn, return_feat=True)
        assert O.rel_l2(plan.dense_of(t, out), ref) <= max(1e-5, 3 * O.rel_l2(p32, ref)), node
        assert np.abs(fm[t] - f1).max() <= max(1e-5, 3 * float(np.abs(f32 - f1).max())), node
    adj, feat, label, w, eng = _graph_setup(seed + 10, L, bn, False, hid, emb, d, 3)
    gids = list(range(12))
    n = adj.shape[1]
    dense = {g: O.draw_m0(n, seed=900 + g) for g in gids}
    rc = {g: eng.graph_rows_cols(g) for g in gids}
    edge_off = eng.plan_graphs(gids)
    out = np.zeros(int(edge_off[-1]), np.float32)
    fm = np.zeros((len(gids), d), np.float32)
    eng.explain_graphs_host(eng.make_hparams(num_epochs=2), np.concatenate([dense[g][rc[g]] for g in gids]).astype(np.float32), out, fm)
    eng.close()
    for t, g in enumerate(gids):
        args = (np.asarray(adj[g], np.float64), feat[g], int(label[g]), None, 0, w, dense[g], O.default_hparams(num_epochs=2))
        ref, f1 = O.explain_dense_torch(*args, graph_mode=True, bn=bn, dtype=torch.float64, return_feat=True)
        p32, f32 = O.explain_dense_torch(*args, graph_mode=True, bn=bn, return_feat=True)
        assert O.rel_l2(out[edge_off[t]:edge_off[t + 1]], ref[rc[g]]) <= max(1e-5, 3 * O.rel_l2(p32[rc[g]], ref[rc[g]])), g
        assert np.abs(fm[t] - f1).max() <= max(1e-5, 3 * float(np.abs(f32 - f1).max())), g


def test_wide_layers_large_subgraph_deterministic_and_order_free():
    """A hub whose 5-hop set has more than 1500 nodes, against the port; then Philox-initialised reruns are bit-identical, whatever
    the order of the batch."""
    s = _node_setup(41, 5, True, False, 144, 144, 12, 3, N=2000, m=2)
    hub = int(np.argmax(np.diff(s.rowptr)))
    plan = s.eng.plan_nodes([hub], 5)
    assert plan.n(0) > 1500
    m0, dense = _m0(plan, 9)
    out = np.zeros(plan.total_edges, np.float32)
    fm = np.zeros((1, 12), np.float32)
    s.eng.explain_nodes_host(s.eng.make_hparams(num_epochs=5), m0, out, fm)
    A, X, gt, pl, idx = _sub(s, hub)
    _check(plan.dense_of(0, out), fm[0], s.w, (A, X, gt, pl, idx, s.w, dense[0]), dict(hp=O.default_hparams(num_epochs=5), bn=True))
    nodes = [3, 17, hub, 120, 999]
    hp = s.eng.make_hparams(num_epochs=10, init=_abi.GX_INIT_PHILOX, seed=5)
    res = {}
    for order in (nodes, nodes[::-1], nodes):
        plan = s.eng.plan_nodes(order, 5)
        out = np.zeros(plan.total_edges, np.float32)
        fm = np.zeros((plan.count, 12), np.float32)
        s.eng.explain_nodes_host(hp, None, out, fm)
        for t, node in enumerate(order):
            got = np.concatenate([out[plan.edge_off[t]:plan.edge_off[t + 1]], fm[t]])
            if node in res:
                assert np.array_equal(res[node], got), node
            res[node] = got
    s.eng.close()


def test_wide_layers_graphs_deterministic_and_order_free():
    adj, feat, label, w, eng = _graph_setup(42, 4, True, False, 256, 256, 14, 3)
    hp = eng.make_hparams(num_epochs=30, init=_abi.GX_INIT_PHILOX, seed=11)
    res = {}
    for gids in ([0, 4, 7, 11], [11, 7, 4, 0], [0, 4, 7, 11]):
        edge_off = eng.plan_graphs(gids)
        out = np.zeros(int(edge_off[-1]), np.float32)
        fm = np.zeros((len(gids), 14), np.float32)
        eng.explain_graphs_host(hp, None, out, fm)
        for t, g in enumerate(gids):
            got = np.concatenate([out[edge_off[t]:edge_off[t + 1]], fm[t]])
            if g in res:
                assert np.array_equal(res[g], got), g
            res[g] = got
    eng.close()


def _pad_129(w, L):
    """A 128 / 128 model with one zero hidden / output column appended to every layer (zero weights and bias, zero pred_model column):
    the same function at width 129.  Without --bn: a zero column would enter the standardisation's statistics."""
    p = {}
    for l in range(1, L + 1):
        W = w["W%d" % l]
        rows = W.shape[0] + (1 if l > 1 else 0)
        P = np.zeros((rows, W.shape[1] + 1), np.float32)
        P[:W.shape[0], :W.shape[1]] = W
        p["W%d" % l] = P
        p["b%d" % l] = np.append(w["b%d" % l], np.float32(0))
    Wp = w["Wp"]
    p["Wp"] = np.insert(Wp, [128 * k for k in range(1, L + 1)], 0.0, axis=1).astype(np.float32)
    p["bp"] = w["bp"]
    return p


@pytest.mark.parametrize("graph_mode", [False, True])
def test_padded_128_model_agrees_with_narrow_kernel(graph_mode):
    """Old path against new path: the same model at 128 (KW = 4, per-row products) and zero-padded to 129 (the row-block path)."""
    L, d, E = 3, 12, 10
    w = random_model(np.random.default_rng(77), d, 128, 128, 3, L)
    wp = _pad_129(w, L)
    assert wp["Wp"].shape[1] == 3 * 129
    outs = []
    for weights in (w, wp):
        if graph_mode:
            eng = gnnx.Engine(0)
            eng.set_model(weights, num_layers=L)
            feat = (np.random.default_rng(5).normal(size=GG["adj"].shape[:2] + (d,)) * (GG["adj"].sum(2, keepdims=True) > 0)).astype(np.float32)
            eng.set_graph_batch(GG["adj"], feat, GG["label"])
            gids = list(range(12))
            edge_off = eng.plan_graphs(gids)
            m0 = np.concatenate([O.draw_m0(int(GG["max_nodes"]), seed=40 + g)[eng.graph_rows_cols(g)] for g in gids]).astype(np.float32)
            out = np.zeros(int(edge_off[-1]), np.float32)
            fm = np.zeros((len(gids), d), np.float32)
            eng.explain_graphs_host(eng.make_hparams(num_epochs=E), m0, out, fm)
        else:
            s = _node_setup(78, L, False, False, 128, 128, d, 3)
            s.eng.set_model(weights, num_layers=L)
            eng = s.eng
            plan = eng.plan_nodes(list(range(0, 48, 3)), L)
            m0, _ = _m0(plan, 11)
            out = np.zeros(plan.total_edges, np.float32)
            fm = np.zeros((plan.count, d), np.float32)
            eng.explain_nodes_host(eng.make_hparams(num_epochs=E), m0, out, fm)
        eng.close()
        outs.append((out, fm))
    assert O.rel_l2(outs[1][0], outs[0][0]) <= 1e-5
    assert O.rel_l2(outs[1][1], outs[0][1]) <= 1e-5


@pytest.mark.parametrize("L,bn,hid,emb,d", [(3, False, 256, 256, 16), (5, True, 160, 136, 10), (2, False, 20, 256, 300)])
def test_wide_layers_model_forward_matches_port(L, bn, hid, emb, d):
    """gx_model_forward with rows of 256 floats."""
    s = _node_setup(70 + L, L, bn, False, hid, emb, d, 4, N=300, m=3)
    got = s.eng.model_forward()
    s.eng.close()
    assert np.abs(got - s.pred).max() <= 2e-5 * max(1.0, np.abs(s.pred).max())


def test_wide_layers_refusals():
    s = _node_setup(61, 3, False, False, 256, 256, 10, 3)
    plan = s.eng.plan_nodes([0, 4], 3)
    m0, dense = _m0(plan, 3)
    out = np.zeros(plan.total_edges, np.float32)
    hp = s.eng.make_hparams(num_epochs=5)
    te = plan.total_edges
    calls = [lambda: s.eng.grad_nodes_host(out),
             lambda: s.eng.explain_nodes_ex(hp, m0, out, trace=np.zeros((2, 5, _abi.GX_TRACE_COLS), np.float32)),
             lambda: s.eng.explain_nodes_ex(hp, m0, out, state_out=dict(M=np.zeros(te, np.float32), m=np.zeros(te, np.float32),
                                                                         v=np.zeros(te, np.float32))),
             lambda: s.eng.explain_nodes_ex(s.eng.make_hparams(num_epochs=5, init=_abi.GX_INIT_STATE), m0, out,
                                            state_in=dict(m=np.zeros(te, np.float32), v=np.zeros(te, np.float32))),
             lambda: s.eng.explain_nodes_unconstrained(hp, np.concatenate([M.reshape(-1) for M in dense]).astype(np.float32), out)]
    for call in calls:
        with pytest.raises(_abi.GnnxError) as e:
            call()
        assert e.value.status == GX_ERR_UNSUPPORTED
    rng = np.random.default_rng(0)
    for hid, emb in ((257, 20), (20, 257)):
        with pytest.raises(_abi.GnnxError) as e:
            s.eng.set_model(random_model(rng, 10, hid, emb, 3, 3), num_layers=3)
        assert e.value.status == GX_ERR_UNSUPPORTED and "256" in str(e.value)
    wa = random_model(rng, 10, 160, 160, 3, 3, att=True)
    with pytest.raises(_abi.GnnxError) as e:
        s.eng.set_model(wa, num_layers=3, att=[wa["Wa%d" % l] for l in range(1, 4)])
    assert e.value.status == GX_ERR_UNSUPPORTED and "128" in str(e.value)
    s.eng.close()


# ------------------------------------------------------------------------------------------------------------------ the drop-in Explainer
def test_explainer_dropin_node_mode(tmp_path, capsys):
    """Explainer(pred=None) on a 256 / 256 model: predicted labels from gx_model_forward, masks against the port, the notice, the .npy
    files; unconstrained=True names the width."""
    L, hid, emb = 3, 256, 256
    s = _node_setup(81, L, True, False, hid, emb, 10, 4)
    s.eng.close()
    args = _args(tmp_path, L, True, False, hid, emb)
    model = gnnx.models.GcnEncoderNode(10, hid, emb, 4, L, bn=True, args=args)
    model.load_state_dict(_state_dict(model, s.w, L))
    ex = gnnx.Explainer(model=model, adj=torch.tensor(s.A[None], dtype=torch.float), feat=torch.tensor(s.feat[None]),
                        label=torch.tensor(s.label[None]), pred=None, train_idx=[], args=args, writer=None, print_training=True,
                        graph_mode=False, graph_idx=0)
    assert np.array_equal(ex._pred_label, s.pred_label)
    nodes = [2, 11, 30]
    torch.manual_seed(3)
    one = ex.explain(nodes[0], graph_idx=0)
    torch.manual_seed(3)
    many = ex.explain_nodes(nodes, args)
    assert np.array_equal(one, many[0])
    torch.manual_seed(3)
    for node, got in zip(nodes, many):
        A, X, gt, pl, idx = _sub(s, node)
        n = A.shape[0]
        M0 = O.draw_m0(n)
        hp = O.default_hparams(num_epochs=20)
        port = O.explain_dense_torch(A, X, s.label[node], pl, idx, s.w, M0, hp, bn=True)
        p64 = O.explain_dense_torch(A, X, s.label[node], pl, idx, s.w, M0, hp, bn=True, dtype=torch.float64)
        assert O.rel_l2(got, port) <= max(1e-4, 3 * O.rel_l2(p64, port)), node
    printed = capsys.readouterr().out
    assert "trace is not built for --bn / num_gc_layers != 3" in printed and "Saved adjacency matrix to" in printed
    assert any(f.startswith("masked_adj_syn1_") and f.endswith(".npy") for f in os.listdir(tmp_path))
    with pytest.raises(NotImplementedError, match="256"):
        ex.explain(nodes[0], graph_idx=0, unconstrained=True)


def test_explainer_dropin_graph_mode(tmp_path, capsys):
    L, C, d, hid, emb = 3, 3, 14, 256, 160
    adj, feat, label, w, eng = _graph_setup(91, L, False, False, hid, emb, d, C)
    eng.close()
    args = _args(tmp_path, L, False, True, hid, emb)
    model = gnnx.models.GcnEncoderGraph(d, hid, emb, C, L, bn=False, args=args)
    model.load_state_dict(_state_dict(model, w, L))
    ex = gnnx.Explainer(model=model, adj=torch.tensor(adj, dtype=torch.float), feat=torch.tensor(feat), label=torch.tensor(label),
                        pred=None, train_idx=[], args=args, writer=None, print_training=True, graph_mode=True, graph_idx=0)
    n = adj.shape[1]
    gids = [1, 3, 8]
    torch.manual_seed(4)
    got = ex.explain_graphs(gids)
    torch.manual_seed(4)
    for g, masked in zip(gids, got):
        M0 = O.draw_m0(n)
        A = np.asarray(adj[g], np.float64)
        hp = O.default_hparams(num_epochs=20)
        port = O.explain_dense_torch(A, feat[g], label[g], None, 0, w, M0, hp, graph_mode=True)
        p64 = O.explain_dense_torch(A, feat[g], label[g], None, 0, w, M0, hp, graph_mode=True, dtype=torch.float64)
        ei, ej = np.nonzero(A)
        assert masked.shape == (n, n)
        assert O.rel_l2(masked[ei, ej], port[ei, ej]) <= max(1e-4, 3 * O.rel_l2(p64[ei, ej], port[ei, ej])), g
    torch.manual_seed(4)
    one = ex.explain(0, graph_idx=gids[0], graph_mode=True)
    assert np.array_equal(one, got[0])
    assert "trace is not built for --bn / num_gc_layers != 3" in capsys.readouterr().out
    assert any(f.endswith(".npy") for f in os.listdir(tmp_path))
    with pytest.raises(NotImplementedError, match="256"):
        ex.explain(0, graph_idx=gids[0], graph_mode=True, unconstrained=True)


def test_wide_layers_sharded_explain_matches_explain_nodes(tmp_path):
    """gnnx.dist on a 256 / 256 model (one rank, gloo, the torch all-gather): the packed masks of explain_nodes_sharded equal
    Explainer.explain_nodes under the same torch seed."""
    import socket
    import torch.distributed as dist
    from gnnx import dist as gdist
    L, hid, emb = 3, 256, 256
    s = _node_setup(95, L, False, False, hid, emb, 10, 4)
    s.eng.close()
    args = _args(tmp_path, L, False, False, hid, emb)
    model = gnnx.models.GcnEncoderNode(10, hid, emb, 4, L, bn=False, args=args)
    model.load_state_dict(_state_dict(model, s.w, L))
    ex = gnnx.Explainer(model=model, adj=torch.tensor(s.A[None], dtype=torch.float), feat=torch.tensor(s.feat[None]),
                        label=torch.tensor(s.label[None]), pred=None, train_idx=[], args=args, writer=None, print_training=False,
                        graph_mode=False, graph_idx=0)
    nodes = [1, 9, 30, 47]
    torch.manual_seed(8)
    dense = ex.explain_nodes(nodes, args, save=False)
    sk = socket.socket(); sk.bind(("127.0.0.1", 0)); port = sk.getsockname()[1]; sk.close()
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=0, world_size=1)
    try:
        torch.manual_seed(8)
        values, offsets, _ = gdist.explain_nodes_sharded(ex, nodes, use_engine_comm=False)
    finally:
        dist.destroy_process_group()
    values = values.cpu().numpy()
    for t, Dn in enumerate(dense):
        ei, ej = np.nonzero(_sub(s, nodes[t])[0])
        assert np.array_equal(values[offsets[t]:offsets[t + 1]], Dn[ei, ej].astype(np.float32)), nodes[t]


# ---------------------------------------------------------------------------------------------------------- the unmodified reference
@pytest.mark.parametrize("case,mode", golden_cases(), ids=lambda c: str(c))
def test_wide_layers_match_reference_golden(case, mode):
    """Every node and graph of tests/golden/wide_layers_golden.npz within max(1e-4, 3 x the reference's own spread) of the reference's
    mask or, for the graphs with a near tie in their max-pool readout (tests/test_oracle_pool_ties.py), of the nearest admissible
    trajectory (tests/pool_oracle.py)."""
    g = np.load(GOLDEN)
    k = lambda s_: g["%s_%s" % (case, s_)]
    w = case_weights(g, case)
    L, bn = int(k("L")), bool(k("bn"))
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bn)
    hp = _hp(eng, int(k("epochs")), str(k("opt")))
    if mode == 0:
        rg = np.load(util.GOLDEN + "/rand_graph.npz")
        rowptr, col = O.csr_from_edges(int(rg["N"]), rg["edges"])
        eng.set_graph_csr(rowptr, col, rg["feat"].astype(np.float32), rg["label"].astype(np.int32), np.argmax(k("pred"), 1).astype(np.int32))
        nodes = [int(v) for v in k("nodes")]
        plan = eng.plan_nodes(nodes, L)
        m0 = np.empty(plan.total_edges, np.float32)
        for t, node in enumerate(nodes):
            assert np.array_equal(plan.neighbors_of(t), g["%s_n%d_nbrs" % (case, node)])
            r, c = plan.rows_cols_of(t)
            m0[plan.edge_off[t]:plan.edge_off[t + 1]] = O.draw_m0(plan.n(t), seed=int(g["%s_n%d_seed" % (case, node)]))[r, c]
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_host(hp, m0, out)
        for t, node in enumerate(nodes):
            tol = max(1e-4, 3 * float(g["%s_n%d_spread" % (case, node)]))
            err = util.rel_l2(out[plan.edge_off[t]:plan.edge_off[t + 1]], g["%s_n%d_mask" % (case, node)])
            assert err <= tol, (case, node, err, tol)
    else:
        G, n = int(GG["num_graphs"]), int(GG["max_nodes"])
        eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
        gids = list(range(G))
        edge_off = eng.plan_graphs(gids)
        rc = [eng.graph_rows_cols(gi) for gi in gids]
        m0 = np.concatenate([O.draw_m0(n, seed=int(GG["g%d_seed" % gi]))[rc[gi]] for gi in gids]).astype(np.float32)
        out = np.zeros(int(edge_off[-1]), np.float32)
        eng.explain_graphs_host(hp, m0, out)
        for gi in gids:
            Dm = np.zeros((n, n))
            Dm[rc[gi]] = out[edge_off[gi]:edge_off[gi + 1]]
            ei, ej = np.nonzero(GG["adj"][gi])
            tol = max(1e-4, 3 * float(g["%s_g%d_spread" % (case, gi)]))
            err = util.rel_l2(Dm[ei, ej], g["%s_g%d_mask" % (case, gi)])
            if gi in NEAR_TIES.get(("wide_layers", case), {}):   # a sub-ulp arg-max margin: the nearest admissible trajectory
                A = np.asarray(GG["adj"][gi], np.float64)
                err = PO.nearest_admissible(Dm[ei, ej], g["%s_g%d_mask" % (case, gi)], A, GG["feat"][gi].astype(np.float32),
                                            int(GG["label"][gi]), w, O.draw_m0(n, seed=int(GG["g%d_seed" % gi])),
                                            O.default_hparams(num_epochs=int(k("epochs")), opt=str(k("opt"))), bn)
            assert err <= tol, (case, gi, err, tol)
    eng.close()


@pytest.mark.parametrize("case", [c for c, mode in golden_cases() if mode == 0])
def test_wide_layers_model_forward_matches_reference_pred(case):
    """gx_model_forward against the reference model's own predictions on the rand graph."""
    g = np.load(GOLDEN)
    k = lambda s_: g["%s_%s" % (case, s_)]
    rg = np.load(util.GOLDEN + "/rand_graph.npz")
    rowptr, col = O.csr_from_edges(int(rg["N"]), rg["edges"])
    eng = gnnx.Engine(0)
    eng.set_model(case_weights(g, case), num_layers=int(k("L")), bn=bool(k("bn")))
    eng.set_graph_csr(rowptr, col, rg["feat"].astype(np.float32), rg["label"].astype(np.int32), np.zeros(int(rg["N"]), np.int32))
    got = eng.model_forward()
    eng.close()
    ref = k("pred")
    assert np.abs(got - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max()), case
