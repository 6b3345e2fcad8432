"""Attention models (--method att) on the GPU: explain_var.cu's attention path through the C ABI and the drop-in Explainer, node and
graph mode, against the port (oracle/gnnx_oracle.explain_dense_torch) in fp32 and fp64."""
import os
import types

import numpy as np
import pytest
import torch

import gnnx
import gnnx_oracle as O
import util
from gnnx import _abi
from test_oracle_att import random_att_model

pytestmark = pytest.mark.gpu
GX_ERR_UNSUPPORTED = -3


def _ba_graph(seed, N, m=2):
    import networkx as nx
    G = nx.barabasi_albert_graph(N, m, seed=seed)
    return O.csr_from_edges(N, np.array(G.edges(), dtype=np.int64))


def _node_setup(seed, L, bn, hid, emb, d, C, N=48, m=2):
    rng = np.random.default_rng(seed)
    rowptr, col = _ba_graph(seed, N, m)
    A = O.dense_from_csr(rowptr, col)
    feat = rng.normal(size=(N, d)).astype(np.float32)
    label = rng.integers(0, C, N).astype(np.int32)
    w = random_att_model(rng, d, hid, emb, C, L)
    pred = O.model_pred(A, feat, w, bn=bn)
    pred_label = np.argmax(pred, 1).astype(np.int32)
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bn, att=[w["Wa%d" % l] for l in range(1, L + 1)])
    eng.set_graph_csr(rowptr, col, feat, label, pred_label)
    return types.SimpleNamespace(rng=rng, rowptr=rowptr, col=col, A=A, feat=feat, label=label, w=w, pred=pred, pred_label=pred_label,
                                 eng=eng, L=L, bn=bn, d=d)


def _m0(s, plan, seed):
    m0 = np.empty(plan.total_edges, np.float32)
    dense = []
    for t in range(plan.count):
        M0 = O.draw_m0(plan.n(t), seed=seed + t)
        r, c = plan.rows_cols_of(t)
        m0[plan.edge_off[t]:plan.edge_off[t + 1]] = M0[r, c]
        dense.append(M0)
    return m0, dense


def _sub(s, node):
    idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(s.rowptr, s.col, s.feat, s.label, node, s.L)
    return O.dense_from_csr(srp, scol), sfeat, slabel[idx], s.pred_label[nbrs], idx


RANDOM = [  # seed, L, bn, hid, emb, d, C, opt, scheduler
    (1, 3, False, 20, 20, 7, 4, "adam", "none"),
    (2, 2, True, 20, 20, 10, 3, "adam", "none"),
    (3, 4, False, 33, 33, 7, 4, "sgd", "none"),
    (4, 3, True, 64, 64, 128, 5, "rmsprop", "none"),
    (5, 4, True, 128, 128, 7, 3, "adagrad", "none"),
    (6, 2, False, 20, 33, 128, 2, "adam", "step"),
    (7, 3, False, 64, 20, 20, 4, "adam", "cos"),
]


@pytest.mark.parametrize("case", RANDOM, ids=lambda c: "s%d_L%d%s_h%d_e%d_d%d_%s_%s" % (c[0], c[1], "_bn" if c[2] else "", c[3], c[4], c[5],
                                                                                       c[7], c[8]))
def test_att_nodes_match_port(case):
    seed, L, bn, hid, emb, d, C, opt, sched = case
    s = _node_setup(seed, L, bn, hid, emb, d, C)
    nodes = [0, 7, 23, 47]
    plan = s.eng.plan_nodes(nodes, L)
    m0, dense = _m0(s, plan, 500 * seed)
    E = 20
    over = dict(opt=opt, opt_scheduler=sched, opt_decay_step=5, opt_decay_rate=0.5, opt_restart=8)
    hp = s.eng.make_hparams(num_epochs=E)
    hp.opt = _abi.GX_OPT[opt]; hp.opt_scheduler = _abi.GX_SCHED[sched]
    hp.opt_decay_step, hp.opt_decay_rate, hp.opt_restart = 5, 0.5, 8
    out = np.zeros(plan.total_edges, np.float32)
    fm = np.zeros((plan.count, d), np.float32)
    s.eng.explain_nodes_host(hp, m0, out, fm)
    for t, node in enumerate(nodes):
        A, X, gt, pl, idx = _sub(s, node)
        ohp = O.default_hparams(num_epochs=E, **over)
        port = O.explain_dense_torch(A, X, gt, pl, idx, s.w, dense[t], ohp, bn=bn)
        p64 = O.explain_dense_torch(A, X, gt, pl, idx, s.w, dense[t], ohp, bn=bn, dtype=torch.float64)
        tol = max(1e-4, 3 * O.rel_l2(p64, port))
        err = O.rel_l2(plan.dense_of(t, out), port)
        assert err <= tol, (node, err, tol)
    assert np.isfinite(fm).all() and (fm > 0).all() and (fm < 1).all()
    s.eng.close()


@pytest.mark.parametrize("seed,L,bn,hid,d", [(11, 3, False, 20, 7), (12, 2, True, 20, 10), (13, 4, True, 33, 128), (14, 3, False, 128, 64)])
def test_att_one_update_matches_fp64_spec(seed, L, bn, hid, d):
    """num_epochs = 2: one update; the mask and the feature mask against the fp64 port within 1e-5."""
    s = _node_setup(seed, L, bn, hid, hid, d, 4)
    nodes = list(range(0, 48, 5))
    plan = s.eng.plan_nodes(nodes, L)
    m0, dense = _m0(s, plan, 70 * seed)
    out = np.zeros(plan.total_edges, np.float32)
    fm = np.zeros((plan.count, d), np.float32)
    s.eng.explain_nodes_host(s.eng.make_hparams(num_epochs=2), m0, out, fm)
    for t, node in enumerate(nodes):
        A, X, gt, pl, idx = _sub(s, node)
        ref, f1 = O.explain_dense_torch(A, X, gt, pl, idx, s.w, dense[t], O.default_hparams(num_epochs=2), bn=bn, dtype=torch.float64,
                                       return_feat=True)
        assert O.rel_l2(plan.dense_of(t, out), ref) <= 1e-5, node
        assert np.abs(fm[t] - f1).max() <= 1e-5, node   # the feature mask after the one update
    s.eng.close()


def test_att_large_subgraph_deterministic_and_order_free():
    s = _node_setup(21, 2, False, 20, 20, 8, 3, N=4000, m=3)   # the hub's 2-hop set has 1910 nodes
    deg = np.diff(s.rowptr)
    hub = int(np.argmax(deg))
    plan = s.eng.plan_nodes([hub], 2)
    assert plan.n(0) >= 1500
    m0, dense = _m0(s, plan, 9)
    out = np.zeros(plan.total_edges, np.float32)
    s.eng.explain_nodes_host(s.eng.make_hparams(num_epochs=5), m0, out)
    A, X, gt, pl, idx = _sub(s, hub)
    ohp = O.default_hparams(num_epochs=5)
    port = O.explain_dense_torch(A, X, gt, pl, idx, s.w, dense[0], ohp)
    p64 = O.explain_dense_torch(A, X, gt, pl, idx, s.w, dense[0], ohp, dtype=torch.float64)
    assert O.rel_l2(plan.dense_of(0, out), port) <= max(1e-4, 3 * O.rel_l2(p64, port))
    # determinism and independence of the batch order (Philox init: keyed by node and slot)
    nodes = [3, 17, hub, 120, 999]
    hp = s.eng.make_hparams(num_epochs=30, init=_abi.GX_INIT_PHILOX, seed=5)
    res = {}
    for order in (nodes, nodes[::-1], nodes):
        plan = s.eng.plan_nodes(order, 2)
        out = np.zeros(plan.total_edges, np.float32)
        s.eng.explain_nodes_host(hp, None, out)
        for t, node in enumerate(order):
            got = out[plan.edge_off[t]:plan.edge_off[t + 1]].copy()
            if node in res:
                assert np.array_equal(res[node], got), node
            res[node] = got
    s.eng.close()


def test_att_philox_init_matches_non_att_path():
    """num_epochs = 1 returns sigmoid-symmetrised M0: the attention model draws the same Philox numbers as the plain variant."""
    s = _node_setup(31, 3, True, 20, 20, 7, 3)
    plain = gnnx.Engine(0)
    plain.set_model(s.w, num_layers=3, bn=True)
    plain.set_graph_csr(s.rowptr, s.col, s.feat, s.label, s.pred_label)
    nodes = [0, 5, 9]
    outs = []
    for eng in (s.eng, plain):
        plan = eng.plan_nodes(nodes, 3)
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_host(eng.make_hparams(num_epochs=1, init=_abi.GX_INIT_PHILOX, seed=77), None, out)
        outs.append(out)
    assert np.array_equal(outs[0], outs[1])
    s.eng.close(); plain.close()


@pytest.mark.parametrize("L,bn,d", [(3, False, 7), (2, True, 10), (4, True, 128)])
def test_att_model_forward_matches_port(L, bn, d):
    s = _node_setup(40 + L, L, bn, 20, 20, d, 4)
    got = s.eng.model_forward()
    assert np.abs(got - s.pred).max() <= 2e-5 * max(1.0, np.abs(s.pred).max())
    s.eng.close()


def test_att_refusals():
    s = _node_setup(51, 3, False, 20, 20, 7, 3)
    plan = s.eng.plan_nodes([0, 4], 3)
    m0, _ = _m0(s, plan, 3)
    out = np.zeros(plan.total_edges, np.float32)
    hp = s.eng.make_hparams(num_epochs=5)
    with pytest.raises(_abi.GnnxError) as e:
        s.eng.grad_nodes_host(out)
    assert e.value.status == GX_ERR_UNSUPPORTED
    with pytest.raises(_abi.GnnxError) as e:
        s.eng.explain_nodes_ex(hp, m0, out, trace=np.zeros((2, 5, _abi.GX_TRACE_COLS), np.float32))
    assert e.value.status == GX_ERR_UNSUPPORTED
    te = plan.total_edges
    with pytest.raises(_abi.GnnxError) as e:
        s.eng.explain_nodes_ex(s.eng.make_hparams(num_epochs=5, init=_abi.GX_INIT_STATE), m0, out,
                               state_in=dict(m=np.zeros(te, np.float32), v=np.zeros(te, np.float32)))
    assert e.value.status == GX_ERR_UNSUPPORTED
    with pytest.raises(_abi.GnnxError) as e:
        s.eng.explain_nodes_unconstrained(hp, None, out)
    assert e.value.status == GX_ERR_UNSUPPORTED
    s.eng.close()


def _args(tmp_path, L, bn, graph):
    return types.SimpleNamespace(num_gc_layers=L, num_epochs=20, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                 mask_bias=False, gpu=False, bias=True, bn=bn, method="att", dataset="graphs" if graph else "syn1",
                                 bmname=None, hidden_dim=20, output_dim=20, name_suffix="", explainer_suffix="", logdir=str(tmp_path))


def _reference_state_dict(model, w, L):
    keys = ["conv_first"] + ["conv_block.%d" % i for i in range(L - 2)] + ["conv_last"]
    sd = {}
    for l, k in enumerate(keys, 1):
        sd[k + ".weight"] = w["W%d" % l]; sd[k + ".att_weight"] = w["Wa%d" % l]; sd[k + ".bias"] = w["b%d" % l]
    sd["pred_model.weight"] = w["Wp"]; sd["pred_model.bias"] = w["bp"]
    assert set(sd) == set(model.state_dict())
    return {k: torch.tensor(v) for k, v in sd.items()}


@pytest.mark.parametrize("L,bn", [(3, False), (2, True)])
def test_explainer_dropin_node_mode(tmp_path, capsys, L, bn):
    s = _node_setup(60 + L, L, bn, 20, 20, 7, 4)
    s.eng.close()
    args = _args(tmp_path, L, bn, False)
    model = gnnx.models.GcnEncoderNode(7, 20, 20, 4, L, bn=bn, args=args)
    assert model.att and all(hasattr(m, "att_weight") for m in model.modules() if isinstance(m, gnnx.models.GraphConv))
    model.load_state_dict(_reference_state_dict(model, s.w, L))
    adj = torch.tensor(s.A[None], dtype=torch.float)
    ex = gnnx.Explainer(model=model, adj=adj, feat=torch.tensor(s.feat[None]), label=torch.tensor(s.label[None]), pred=None,
                        train_idx=[], args=args, writer=None, print_training=True, graph_mode=False, graph_idx=0)
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
        port = O.explain_dense_torch(A, X, s.label[node], pl, idx, s.w, M0, O.default_hparams(num_epochs=20), bn=bn)
        p64 = O.explain_dense_torch(A, X, s.label[node], pl, idx, s.w, M0, O.default_hparams(num_epochs=20), bn=bn, dtype=torch.float64)
        assert O.rel_l2(got, port) <= max(1e-4, 3 * O.rel_l2(p64, port)), node
    printed = capsys.readouterr().out
    assert "trace is not built for attention models" in printed and "Saved adjacency matrix to" in printed
    assert any(f.startswith("masked_adj_syn1_att_") and f.endswith(".npy") for f in os.listdir(tmp_path))
    with pytest.raises(NotImplementedError):
        ex.explain(nodes[0], unconstrained=True)
    with pytest.raises(NotImplementedError):
        ex.explain(nodes[0], model="att")


def test_explainer_dropin_graph_mode(tmp_path, capsys):
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    d, C, L = gg["feat"].shape[2], 2, 3
    rng = np.random.default_rng(70)
    w = random_att_model(rng, d, 20, 20, C, L)
    args = _args(tmp_path, L, False, True)
    model = gnnx.models.GcnEncoderGraph(d, 20, 20, C, L, bn=False, args=args)
    model.load_state_dict(_reference_state_dict(model, w, L))
    label = np.asarray(gg["label"]) % C
    ex = gnnx.Explainer(model=model, adj=torch.tensor(gg["adj"], dtype=torch.float), feat=torch.tensor(gg["feat"]),
                        label=torch.tensor(label), pred=None, train_idx=[], args=args, writer=None, print_training=True,
                        graph_mode=True, graph_idx=0)
    n = int(gg["max_nodes"])
    gids = [1, 3, 8]
    torch.manual_seed(4)
    got = ex.explain_graphs(gids)
    torch.manual_seed(4)
    for g, masked in zip(gids, got):
        M0 = O.draw_m0(n)
        A = np.asarray(gg["adj"][g], np.float64)
        port = O.explain_dense_torch(A, gg["feat"][g], label[g], None, 0, w, M0, O.default_hparams(num_epochs=20), graph_mode=True)
        p64 = O.explain_dense_torch(A, gg["feat"][g], label[g], None, 0, w, M0, O.default_hparams(num_epochs=20), graph_mode=True,
                                   dtype=torch.float64)
        ei, ej = np.nonzero(A)
        assert masked.shape == (n, n)
        assert O.rel_l2(masked[ei, ej], port[ei, ej]) <= max(1e-4, 3 * O.rel_l2(p64[ei, ej], port[ei, ej])), g
    torch.manual_seed(4)
    one = ex.explain(0, graph_idx=gids[0], graph_mode=True)
    assert np.array_equal(one, got[0])
    assert "trace is not built for attention models" in capsys.readouterr().out
    assert any(f.endswith(".npy") for f in os.listdir(tmp_path))
    with pytest.raises(NotImplementedError):
        ex.explain(0, graph_idx=1, graph_mode=True, unconstrained=True)


# ---------------------------------------------------------------------------------------------------------- the unmodified reference
from test_oracle_att import GOLDEN, case_weights, fixture_graph, golden_cases  # noqa: E402


def _att_list(w, L):
    return [w["Wa%d" % l] for l in range(1, L + 1)]


@pytest.mark.parametrize("case,mode", golden_cases(), ids=lambda c: str(c))
def test_att_matches_reference_golden(case, mode):
    """Every node and graph of tests/golden/att_golden.npz within max(1e-4, 3 x the reference's own spread)."""
    g = np.load(GOLDEN)
    k = lambda s_: g["%s_%s" % (case, s_)]
    w = case_weights(g, case)
    L, bn = int(k("L")), bool(k("bn"))
    hp_of = lambda eng: eng.make_hparams(num_epochs=int(k("epochs")))
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bn, att=_att_list(w, L))
    if mode == 0:
        rowptr, col, _, label = fixture_graph(str(k("graph")))
        eng.set_graph_csr(rowptr, col, k("feat"), label, np.argmax(k("pred"), 1).astype(np.int32))
        nodes = [int(v) for v in k("nodes")]
        plan = eng.plan_nodes(nodes, L)
        m0 = np.empty(plan.total_edges, np.float32)
        for t, node in enumerate(nodes):
            assert np.array_equal(plan.neighbors_of(t), g["%s_n%d_nbrs" % (case, node)])
            r, c = plan.rows_cols_of(t)
            m0[plan.edge_off[t]:plan.edge_off[t + 1]] = O.draw_m0(plan.n(t), seed=int(g["%s_n%d_seed" % (case, node)]))[r, c]
        hp = hp_of(eng)
        hp.opt = _abi.GX_OPT[str(k("opt"))]
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_host(hp, m0, out)
        for t, node in enumerate(nodes):   # edge slots in row-major order, as the reference's nonzero entries
            tol = max(1e-4, 3 * float(g["%s_n%d_spread" % (case, node)]))
            err = util.rel_l2(out[plan.edge_off[t]:plan.edge_off[t + 1]], g["%s_n%d_mask" % (case, node)])
            assert err <= tol, (case, node, err, tol)
    else:
        gg = np.load(util.GOLDEN + "/graphs_golden.npz")
        G, n = int(gg["num_graphs"]), int(gg["max_nodes"])
        eng.set_graph_batch(gg["adj"], gg["feat"], gg["label"])
        gids = list(range(G))
        edge_off = eng.plan_graphs(gids)
        rc = [eng.graph_rows_cols(gi) for gi in gids]
        m0 = np.concatenate([O.draw_m0(n, seed=int(gg["g%d_seed" % gi]))[rc[gi]] for gi in gids]).astype(np.float32)
        out = np.zeros(int(edge_off[-1]), np.float32)
        eng.explain_graphs_host(hp_of(eng), m0, out)
        for gi in gids:
            D = np.zeros((n, n))
            D[rc[gi]] = out[edge_off[gi]:edge_off[gi + 1]]
            ei, ej = np.nonzero(gg["adj"][gi])
            tol = max(1e-4, 3 * float(g["%s_g%d_spread" % (case, gi)]))
            err = util.rel_l2(D[ei, ej], g["%s_g%d_mask" % (case, gi)])
            assert err <= tol, (case, gi, err, tol)
    eng.close()


@pytest.mark.parametrize("case", [c for c, mode in golden_cases() if mode == 0])
def test_att_model_forward_matches_reference_pred(case):
    """gx_model_forward against the reference model's own predictions, on the fixture graph and with a self loop on every node
    (the raw adjacency keeps s_ii)."""
    g = np.load(GOLDEN)
    k = lambda s_: g["%s_%s" % (case, s_)]
    w = case_weights(g, case)
    L, bn = int(k("L")), bool(k("bn"))
    if int(k("hid")) > 32:
        pytest.skip("gx_model_forward builds widths up to 32")
    rowptr, col, A, label = fixture_graph(str(k("graph")))
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bn, att=_att_list(w, L))
    for adj, ref in ((A, k("pred")), (A + np.eye(len(A), dtype=A.dtype), k("pred_loop"))):
        rp, cl = O.csr_from_dense(adj)
        eng.set_graph_csr(rp, cl, k("feat"), label, np.zeros(len(A), np.int32))
        got = eng.model_forward()
        assert np.abs(got - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max()), case
    eng.close()


def test_att_sharded_explain_matches_explain_nodes(tmp_path):
    """gnnx.dist on an attention model (one rank, gloo, the torch all-gather): the packed masks of explain_nodes_sharded equal
    Explainer.explain_nodes under the same torch seed."""
    import socket
    import torch.distributed as dist
    from gnnx import dist as gdist
    s = _node_setup(81, 3, False, 20, 20, 7, 4)
    s.eng.close()
    args = _args(tmp_path, 3, False, False)
    model = gnnx.models.GcnEncoderNode(7, 20, 20, 4, 3, bn=False, args=args)
    model.load_state_dict(_reference_state_dict(model, s.w, 3))
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
    for t, D in enumerate(dense):   # the packed entries are the row-major sub-adjacency slots
        ei, ej = np.nonzero(_sub(s, nodes[t])[0])
        assert np.array_equal(values[offsets[t]:offsets[t + 1]], D[ei, ej].astype(np.float32)), nodes[t]
