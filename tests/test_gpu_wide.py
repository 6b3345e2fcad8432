"""GPU (-m gpu): inputs wider than 128 features (explain_var.cu's wide path, 129 <= d <= 4096) through the C ABI, the drop-in Explainer
and gnnx.dist, node and graph mode, against the torch port (oracle/gnnx_oracle.explain_dense_torch) in fp32 and fp64."""
import os
import types

import numpy as np
import pytest
import torch

import gnnx
import gnnx_oracle as O
import util
from gnnx import _abi

pytestmark = pytest.mark.gpu
GX_ERR_UNSUPPORTED = -3


def random_model(rng, d, hid, emb, C, L):
    """A model whose layer-1 pre-activations stay O(1) at any d (W1 scaled by 1 / sqrt(d))."""
    dims = [d] + [hid] * (L - 1) + [emb]
    w = {}
    for l in range(1, L + 1):
        w["W%d" % l] = (rng.normal(size=(dims[l - 1], dims[l])) * (0.5 if l > 1 else 2.0 / np.sqrt(d))).astype(np.float32)
        w["b%d" % l] = (rng.normal(size=dims[l]) * 0.5).astype(np.float32)
    w["Wp"] = (rng.normal(size=(C, hid * (L - 1) + emb)) * 0.5).astype(np.float32)
    w["bp"] = (rng.normal(size=C) * 0.5).astype(np.float32)
    return w


def _node_setup(seed, L, bn, hid, emb, d, C, N=48, m=2):
    import networkx as nx
    rng = np.random.default_rng(seed)
    rowptr, col = O.csr_from_edges(N, np.array(nx.barabasi_albert_graph(N, m, seed=seed).edges(), dtype=np.int64))
    A = O.dense_from_csr(rowptr, col)
    feat = rng.normal(size=(N, d)).astype(np.float32)
    label = rng.integers(0, C, N).astype(np.int32)
    w = random_model(rng, d, hid, emb, C, L)
    with torch.no_grad():
        pred = O._gcn_forward_torch(torch.tensor(feat[None]), torch.tensor(A[None], dtype=torch.float), O.weights_to_torch(w, False),
                                    False, bn=bn)[0].numpy()
    pred_label = np.argmax(pred, 1).astype(np.int32)
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bn)
    eng.set_graph_csr(rowptr, col, feat, label, pred_label)
    return types.SimpleNamespace(rowptr=rowptr, col=col, A=A, feat=feat, label=label, w=w, pred=pred, pred_label=pred_label, eng=eng,
                                 L=L, bn=bn, d=d)


def _m0(plan, seed):
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


def _hp(eng, E, opt="adam", sched="none", **over):
    hp = eng.make_hparams(num_epochs=E, **over)
    hp.opt = _abi.GX_OPT[opt]; hp.opt_scheduler = _abi.GX_SCHED[sched]
    hp.opt_decay_step, hp.opt_decay_rate, hp.opt_restart = 5, 0.5, 8
    return hp


def _ohp(E, opt="adam", sched="none"):
    return O.default_hparams(num_epochs=E, opt=opt, opt_scheduler=sched, opt_decay_step=5, opt_decay_rate=0.5, opt_restart=8)


def _check(got, fm, port_args, port_kw):
    """Edge mask within max(1e-4, 3 x the port's fp32 / fp64 distance); feature mask within max(1e-4, 3 x the same distance on it)."""
    port, f32 = O.explain_dense_torch(*port_args, return_feat=True, **port_kw)
    p64, f64 = O.explain_dense_torch(*port_args, return_feat=True, dtype=torch.float64, **port_kw)
    tol = max(1e-4, 3 * O.rel_l2(p64, port))
    err = O.rel_l2(got, port)
    assert err <= tol, ("edge mask", err, tol)
    ftol = max(1e-4, 3 * float(np.abs(f64 - f32).max()))
    ferr = float(np.abs(fm - f32).max())
    assert ferr <= ftol, ("feature mask", ferr, ftol)


NODE_CASES = [  # seed, L, bn, hid, emb, d, C, opt, scheduler
    (1, 3, False, 20, 20, 129, 4, "adam", "none"),
    (2, 2, True, 20, 20, 200, 3, "sgd", "none"),
    (3, 4, False, 64, 33, 513, 4, "rmsprop", "step"),
    (4, 3, True, 128, 128, 1433, 5, "adagrad", "cos"),
    (5, 2, False, 33, 20, 4096, 3, "sgd", "cos"),   # (Adam on 4096 weak feature gradients is chaotic: the port's own fp32 / fp64 runs part)
    (6, 4, True, 40, 40, 300, 3, "adam", "step"),
]


@pytest.mark.parametrize("case", NODE_CASES, ids=lambda c: "s%d_L%d%s_h%d_e%d_d%d_%s_%s" % (c[0], c[1], "_bn" if c[2] else "", c[3], c[4],
                                                                                            c[5], c[7], c[8]))
def test_wide_nodes_match_port(case):
    seed, L, bn, hid, emb, d, C, opt, sched = case
    s = _node_setup(seed, L, bn, hid, emb, d, C)
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
        _check(plan.dense_of(t, out), fm[t], (A, X, gt, pl, idx, s.w, dense[t]), dict(hp=_ohp(E, opt, sched), bn=bn))


GRAPH_CASES = [  # seed, L, bn, hid, emb, d, C, opt, scheduler
    (11, 3, False, 20, 20, 190, 3, "adam", "none"),
    (12, 4, True, 64, 48, 300, 4, "sgd", "step"),
    (13, 2, True, 128, 128, 1433, 2, "rmsprop", "cos"),
    (14, 3, False, 33, 33, 4096, 3, "adagrad", "none"),
]


def _graph_setup(seed, L, bn, hid, emb, d, C):
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    rng = np.random.default_rng(seed)
    adj = gg["adj"]
    labels = rng.integers(0, d, size=adj.shape[:2])
    feat = (np.eye(d, dtype=np.float32)[labels] * (adj.sum(2, keepdims=True) > 0)).astype(np.float32)   # one-hot node labels
    label = np.asarray(gg["label"]) % C
    w = random_model(rng, d, hid, emb, C, L)
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bn)
    eng.set_graph_batch(adj, feat, label)
    return adj, feat, label, w, eng


@pytest.mark.parametrize("case", GRAPH_CASES, ids=lambda c: "s%d_L%d%s_h%d_d%d_%s_%s" % (c[0], c[1], "_bn" if c[2] else "", c[3], c[5],
                                                                                         c[7], c[8]))
def test_wide_graphs_match_port(case):
    seed, L, bn, hid, emb, d, C, opt, sched = case
    adj, feat, label, w, eng = _graph_setup(seed, L, bn, hid, emb, d, C)
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
        D = np.zeros((n, n))
        D[rc[g]] = out[edge_off[t]:edge_off[t + 1]]
        _check(D, fm[t], (np.asarray(adj[g], np.float64), feat[g], int(label[g]), None, 0, w, dense[g]),
               dict(hp=_ohp(E, opt, sched), bn=bn, graph_mode=True))


def test_wide_one_update_matches_fp64_port():
    """num_epochs = 2: one update; edge and feature masks within 1e-5 of the fp64 port, node and graph mode."""
    s = _node_setup(21, 3, True, 40, 40, 300, 4)
    nodes = list(range(0, 48, 5))
    plan = s.eng.plan_nodes(nodes, 3)
    m0, dense = _m0(plan, 70)
    out = np.zeros(plan.total_edges, np.float32)
    fm = np.zeros((plan.count, 300), np.float32)
    s.eng.explain_nodes_host(s.eng.make_hparams(num_epochs=2), m0, out, fm)
    s.eng.close()
    for t, node in enumerate(nodes):
        A, X, gt, pl, idx = _sub(s, node)
        ref, f1 = O.explain_dense_torch(A, X, gt, pl, idx, s.w, dense[t], O.default_hparams(num_epochs=2), bn=True, dtype=torch.float64,
                                   return_feat=True)
        assert O.rel_l2(plan.dense_of(t, out), ref) <= 1e-5, node
        assert np.abs(fm[t] - f1).max() <= 1e-5, node
    adj, feat, label, w, eng = _graph_setup(22, 4, True, 20, 20, 190, 3)
    gids = list(range(12))
    n = adj.shape[1]
    dense = {g: O.draw_m0(n, seed=900 + g) for g in gids}
    rc = {g: eng.graph_rows_cols(g) for g in gids}
    edge_off = eng.plan_graphs(gids)
    out = np.zeros(int(edge_off[-1]), np.float32)
    fm = np.zeros((len(gids), 190), np.float32)
    eng.explain_graphs_host(eng.make_hparams(num_epochs=2), np.concatenate([dense[g][rc[g]] for g in gids]).astype(np.float32), out, fm)
    eng.close()
    for t, g in enumerate(gids):
        ref, f1 = O.explain_dense_torch(np.asarray(adj[g], np.float64), feat[g], int(label[g]), None, 0, w, dense[g],
                                   O.default_hparams(num_epochs=2), graph_mode=True, bn=True, dtype=torch.float64, return_feat=True)
        assert O.rel_l2(out[edge_off[t]:edge_off[t + 1]], ref[rc[g]]) <= 1e-5, g
        assert np.abs(fm[t] - f1).max() <= 1e-5, g


def test_wide_large_subgraph_deterministic_and_order_free():
    s = _node_setup(31, 2, False, 20, 20, 200, 3, N=4000, m=3)   # the hub's 2-hop set has more than 1500 nodes
    hub = int(np.argmax(np.diff(s.rowptr)))
    plan = s.eng.plan_nodes([hub], 2)
    assert plan.n(0) >= 1500
    m0, dense = _m0(plan, 9)
    out = np.zeros(plan.total_edges, np.float32)
    fm = np.zeros((1, 200), np.float32)
    s.eng.explain_nodes_host(s.eng.make_hparams(num_epochs=5), m0, out, fm)
    A, X, gt, pl, idx = _sub(s, hub)
    _check(plan.dense_of(0, out), fm[0], (A, X, gt, pl, idx, s.w, dense[0]), dict(hp=O.default_hparams(num_epochs=5)))
    nodes = [3, 17, hub, 120, 999]
    hp = s.eng.make_hparams(num_epochs=30, init=_abi.GX_INIT_PHILOX, seed=5)
    res = {}
    for order in (nodes, nodes[::-1], nodes):
        plan = s.eng.plan_nodes(order, 2)
        out = np.zeros(plan.total_edges, np.float32)
        fm = np.zeros((plan.count, 200), np.float32)
        s.eng.explain_nodes_host(hp, None, out, fm)
        for t, node in enumerate(order):
            got = np.concatenate([out[plan.edge_off[t]:plan.edge_off[t + 1]], fm[t]])
            if node in res:
                assert np.array_equal(res[node], got), node
            res[node] = got
    s.eng.close()


def test_wide_philox_init():
    """num_epochs = 1 returns (sigmoid(M0_ij) + sigmoid(M0_ji)) / 2 of the Philox draws (gnnx_oracle.philox_m0), graph mode."""
    adj, feat, label, w, eng = _graph_setup(41, 3, False, 20, 20, 190, 3)
    gids = list(range(12))
    edge_off = eng.plan_graphs(gids)
    n, seed = adj.shape[1], 99
    want = []
    for g in gids:
        r, c = eng.graph_rows_cols(g)
        S = np.full((n, n), np.nan)
        S[r, c] = 1 / (1 + np.exp(-O.philox_m0(seed, g, len(r), n)))
        want.append((S[r, c] + S[c, r]) / 2)
    out = np.zeros(int(edge_off[-1]), np.float32)
    eng.explain_graphs_host(eng.make_hparams(num_epochs=1, init=_abi.GX_INIT_PHILOX, seed=seed), None, out)
    eng.close()
    assert np.abs(out - np.concatenate(want)).max() <= 1e-6


def test_wide_path_agrees_with_narrow_kernel_on_a_padded_model():
    """A d = 128 model and the same model with one zero feature column and a zero W1 row (d = 129, the wide path) compute the same
    explanation; coef_feat_size is scaled by 129 / 128 so that the mean's gradient per feature, c_feat / d, is the same too."""
    s = _node_setup(51, 3, True, 40, 40, 128, 4)
    w129 = dict(s.w)
    w129["W1"] = np.vstack([s.w["W1"], np.zeros((1, 40), np.float32)])
    feat129 = np.hstack([s.feat, np.zeros((len(s.feat), 1), np.float32)])
    wide = gnnx.Engine(0)
    wide.set_model(w129, num_layers=3, bn=True)
    wide.set_graph_csr(s.rowptr, s.col, feat129, s.label, s.pred_label)
    nodes = [0, 9, 21, 40]
    outs, fms = [], []
    for eng, d, cf in ((s.eng, 128, 1.0), (wide, 129, 129.0 / 128.0)):
        plan = eng.plan_nodes(nodes, 3)
        m0, _ = _m0(plan, 5)
        out = np.zeros(plan.total_edges, np.float32)
        fm = np.zeros((plan.count, d), np.float32)
        hp = eng.make_hparams(num_epochs=10)
        hp.coef_feat_size = cf
        eng.explain_nodes_host(hp, m0, out, fm)
        outs.append(out); fms.append(fm)
        eng.close()
    assert util.rel_l2(outs[1], outs[0]) <= 1e-5
    assert util.rel_l2(fms[1][:, :128], fms[0]) <= 1e-5 and np.all(fms[1][:, 128] < 0.5)   # the zero column only feels c_feat / d


def test_wide_refusals():
    s = _node_setup(61, 3, False, 20, 20, 300, 3)
    plan = s.eng.plan_nodes([0, 4], 3)
    m0, _ = _m0(plan, 3)
    out = np.zeros(plan.total_edges, np.float32)
    hp = s.eng.make_hparams(num_epochs=5)
    te = plan.total_edges
    calls = [lambda: s.eng.grad_nodes_host(out),
             lambda: s.eng.explain_nodes_ex(hp, m0, out, trace=np.zeros((2, 5, _abi.GX_TRACE_COLS), np.float32)),
             lambda: s.eng.explain_nodes_ex(hp, m0, out, state_out=dict(M=np.zeros(te, np.float32), m=np.zeros(te, np.float32),
                                                                         v=np.zeros(te, np.float32))),
             lambda: s.eng.explain_nodes_ex(s.eng.make_hparams(num_epochs=5, init=_abi.GX_INIT_STATE), m0, out,
                                            state_in=dict(m=np.zeros(te, np.float32), v=np.zeros(te, np.float32))),
             lambda: s.eng.explain_nodes_unconstrained(hp, None, out)]
    for call in calls:
        with pytest.raises(_abi.GnnxError) as e:
            call()
        assert e.value.status == GX_ERR_UNSUPPORTED
    rng = np.random.default_rng(0)
    att = [rng.normal(size=(300, 300)).astype(np.float32)] + [rng.normal(size=(20, 20)).astype(np.float32)] * 2
    too_wide = random_model(rng, 4097, 20, 20, 3, 3)
    for kw, w in ((dict(att=att), s.w), ({}, too_wide)):
        with pytest.raises(_abi.GnnxError) as e:
            s.eng.set_model(w, num_layers=3, **kw)
        assert e.value.status == GX_ERR_UNSUPPORTED
    s.eng.close()


@pytest.mark.parametrize("d,L,bn", [(300, 3, False), (4096, 2, True)])
def test_wide_model_forward_matches_port(d, L, bn):
    s = _node_setup(70 + L, L, bn, 20, 20, d, 4)
    got = s.eng.model_forward()
    s.eng.close()
    assert np.abs(got - s.pred).max() <= 2e-5 * max(1.0, np.abs(s.pred).max())


def _args(tmp_path, L, bn, graph, hid=20):
    return types.SimpleNamespace(num_gc_layers=L, num_epochs=20, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                 mask_bias=False, gpu=False, bias=True, bn=bn, method="base", dataset="graphs" if graph else "syn1",
                                 bmname=None, hidden_dim=hid, output_dim=hid, name_suffix="", explainer_suffix="", logdir=str(tmp_path))


def _state_dict(model, w, L):
    keys = ["conv_first"] + ["conv_block.%d" % i for i in range(L - 2)] + ["conv_last"]
    sd = {}
    for l, k in enumerate(keys, 1):
        sd[k + ".weight"] = w["W%d" % l]; sd[k + ".bias"] = w["b%d" % l]
    sd["pred_model.weight"] = w["Wp"]; sd["pred_model.bias"] = w["bp"]
    assert set(sd) == set(model.state_dict())
    return {k: torch.tensor(v) for k, v in sd.items()}


def _node_explainer(tmp_path, seed, L, bn, d, print_training):
    s = _node_setup(seed, L, bn, 20, 20, d, 4)
    s.eng.close()
    args = _args(tmp_path, L, bn, False)
    model = gnnx.models.GcnEncoderNode(d, 20, 20, 4, L, bn=bn, args=args)
    model.load_state_dict(_state_dict(model, s.w, L))
    ex = gnnx.Explainer(model=model, adj=torch.tensor(s.A[None], dtype=torch.float), feat=torch.tensor(s.feat[None]),
                        label=torch.tensor(s.label[None]), pred=None, train_idx=[], args=args, writer=None, print_training=print_training,
                        graph_mode=False, graph_idx=0)
    return s, args, ex


def test_explainer_dropin_node_mode(tmp_path, capsys):
    s, args, ex = _node_explainer(tmp_path, 81, 3, True, 300, True)
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
    assert "trace is not built for inputs wider than 128 features" in printed and "Saved adjacency matrix to" in printed
    assert any(f.startswith("masked_adj_syn1_") and f.endswith(".npy") for f in os.listdir(tmp_path))
    with pytest.raises(NotImplementedError):
        ex.explain(nodes[0], unconstrained=True)


def test_explainer_dropin_graph_mode(tmp_path, capsys):
    L, C, d = 4, 3, 190
    adj, feat, label, w, eng = _graph_setup(91, L, True, 20, 20, d, C)
    eng.close()
    args = _args(tmp_path, L, True, True)
    model = gnnx.models.GcnEncoderGraph(d, 20, 20, C, L, bn=True, args=args)
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
        port = O.explain_dense_torch(A, feat[g], label[g], None, 0, w, M0, hp, graph_mode=True, bn=True)
        p64 = O.explain_dense_torch(A, feat[g], label[g], None, 0, w, M0, hp, graph_mode=True, bn=True, dtype=torch.float64)
        ei, ej = np.nonzero(A)
        assert masked.shape == (n, n)
        assert O.rel_l2(masked[ei, ej], port[ei, ej]) <= max(1e-4, 3 * O.rel_l2(p64[ei, ej], port[ei, ej])), g
    torch.manual_seed(4)
    one = ex.explain(0, graph_idx=gids[0], graph_mode=True)
    assert np.array_equal(one, got[0])
    assert "trace is not built for inputs wider than 128 features" in capsys.readouterr().out
    assert any(f.endswith(".npy") for f in os.listdir(tmp_path))
    with pytest.raises(NotImplementedError):
        ex.explain(0, graph_idx=1, graph_mode=True, unconstrained=True)


def test_wide_sharded_explain_matches_explain_nodes(tmp_path):
    """gnnx.dist on a wide model (one rank, gloo, the torch all-gather): the packed masks of explain_nodes_sharded equal
    Explainer.explain_nodes under the same torch seed."""
    import socket
    import torch.distributed as dist
    from gnnx import dist as gdist
    s, args, ex = _node_explainer(tmp_path, 95, 3, False, 513, False)
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
    for t, D in enumerate(dense):
        ei, ej = np.nonzero(_sub(s, nodes[t])[0])
        assert np.array_equal(values[offsets[t]:offsets[t + 1]], D[ei, ej].astype(np.float32)), nodes[t]


# ---------------------------------------------------------------------------------------------------------- the unmodified reference
import pool_oracle as PO  # noqa: E402
from test_oracle_pool_ties import NEAR_TIES  # noqa: E402
from test_oracle_wide import GOLDEN, case_weights, golden_cases  # noqa: E402


@pytest.mark.parametrize("case,mode", golden_cases(), ids=lambda c: str(c))
def test_wide_matches_reference_golden(case, mode):
    """Every node and graph of tests/golden/wide_golden.npz (d = 300 node mode, d = 190 one-hot graph mode) within
    max(1e-4, 3 x the reference's own spread)."""
    g = np.load(GOLDEN)
    k = lambda s_: g["%s_%s" % (case, s_)]
    w = case_weights(g, case)
    L, bn = int(k("L")), bool(k("bn"))
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bn)
    hp = _hp(eng, int(k("epochs")), str(k("opt")))
    if mode == 0:
        rg = np.load(util.GOLDEN + "/rand_graph.npz")
        N = int(rg["N"])
        rowptr, col = O.csr_from_edges(N, rg["edges"])
        eng.set_graph_csr(rowptr, col, k("feat"), rg["label"].astype(np.int32), np.argmax(k("pred"), 1).astype(np.int32))
        nodes = [int(v) for v in k("nodes")]
        plan = eng.plan_nodes(nodes, L)
        m0 = np.empty(plan.total_edges, np.float32)
        for t, node in enumerate(nodes):
            assert np.array_equal(plan.neighbors_of(t), g["%s_n%d_nbrs" % (case, node)])
            r, c = plan.rows_cols_of(t)
            m0[plan.edge_off[t]:plan.edge_off[t + 1]] = O.draw_m0(plan.n(t), seed=int(g["%s_n%d_seed" % (case, node)]))[r, c]
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_host(hp, m0, out)
        for t, node in enumerate(nodes):   # edge slots in row-major order, as the reference's nonzero entries
            tol = max(1e-4, 3 * float(g["%s_n%d_spread" % (case, node)]))
            err = util.rel_l2(out[plan.edge_off[t]:plan.edge_off[t + 1]], g["%s_n%d_mask" % (case, node)])
            assert err <= tol, (case, node, err, tol)
    else:
        gg = np.load(util.GOLDEN + "/graphs_golden.npz")
        G, n = int(gg["num_graphs"]), int(gg["max_nodes"])
        eng.set_graph_batch(gg["adj"], k("feat"), gg["label"])
        gids = list(range(G))
        edge_off = eng.plan_graphs(gids)
        rc = [eng.graph_rows_cols(gi) for gi in gids]
        m0 = np.concatenate([O.draw_m0(n, seed=int(gg["g%d_seed" % gi]))[rc[gi]] for gi in gids]).astype(np.float32)
        out = np.zeros(int(edge_off[-1]), np.float32)
        eng.explain_graphs_host(hp, m0, out)
        for gi in gids:
            D = np.zeros((n, n))
            D[rc[gi]] = out[edge_off[gi]:edge_off[gi + 1]]
            ei, ej = np.nonzero(gg["adj"][gi])
            tol = max(1e-4, 3 * float(g["%s_g%d_spread" % (case, gi)]))
            err = util.rel_l2(D[ei, ej], g["%s_g%d_mask" % (case, gi)])
            if gi in NEAR_TIES.get(("wide", case), {}):   # a sub-ulp arg-max margin: the nearest admissible trajectory
                err = PO.nearest_admissible(D[ei, ej], g["%s_g%d_mask" % (case, gi)], np.asarray(gg["adj"][gi], np.float64),
                                            k("feat")[gi].astype(np.float32), int(gg["label"][gi]), w,
                                            O.draw_m0(n, seed=int(gg["g%d_seed" % gi])),
                                            O.default_hparams(num_epochs=int(k("epochs")), opt=str(k("opt"))), bn)
            assert err <= tol, (case, gi, err, tol)
    eng.close()


@pytest.mark.parametrize("case", [c for c, mode in golden_cases() if mode == 0])
def test_wide_model_forward_matches_reference_pred(case):
    """gx_model_forward at d = 300 against the reference model's own predictions on the rand graph."""
    g = np.load(GOLDEN)
    k = lambda s_: g["%s_%s" % (case, s_)]
    rg = np.load(util.GOLDEN + "/rand_graph.npz")
    rowptr, col = O.csr_from_edges(int(rg["N"]), rg["edges"])
    eng = gnnx.Engine(0)
    eng.set_model(case_weights(g, case), num_layers=int(k("L")), bn=bool(k("bn")))
    eng.set_graph_csr(rowptr, col, k("feat"), rg["label"].astype(np.int32), np.zeros(int(rg["N"]), np.int32))
    got = eng.model_forward()
    eng.close()
    ref = k("pred")
    assert np.abs(got - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max()), case
