"""GPU (-m gpu): GCNs with five to seven graph-convolution layers (num_gc_layers 5 .. 7, n_hops = num_gc_layers) on the model-variant
kernel (explain_var.cu), the unconstrained kernel (explain_dense.cu) and the model forward (forward.cu), through the C ABI, the drop-in
Explainer and gnnx.dist, node and graph mode: against the masks the unmodified reference returned (tests/golden/deep_golden.npz) and
against the torch port (oracle/gnnx_oracle.explain_dense_torch) in fp32 and fp64."""
import os
import types

import numpy as np
import pytest
import torch

import gnnx
import gnnx_oracle as O
import util
from gnnx import _abi
from test_oracle_deep import GOLDEN, case_weights, golden_cases

pytestmark = pytest.mark.gpu
GX_ERR_UNSUPPORTED = -3
GG = np.load(os.path.join(util.GOLDEN, "graphs_golden.npz"))


def random_model(rng, d, hid, emb, C, L, att=False):
    """Weights whose pre-activations stay O(1) at any width (each W scaled by 1.5 / sqrt(fan-in)), biases N(0, 0.3); att: Wa1 .. WaL."""
    dims = [d] + [hid] * (L - 1) + [emb]
    w = {}
    for l in range(1, L + 1):
        w["W%d" % l] = (rng.normal(size=(dims[l - 1], dims[l])) * 1.5 / np.sqrt(dims[l - 1])).astype(np.float32)
        w["b%d" % l] = (rng.normal(size=dims[l]) * 0.3).astype(np.float32)
        if att:
            w["Wa%d" % l] = (rng.normal(size=(dims[l - 1], dims[l - 1])) / np.sqrt(dims[l - 1])).astype(np.float32)
    w["Wp"] = (rng.normal(size=(C, hid * (L - 1) + emb)) * 0.5).astype(np.float32)
    w["bp"] = (rng.normal(size=C) * 0.3).astype(np.float32)
    return w


def _att_list(w, L):
    return [w["Wa%d" % l] for l in range(1, L + 1)] if "Wa1" in w else None


def _node_setup(seed, L, bn, att, hid, emb, d, C, N=48, m=2):
    import networkx as nx
    rng = np.random.default_rng(seed)
    rowptr, col = O.csr_from_edges(N, np.array(nx.barabasi_albert_graph(N, m, seed=seed).edges(), dtype=np.int64))
    A = O.dense_from_csr(rowptr, col)
    feat = rng.normal(size=(N, d)).astype(np.float32)
    label = rng.integers(0, C, N).astype(np.int32)
    w = random_model(rng, d, hid, emb, C, L, att)
    pred = O.model_pred(A, feat, w, bn=bn)
    pred_label = np.argmax(pred, 1).astype(np.int32)
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bn, att=_att_list(w, L))
    eng.set_graph_csr(rowptr, col, feat, label, pred_label)
    return types.SimpleNamespace(rowptr=rowptr, col=col, A=A, feat=feat, label=label, w=w, pred=pred, pred_label=pred_label, eng=eng,
                                 L=L, bn=bn, d=d)


def _graph_setup(seed, L, bn, att, hid, emb, d, C):
    rng = np.random.default_rng(seed)
    adj = GG["adj"]
    feat = (rng.normal(size=adj.shape[:2] + (d,)) * (adj.sum(2, keepdims=True) > 0)).astype(np.float32)
    label = np.asarray(GG["label"]) % C
    w = random_model(rng, d, hid, emb, C, L, att)
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bn, att=_att_list(w, L))
    eng.set_graph_batch(adj, feat, label)
    return adj, feat, label, w, eng


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


def _check(got, fm, w, port_args, port_kw):
    """Edge mask within max(1e-4, 3 x the port's fp32 / fp64 distance); feature mask within max(1e-4, 3 x the same distance on it)."""
    port, f32 = O.explain_dense_torch(*port_args, return_feat=True, **port_kw)
    p64, f64 = O.explain_dense_torch(*port_args, return_feat=True, dtype=torch.float64, **port_kw)
    tol = max(1e-4, 3 * O.rel_l2(p64, port))
    err = O.rel_l2(got, port)
    assert err <= tol, ("edge mask", err, tol)
    ftol = max(1e-4, 3 * float(np.abs(f64 - f32).max()))
    ferr = float(np.abs(fm - f32).max())
    assert ferr <= ftol, ("feature mask", ferr, ftol)


# seed, L, bn, att, hid, emb, d, C, opt, scheduler.  Conv weights: 20 and 64 wide stay in shared memory (L = 7, 64 / 64 at d = 128:
# 32 768 of the 36 864 staged words), 128 wide go through L2.  pred_model: C (PD + 1) <= 2048 in shared memory (L = 7, 64 / 64, C = 4:
# 1 796 words), beyond through L2 (the 128-wide cases).  d = 300: the wide path.
CASES = [
    (1, 5, False, False, 20, 20, 10, 4, "adam", "none"),
    (2, 6, True, False, 64, 64, 16, 3, "sgd", "step"),
    (3, 7, False, False, 128, 128, 12, 4, "rmsprop", "cos"),
    (4, 7, True, False, 64, 64, 128, 4, "adagrad", "none"),
    (5, 5, False, True, 20, 20, 8, 3, "adam", "none"),
    (6, 6, False, True, 32, 24, 12, 3, "sgd", "cos"),   # (--bn + attention at 6 layers is chaotic in graph mode: the ports part)
    (7, 6, False, False, 40, 40, 300, 3, "adam", "step"),
    (8, 5, True, False, 128, 96, 20, 5, "adam", "cos"),
]


def _case_id(c):
    return "s%d_L%d%s%s_h%d_e%d_d%d_%s_%s" % (c[0], c[1], "_bn" if c[2] else "", "_att" if c[3] else "", c[4], c[5], c[6], c[8], c[9])


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_deep_nodes_match_port(case):
    seed, L, bn, att, hid, emb, d, C, opt, sched = case
    s = _node_setup(seed, L, bn, att, hid, emb, d, C)
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
def test_deep_graphs_match_port(case):
    seed, L, bn, att, hid, emb, d, C, opt, sched = case
    adj, feat, label, w, eng = _graph_setup(seed + 20, L, bn, att, hid, emb, d, C)
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


ONE_UPDATE = [(31, 7, True, False, 20, 20, 16), (32, 5, False, True, 20, 20, 10), (33, 6, False, False, 128, 128, 24),
              (34, 5, True, False, 40, 40, 300)]


@pytest.mark.parametrize("case", ONE_UPDATE, ids=lambda c: "L%d%s%s_h%d_d%d" % (c[1], "_bn" if c[2] else "", "_att" if c[3] else "", c[4], c[6]))
def test_deep_one_update_matches_fp64_port(case):
    """num_epochs = 2: one update; edge and feature masks within 1e-5 of the fp64 port (or 3 x the fp32 port's distance from it, where
    the step is ill-conditioned: graph 10 under the 5-layer attention model), node and graph mode."""
    seed, L, bn, att, hid, emb, d = case
    s = _node_setup(seed, L, bn, att, hid, emb, d, 4)
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
    adj, feat, label, w, eng = _graph_setup(seed + 10, L, bn, att, hid, emb, d, 3)
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


def test_deep_large_subgraph_deterministic_and_order_free():
    """A hub whose 6-hop set has more than 1500 nodes, against the port; then Philox-initialised reruns are bit-identical, whatever
    the order of the batch."""
    s = _node_setup(41, 6, True, False, 20, 20, 12, 3, N=2000, m=2)
    hub = int(np.argmax(np.diff(s.rowptr)))
    plan = s.eng.plan_nodes([hub], 6)
    assert plan.n(0) > 1500
    m0, dense = _m0(plan, 9)
    out = np.zeros(plan.total_edges, np.float32)
    fm = np.zeros((1, 12), np.float32)
    s.eng.explain_nodes_host(s.eng.make_hparams(num_epochs=5), m0, out, fm)
    A, X, gt, pl, idx = _sub(s, hub)
    _check(plan.dense_of(0, out), fm[0], s.w, (A, X, gt, pl, idx, s.w, dense[0]), dict(hp=O.default_hparams(num_epochs=5), bn=True))
    nodes = [3, 17, hub, 120, 999]
    hp = s.eng.make_hparams(num_epochs=30, init=_abi.GX_INIT_PHILOX, seed=5)
    res = {}
    for order in (nodes, nodes[::-1], nodes):
        plan = s.eng.plan_nodes(order, 6)
        out = np.zeros(plan.total_edges, np.float32)
        fm = np.zeros((plan.count, 12), np.float32)
        s.eng.explain_nodes_host(hp, None, out, fm)
        for t, node in enumerate(order):
            got = np.concatenate([out[plan.edge_off[t]:plan.edge_off[t + 1]], fm[t]])
            if node in res:
                assert np.array_equal(res[node], got), node
            res[node] = got
    s.eng.close()


def test_deep_graphs_deterministic_and_order_free():
    adj, feat, label, w, eng = _graph_setup(42, 7, False, False, 64, 64, 14, 3)
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


@pytest.mark.parametrize("L", [5, 7])
def test_deep_unconstrained_matches_port(L):
    """unconstrained=True (explain_dense.cu: the pair product over d + hid (L - 1) + emb columns) against the line-by-line port."""
    E = 10
    fx = util.load_fixture("rand")
    rng = np.random.default_rng(60 + L)
    Wn = random_model(rng, fx.feat.shape[1], 20, 20, 3, L)
    Wg = random_model(rng, GG["feat"].shape[2], 24, 16, 2, L)
    eng = gnnx.Engine(0)
    eng.set_model(Wn, num_layers=L, bn=L == 7)
    eng.set_graph_csr(fx.rowptr, fx.col, fx.feat, fx.label, fx.pred_label)
    nodes = [33, 0]
    plan = eng.plan_nodes(nodes, L)
    m0 = [O.draw_m0(plan.n(t), seed=int(fx.gold["n%d_seed" % v])) for t, v in enumerate(nodes)]
    out = np.zeros(plan.total_edges, np.float32)
    eng.explain_nodes_unconstrained(eng.make_hparams(num_epochs=E), np.concatenate([M.reshape(-1) for M in m0]).astype(np.float32), out)
    eng.close()
    for t, v in enumerate(nodes):
        idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(fx.rowptr, fx.col, fx.feat, fx.label, v, L)
        A = O.dense_from_csr(srp, scol); ei, ej = np.nonzero(A)
        port = O.explain_dense_torch(A, X, int(lab[idx]), fx.pred_label[nbrs], idx, Wn, m0[t], hp=O.default_hparams(num_epochs=E),
                                     bn=L == 7, unconstrained=True)
        assert util.rel_l2(out[plan.edge_off[t]:plan.edge_off[t + 1]], port[ei, ej]) <= 1e-4, (L, v)
    eng = gnnx.Engine(0)
    eng.set_model(Wg, num_layers=L, bn=L == 5)
    eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
    gids = [2, 7]
    n = int(GG["max_nodes"])
    m0 = [O.draw_m0(n, seed=int(GG["g%d_seed" % g])) for g in gids]
    edge_off = eng.plan_graphs(gids)
    out = np.zeros(int(edge_off[-1]), np.float32)
    eng.explain_graphs_unconstrained(eng.make_hparams(num_epochs=E), np.concatenate([M.reshape(-1) for M in m0]).astype(np.float32), out)
    eng.close()
    for t, g in enumerate(gids):
        A = GG["adj"][g].astype(np.float64); ei, ej = np.nonzero(A)
        port = O.explain_dense_torch(A, GG["feat"][g], int(GG["label"][g]), None, 0, Wg, m0[t], hp=O.default_hparams(num_epochs=E),
                                     graph_mode=True, bn=L == 5, unconstrained=True)
        assert util.rel_l2(out[edge_off[t]:edge_off[t + 1]], port[ei, ej]) <= 1e-4, (L, g)


@pytest.mark.parametrize("L,bn,att,hid,emb,d", [(5, False, False, 64, 48, 16), (7, True, False, 128, 128, 10), (6, False, True, 40, 40, 12),
                                                (5, True, False, 20, 20, 300)])
def test_deep_model_forward_matches_port(L, bn, att, hid, emb, d):
    """gx_model_forward at every width gx_set_model accepts: rows of 32 / 64 / 128 floats."""
    s = _node_setup(70 + L, L, bn, att, hid, emb, d, 4, N=300, m=3)
    got = s.eng.model_forward()
    s.eng.close()
    assert np.abs(got - s.pred).max() <= 2e-5 * max(1.0, np.abs(s.pred).max())


def test_deep_refusals():
    s = _node_setup(61, 5, False, False, 20, 20, 10, 3)
    plan = s.eng.plan_nodes([0, 4], 5)
    m0, _ = _m0(plan, 3)
    out = np.zeros(plan.total_edges, np.float32)
    hp = s.eng.make_hparams(num_epochs=5)
    te = plan.total_edges
    calls = [lambda: s.eng.grad_nodes_host(out),
             lambda: s.eng.explain_nodes_ex(hp, m0, out, trace=np.zeros((2, 5, _abi.GX_TRACE_COLS), np.float32)),
             lambda: s.eng.explain_nodes_ex(hp, m0, out, state_out=dict(M=np.zeros(te, np.float32), m=np.zeros(te, np.float32),
                                                                         v=np.zeros(te, np.float32))),
             lambda: s.eng.explain_nodes_ex(s.eng.make_hparams(num_epochs=5, init=_abi.GX_INIT_STATE), m0, out,
                                            state_in=dict(m=np.zeros(te, np.float32), v=np.zeros(te, np.float32)))]
    for call in calls:
        with pytest.raises(_abi.GnnxError) as e:
            call()
        assert e.value.status == GX_ERR_UNSUPPORTED
    w8 = random_model(np.random.default_rng(0), 10, 20, 20, 3, 8)
    for kw in ({}, dict(att=[np.eye(10, dtype=np.float32)] + [np.eye(20, dtype=np.float32)] * 7)):
        with pytest.raises(_abi.GnnxError) as e:
            s.eng.set_model(w8, num_layers=8, **kw)
        assert e.value.status == GX_ERR_UNSUPPORTED and "[2,7]" in str(e.value)
    s.eng.close()


# ------------------------------------------------------------------------------------------------------------------ the drop-in Explainer
def _args(tmp_path, L, bn, graph, hid=20, emb=20):
    return types.SimpleNamespace(num_gc_layers=L, num_epochs=20, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                 mask_bias=False, gpu=False, bias=True, bn=bn, method="base", dataset="graphs" if graph else "syn1",
                                 bmname=None, hidden_dim=hid, output_dim=emb, name_suffix="", explainer_suffix="", logdir=str(tmp_path))


def _state_dict(model, w, L):
    keys = ["conv_first"] + ["conv_block.%d" % i for i in range(L - 2)] + ["conv_last"]
    sd = {}
    for l, k in enumerate(keys, 1):
        sd[k + ".weight"] = w["W%d" % l]; sd[k + ".bias"] = w["b%d" % l]
    sd["pred_model.weight"] = w["Wp"]; sd["pred_model.bias"] = w["bp"]
    assert set(sd) == set(model.state_dict())
    return {k: torch.tensor(v) for k, v in sd.items()}


def _node_explainer(tmp_path, seed, L, bn, hid, emb, print_training):
    s = _node_setup(seed, L, bn, False, hid, emb, 10, 4)
    s.eng.close()
    args = _args(tmp_path, L, bn, False, hid, emb)
    model = gnnx.models.GcnEncoderNode(10, hid, emb, 4, L, bn=bn, args=args)
    model.load_state_dict(_state_dict(model, s.w, L))
    ex = gnnx.Explainer(model=model, adj=torch.tensor(s.A[None], dtype=torch.float), feat=torch.tensor(s.feat[None]),
                        label=torch.tensor(s.label[None]), pred=None, train_idx=[], args=args, writer=None, print_training=print_training,
                        graph_mode=False, graph_idx=0)
    return s, args, ex


@pytest.mark.parametrize("hid,emb", [(20, 20), (64, 48), (128, 128)])
def test_explainer_dropin_node_mode(tmp_path, capsys, hid, emb):
    """Explainer(pred=None) at L = 5: the predicted labels come from gx_model_forward (widths 64 and 128: rows of 64 / 128 floats)."""
    s, args, ex = _node_explainer(tmp_path, 81, 5, True, hid, emb, True)
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
    nb = ex.neighborhoods
    assert np.array_equal(nb[0], O.neighborhoods_dense(s.A[None], 5)[0])


def test_explainer_dropin_graph_mode(tmp_path, capsys):
    L, C, d = 5, 3, 14
    adj, feat, label, w, eng = _graph_setup(91, L, False, False, 20, 20, d, C)
    eng.close()
    args = _args(tmp_path, L, False, True)
    model = gnnx.models.GcnEncoderGraph(d, 20, 20, C, L, bn=False, args=args)
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


def test_deep_sharded_explain_matches_explain_nodes(tmp_path):
    """gnnx.dist on a 7-layer model (one rank, gloo, the torch all-gather): the packed masks of explain_nodes_sharded equal
    Explainer.explain_nodes under the same torch seed."""
    import socket
    import torch.distributed as dist
    from gnnx import dist as gdist
    s, args, ex = _node_explainer(tmp_path, 95, 7, False, 20, 20, False)
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
def test_deep_matches_reference_golden(case, mode):
    """Every node and graph of tests/golden/deep_golden.npz within max(1e-4, 3 x the reference's own spread)."""
    g = np.load(GOLDEN)
    k = lambda s_: g["%s_%s" % (case, s_)]
    w = case_weights(g, case)
    L, bn = int(k("L")), bool(k("bn"))
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bn, att=_att_list(w, L))
    hp = _hp(eng, int(k("epochs")), str(k("opt")))
    if mode == 0:
        rg = np.load(util.GOLDEN + "/rand_graph.npz")
        N = int(rg["N"])
        rowptr, col = O.csr_from_edges(N, rg["edges"])
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
        for t, node in enumerate(nodes):   # edge slots in row-major order, as the reference's nonzero entries
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
            assert err <= tol, (case, gi, err, tol)
    eng.close()


@pytest.mark.parametrize("case", [c for c, mode in golden_cases() if mode == 0])
def test_deep_model_forward_matches_reference_pred(case):
    """gx_model_forward against the reference model's own predictions on the rand graph."""
    g = np.load(GOLDEN)
    k = lambda s_: g["%s_%s" % (case, s_)]
    rg = np.load(util.GOLDEN + "/rand_graph.npz")
    rowptr, col = O.csr_from_edges(int(rg["N"]), rg["edges"])
    w = case_weights(g, case)
    L = int(k("L"))
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bool(k("bn")), att=_att_list(w, L))
    eng.set_graph_csr(rowptr, col, rg["feat"].astype(np.float32), rg["label"].astype(np.int32), np.zeros(int(rg["N"]), np.int32))
    got = eng.model_forward()
    eng.close()
    ref = k("pred")
    assert np.abs(got - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max()), case
