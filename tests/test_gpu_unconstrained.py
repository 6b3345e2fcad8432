"""GPU (-m gpu): Explainer.explain(..., unconstrained=True) on the dense kernel (explain_dense.cu) through the C ABI and the drop-in
Explainer, against the UNMODIFIED reference's results (tests/golden/unconstrained_golden.npz), the line-by-line port and the fp64
closed form (oracle/gnnx_oracle.py)."""
import importlib.util
import os
import re
import types

import numpy as np
import pytest
import torch

import gnnx
from gnnx import _abi
import dense_oracle as D
import gnnx_oracle as O
import util

pytestmark = pytest.mark.gpu
U = np.load(os.path.join(util.GOLDEN, "unconstrained_golden.npz"))
GG = np.load(os.path.join(util.GOLDEN, "graphs_golden.npz"))
NG, NMAX = int(GG["num_graphs"]), int(GG["max_nodes"])


# ------------------------------------------------------------------------------------ helpers
def dense_m0(plan, seeds):
    return [O.draw_m0(plan.n(t), seed=seeds[t]) for t in range(plan.count)]


def run(eng, hp, m0_list, count, n_t, total_edges, graphs=False, dense=False, trace=False):
    """gx_explain_{nodes,graphs}_unconstrained on the current plan -> (edge_mask, mask_dense list or None, trace, trace_pred)."""
    m0 = None if m0_list is None else np.concatenate([M.reshape(-1) for M in m0_list]).astype(np.float32)
    out = np.zeros(max(int(total_edges), 1), np.float32)
    nn = np.asarray(n_t, np.int64) ** 2
    md = np.zeros(int(nn.sum()), np.float32) if dense else None
    tr = np.zeros((count, hp.num_epochs, _abi.GX_TRACE_COLS), np.float32) if trace else None
    tp = np.zeros((count, hp.num_epochs, eng.num_classes), np.float32) if trace else None
    fn = eng.explain_graphs_unconstrained if graphs else eng.explain_nodes_unconstrained
    fn(hp, m0, out, md, tr, tp)
    mds = None
    if dense:
        offs = np.concatenate([[0], np.cumsum(nn)])
        mds = [md[offs[t]:offs[t + 1]].reshape(n_t[t], n_t[t]) for t in range(count)]
    return out, mds, tr, tp


def run_nodes(eng, plan, hp, m0_list, **kw):
    return run(eng, hp, m0_list, plan.count, [plan.n(t) for t in range(plan.count)], plan.total_edges, **kw)


def run_graphs(eng, gids, hp, m0_list, **kw):
    edge_off = eng.plan_graphs(gids)
    return edge_off, run(eng, hp, m0_list, len(gids), [NMAX] * len(gids), edge_off[-1], graphs=True, **kw)


def graph_engine(W, L=3, bn=False, label=None):
    eng = gnnx.Engine(0)
    eng.set_model(W, num_layers=L, bn=bn)
    eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"] if label is None else label)
    return eng


def graph_weights():
    return {k: GG[k] for k in util.WKEYS}


def var_weights(tag, where):
    pre = "var_%s_%s_" % (tag, where)
    return {k[len(pre):]: U[k] for k in U.files if k.startswith(pre) and k[len(pre):][0] in "Wb"}


def variant_pred_label(fx, W, bn):
    """argmax of a variant model's logits on the whole rand graph (the pred the fixture's Explainer was given)."""
    A = O.dense_from_csr(fx.rowptr, fx.col)
    with torch.no_grad():
        logits = O._gcn_forward_torch(torch.tensor(fx.feat[None], dtype=torch.float), torch.tensor(A[None], dtype=torch.float),
                                      O.weights_to_torch(W, requires_grad=False), False, bn)
    return np.argmax(logits[0].numpy(), axis=1).astype(np.int32)


def node_inputs(fx, plan, t):
    """(A, X, gt, y, idx) of planned node t (3 hops), for the CPU oracle."""
    idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(fx.rowptr, fx.col, fx.feat, fx.label, int(plan.nodes[t]), 3)
    return O.dense_from_csr(srp, scol), X, int(lab[idx]), fx.pred_label[nbrs], idx


def seg(out, off, t):
    return out[off[t]:off[t + 1]]


def tol(spread):
    return max(1e-4, 3.0 * float(spread))


# ------------------------------------------------------------------------------------ against the reference
@pytest.mark.parametrize("which", ["syn1", "syn4", "rand"])
def test_nodes_match_reference(which):
    fx = util.load_fixture(which)
    eng = util.make_engine(fx)
    nodes = [int(v) for v in U[which + "_nodes"]]
    plan = eng.plan_nodes(nodes, 3)
    seeds = [int(fx.gold["n%d_seed" % v]) for v in nodes]
    bad = {}
    for E in (int(e) for e in U["epochs"]):
        out, _, _, _ = run_nodes(eng, plan, eng.make_hparams(num_epochs=E), dense_m0(plan, seeds))
        for t, v in enumerate(nodes):
            key = "%s_n%d_e%d" % (which, v, E)
            err = util.rel_l2(seg(out, plan.edge_off, t), U[key + "_mask"])
            if not err <= tol(U[key + "_spread"]):
                bad[key] = (err, tol(U[key + "_spread"]))
    assert not bad, bad
    eng.close()


def test_graphs_match_reference():
    eng = graph_engine(graph_weights())
    gids = list(range(NG))
    bad = {}
    for E in (int(e) for e in U["epochs"]):
        m0 = [O.draw_m0(NMAX, seed=int(GG["g%d_seed" % g])) for g in gids]
        edge_off, (out, _, _, _) = run_graphs(eng, gids, eng.make_hparams(num_epochs=E), m0)
        for t, g in enumerate(gids):
            key = "graphs_g%d_e%d" % (g, E)
            err = util.rel_l2(seg(out, edge_off, t), U[key + "_mask"])
            if not err <= tol(U[key + "_spread"]):
                bad[key] = (err, tol(U[key + "_spread"]))
    assert not bad, bad
    eng.close()


@pytest.mark.parametrize("tag", ["bn", "L4", "sgd"])
def test_variants_match_reference(tag):
    L, bn, E = int(U["var_%s_L" % tag]), bool(U["var_%s_bn" % tag]), int(U["var_epochs"])
    over = dict(opt=_abi.GX_OPT["sgd"]) if tag == "sgd" else {}
    fx = util.load_fixture("rand")
    Wn = fx.weights if tag == "sgd" else var_weights(tag, "rand")
    pl = fx.pred_label if tag == "sgd" else variant_pred_label(fx, Wn, bn)
    eng = gnnx.Engine(0)
    eng.set_model(Wn, num_layers=L, bn=bn)
    eng.set_graph_csr(fx.rowptr, fx.col, fx.feat, fx.label, pl)
    nodes = [int(v) for v in U["rand_nodes"]]
    plan = eng.plan_nodes(nodes, L)
    out, _, _, _ = run_nodes(eng, plan, eng.make_hparams(num_epochs=E, **over), dense_m0(plan, [int(fx.gold["n%d_seed" % v]) for v in nodes]))
    bad = {}
    for t, v in enumerate(nodes):
        key = "var_%s_rand_n%d" % (tag, v)
        assert np.array_equal(plan.neighbors_of(t), U[key + "_nbrs"])
        err = util.rel_l2(seg(out, plan.edge_off, t), U[key + "_mask"])
        if not err <= tol(U[key + "_spread"]):
            bad[key] = (err, tol(U[key + "_spread"]))
    eng.close()
    eng = graph_engine(graph_weights() if tag == "sgd" else var_weights(tag, "graphs"), L, bn)
    gids = list(range(NG))
    edge_off, (out, _, _, _) = run_graphs(eng, gids, eng.make_hparams(num_epochs=E, **over),
                                          [O.draw_m0(NMAX, seed=int(GG["g%d_seed" % g])) for g in gids])
    for t, g in enumerate(gids):
        key = "var_%s_graphs_g%d" % (tag, g)
        err = util.rel_l2(seg(out, edge_off, t), U[key + "_mask"])
        if not err <= tol(U[key + "_spread"]):
            bad[key] = (err, tol(U[key + "_spread"]))
    assert not bad, bad
    eng.close()


# ------------------------------------------------------------------------------------ one update against the fp64 closed form
def test_one_update_matches_closed_form():
    """num_epochs=2: the mask after ONE update, every fixture node and graph (the chaotic ones included), within 1e-5 of the fp64 spec."""
    bad = {}
    hp_cf = O.default_hparams(num_epochs=2)
    for which in ("syn1", "syn4", "rand"):
        fx = util.load_fixture(which)
        eng = util.make_engine(fx)
        nodes = [int(v) for v in U[which + "_nodes"]]
        plan = eng.plan_nodes(nodes, 3)
        m0 = dense_m0(plan, [int(fx.gold["n%d_seed" % v]) for v in nodes])
        out, _, _, _ = run_nodes(eng, plan, eng.make_hparams(num_epochs=2), m0)
        for t, v in enumerate(nodes):
            A, X, gt, y, idx = node_inputs(fx, plan, t)
            ei, ej = np.nonzero(A)
            cf = D.explain_closed_form(A, X, gt, y, idx, fx.weights, m0[t], hp=hp_cf)
            err = util.rel_l2(seg(out, plan.edge_off, t), cf[ei, ej])
            if not err <= 1e-5:
                bad["%s_n%d" % (which, v)] = err
        eng.close()
    eng = graph_engine(graph_weights())
    gids = list(range(NG))
    m0 = [O.draw_m0(NMAX, seed=int(GG["g%d_seed" % g])) for g in gids]
    edge_off, (out, _, _, _) = run_graphs(eng, gids, eng.make_hparams(num_epochs=2), m0)
    for t, g in enumerate(gids):
        A = GG["adj"][g].astype(np.float64)
        ei, ej = np.nonzero(A)
        cf = D.explain_closed_form(A, GG["feat"][g], int(GG["label"][g]), None, 0, graph_weights(), m0[t], hp=hp_cf, graph_mode=True)
        err = util.rel_l2(seg(out, edge_off, t), cf[ei, ej])
        if not err <= 1e-5:
            bad["g%d" % g] = err
    assert not bad, bad
    eng.close()


# ------------------------------------------------------------------------------------ models and optimisers against the port
def _random_model(rng, d, hid, emb, C, L):
    sc = lambda *s: (rng.normal(size=s) * 0.4).astype(np.float32)
    W = {}
    for l in range(1, L + 1):
        win, wout = (d if l == 1 else hid), (emb if l == L else hid)
        W["W%d" % l], W["b%d" % l] = sc(win, wout), sc(wout)
    W["Wp"], W["bp"] = sc(C, hid * (L - 1) + emb), sc(C)
    return W


CASES = {"wide_bn": dict(hid=64, emb=48, L=3, bn=True), "wide_L2": dict(hid=128, emb=96, L=2, bn=False),
         "rmsprop": dict(opt="rmsprop"), "adagrad": dict(opt="adagrad"),
         "adamstep": dict(opt="adam", opt_scheduler="step", opt_decay_step=3, opt_decay_rate=0.5)}


@pytest.mark.parametrize("case", list(CASES))
def test_models_and_optimisers_match_port(case):
    c = CASES[case]
    E = 10
    fx = util.load_fixture("rand")
    L, bn = c.get("L", 3), c.get("bn", False)
    opt = {k: v for k, v in c.items() if k.startswith("opt")}
    hp_cf = O.default_hparams(num_epochs=E, **opt)
    gx_opt = dict(opt=_abi.GX_OPT[opt["opt"]]) if opt else {}
    if "opt_scheduler" in opt:
        gx_opt.update(opt_scheduler=_abi.GX_SCHED[opt["opt_scheduler"]], opt_decay_step=opt["opt_decay_step"], opt_decay_rate=opt["opt_decay_rate"])
    rng = np.random.default_rng(5)
    Wn = _random_model(rng, fx.feat.shape[1], c["hid"], c["emb"], 3, L) if "hid" in c else fx.weights
    Wg = _random_model(rng, 14, c["hid"], c["emb"], 2, L) if "hid" in c else graph_weights()
    eng = gnnx.Engine(0)
    eng.set_model(Wn, num_layers=L, bn=bn)
    eng.set_graph_csr(fx.rowptr, fx.col, fx.feat, fx.label, fx.pred_label)
    nodes = [33, 149, 0]
    plan = eng.plan_nodes(nodes, L)
    m0 = dense_m0(plan, [int(fx.gold["n%d_seed" % v]) for v in nodes])
    out, _, _, _ = run_nodes(eng, plan, eng.make_hparams(num_epochs=E, **gx_opt), m0)
    for t, v in enumerate(nodes):
        idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(fx.rowptr, fx.col, fx.feat, fx.label, v, L)
        A = O.dense_from_csr(srp, scol); ei, ej = np.nonzero(A)
        port = O.explain_dense_torch(A, X, int(lab[idx]), fx.pred_label[nbrs], idx, Wn, m0[t], hp=hp_cf, bn=bn, unconstrained=True)
        assert util.rel_l2(seg(out, plan.edge_off, t), port[ei, ej]) <= 1e-4, (case, v)
    eng.close()
    eng = graph_engine(Wg, L, bn)
    gids = [2, 7, 9]
    m0 = [O.draw_m0(NMAX, seed=int(GG["g%d_seed" % g])) for g in gids]
    edge_off, (out, _, _, _) = run_graphs(eng, gids, eng.make_hparams(num_epochs=E, **gx_opt), m0)
    for t, g in enumerate(gids):
        A = GG["adj"][g].astype(np.float64); ei, ej = np.nonzero(A)
        port = O.explain_dense_torch(A, GG["feat"][g], int(GG["label"][g]), None, 0, Wg, m0[t], hp=hp_cf, graph_mode=True, bn=bn,
                                     unconstrained=True)
        assert util.rel_l2(seg(out, edge_off, t), port[ei, ej]) <= 1e-4, (case, g)
    eng.close()


def _bench():
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    return bench


def test_large_subgraph_and_refusals():
    """A BA subgraph with 1024 < n <= 4096 against the port; n = 4097, GX_INIT_STATE and mask_act ReLU are refused."""
    rowptr, col = _bench().make_ba_csr(20000, 2, 0)
    N = len(rowptr) - 1
    rng = np.random.default_rng(3)
    d, C = 16, 3
    feat = rng.normal(size=(N, d)).astype(np.float32)
    label = rng.integers(0, C, N).astype(np.int32)
    pl = rng.integers(0, C, N).astype(np.int32)
    W = _random_model(rng, d, 20, 20, C, 3)
    node = next(v for v in range(N - 1, 0, -1) if 1024 < len(O.khop_walk_set(rowptr, col, v, 3)) <= 4096)
    eng = gnnx.Engine(0)
    eng.set_model(W)
    eng.set_graph_csr(rowptr, col, feat, label, pl)
    plan = eng.plan_nodes([node], 3)
    n = plan.n(0)
    assert 1024 < n <= 4096
    m0 = [O.draw_m0(n, seed=9)]
    out, _, _, _ = run_nodes(eng, plan, eng.make_hparams(num_epochs=3), m0)
    idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(rowptr, col, feat, label, node, 3)
    A = O.dense_from_csr(srp, scol); ei, ej = np.nonzero(A)
    port = O.explain_dense_torch(A, X, int(lab[idx]), pl[nbrs], idx, W, m0[0], hp=O.default_hparams(num_epochs=3), unconstrained=True)
    assert util.rel_l2(out[:plan.total_edges], port[ei, ej]) <= 1e-4
    for over in (dict(init=_abi.GX_INIT_STATE), dict(mask_act=1)):
        with pytest.raises(_abi.GnnxError) as e:
            run_nodes(eng, plan, eng.make_hparams(num_epochs=3, **over), m0)
        assert e.value.status == -3, over
    eng.close()
    # a star: the centre's 3-hop set is the centre and its 4096 leaves
    star = np.array([[0, k] for k in range(1, 4097)], np.int64)
    srp_, scol_ = O.csr_from_edges(4097, star)
    eng = gnnx.Engine(0)
    eng.set_model(W)
    eng.set_graph_csr(srp_, scol_, rng.normal(size=(4097, d)).astype(np.float32), np.zeros(4097, np.int32), np.zeros(4097, np.int32))
    plan = eng.plan_nodes([0], 3)
    assert plan.n(0) == 4097
    with pytest.raises(_abi.GnnxError) as e:
        run_nodes(eng, plan, eng.make_hparams(num_epochs=2, init=_abi.GX_INIT_PHILOX), None)
    assert e.value.status == -3
    eng.close()


# ------------------------------------------------------------------------------------ trace, dense output, determinism, init
@pytest.mark.parametrize("which", ["syn1", "rand"])
def test_trace_matches_printed_rows(which):
    fx = util.load_fixture(which)
    eng = util.make_engine(fx)
    E = int(U["trace_epochs"])
    nodes = [int(v) for v in U["trace_%s_nodes" % which]]
    plan = eng.plan_nodes(nodes, 3)
    m0 = dense_m0(plan, [int(fx.gold["n%d_seed" % v]) for v in nodes])
    hp = eng.make_hparams(num_epochs=E)
    out, _, tr, tp = run_nodes(eng, plan, hp, m0, trace=True)
    plain, _, _, _ = run_nodes(eng, plan, hp, m0)
    assert np.array_equal(out, plain)                  # a trace leaves the masks bit-identical
    for t, v in enumerate(nodes):
        ref = U["trace_%s_n%d" % (which, v)]
        loss, dens = tr[t, :, _abi.TR_LOSS_EDGES].astype(np.float64), tr[t, :, _abi.TR_DENSITY].astype(np.float64)
        assert np.all(np.abs(loss - ref[:, 0]) <= 1e-5 * np.abs(ref[:, 0])), (v, loss, ref[:, 0])
        assert np.all(np.abs(dens - ref[:, 1]) <= 1e-5 * np.abs(ref[:, 1])), (v, dens, ref[:, 1])
        assert np.abs(tp[t] - ref[:, 2:]).max() <= 1e-5, v
        terms = sum(tr[t, :, k] for k in (_abi.TR_PRED, _abi.TR_SIZE, _abi.TR_LAP, _abi.TR_ENT, _abi.TR_FEAT))
        assert np.allclose(terms, tr[t, :, _abi.TR_LOSS_EDGES], rtol=1e-6)
    eng.close()


def test_dense_output_determinism_and_batch_independence():
    fx = util.load_fixture("rand")
    eng = util.make_engine(fx)
    nodes = [int(v) for v in U["rand_nodes"]]
    seeds = {v: int(fx.gold["n%d_seed" % v]) for v in nodes}
    hp = eng.make_hparams(num_epochs=30)
    plan = eng.plan_nodes(nodes, 3)
    out, md, _, _ = run_nodes(eng, plan, hp, dense_m0(plan, [seeds[v] for v in nodes]), dense=True)
    again, _, _, _ = run_nodes(eng, plan, hp, dense_m0(plan, [seeds[v] for v in nodes]))
    assert np.array_equal(out, again)
    for t in range(plan.count):
        D = md[t]
        assert np.array_equal(D, D.T) and np.all(np.diag(D) == 0)
        off = ~np.eye(len(D), dtype=bool)
        assert D[off].min() > 0 and D[off].max() < 1
        r, c = plan.rows_cols_of(t)
        assert np.array_equal(D[r, c], seg(out, plan.edge_off, t))   # bit for bit
    sub = [nodes[5], nodes[1], nodes[3]]
    p2 = eng.plan_nodes(sub, 3)
    o2, _, _, _ = run_nodes(eng, p2, hp, dense_m0(p2, [seeds[v] for v in sub]))
    for t, v in enumerate(sub):
        assert np.array_equal(seg(o2, p2.edge_off, t), seg(out, plan.edge_off, nodes.index(v)))
    eng.close()
    eng = graph_engine(graph_weights())
    m0 = {g: O.draw_m0(NMAX, seed=int(GG["g%d_seed" % g])) for g in range(NG)}
    e1, (o1, md1, _, _) = run_graphs(eng, list(range(NG)), hp, [m0[g] for g in range(NG)], dense=True)
    e2, (o2, _, _, _) = run_graphs(eng, [9, 2, 5], hp, [m0[g] for g in (9, 2, 5)])
    for t, g in enumerate((9, 2, 5)):
        assert np.array_equal(seg(o2, e2, t), seg(o1, e1, g))
    for g in range(NG):
        r, c = eng.graph_rows_cols(g)
        assert np.array_equal(md1[g][r, c], seg(o1, e1, g)) and np.array_equal(md1[g], md1[g].T)
    eng.close()


def test_philox_init():
    """GX_INIT_PHILOX, num_epochs=1: the returned dense mask is sym(sigmoid(M0)) (.) (1 - I) of philox_m0(seed, key, n*n, n)."""
    fx = util.load_fixture("rand")
    eng = util.make_engine(fx)
    hp = eng.make_hparams(num_epochs=1, init=_abi.GX_INIT_PHILOX, seed=1234)
    plan = eng.plan_nodes([0, 33], 3)
    _, md, _, _ = run_nodes(eng, plan, hp, None, dense=True)

    def expect(key, n, nn):
        S = 1 / (1 + np.exp(-O.philox_m0(1234, key, n * n, nn).reshape(n, n)))
        return (S + S.T) / 2 * (1 - np.eye(n))
    for t, v in enumerate([0, 33]):
        assert np.abs(md[t] - expect(v, plan.n(t), plan.n(t))).max() <= 1e-6
    eng.close()
    eng = graph_engine(graph_weights())
    _, (_, md, _, _) = run_graphs(eng, [3, 8], hp, None, dense=True)
    for t, g in enumerate([3, 8]):
        assert np.abs(md[t] - expect(g, NMAX, NMAX)).max() <= 1e-6
    eng.close()


# ------------------------------------------------------------------------------------ drop-in Explainer
def _args(tmp_path, **over):
    args = types.SimpleNamespace(num_gc_layers=3, num_epochs=30, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                 mask_bias=False, gpu=False, bias=True, method="base", dataset="rand", bmname=None, hidden_dim=20,
                                 output_dim=20, name_suffix="", explainer_suffix="", logdir=str(tmp_path))
    for k, v in over.items():
        setattr(args, k, v)
    return args


def _load(model, W):
    names = {"W1": "conv_first.weight", "b1": "conv_first.bias", "W2": "conv_block.0.weight", "b2": "conv_block.0.bias",
             "W3": "conv_last.weight", "b3": "conv_last.bias", "Wp": "pred_model.weight", "bp": "pred_model.bias"}
    model.load_state_dict({names[k]: torch.tensor(v) for k, v in W.items()})
    return model


def test_explainer_dropin_node_mode(tmp_path, capsys):
    fx = util.load_fixture("rand")
    args = _args(tmp_path)
    model = _load(gnnx.models.GcnEncoderNode(fx.feat.shape[1], 20, 20, 3, 3, bn=False, args=args), fx.weights)
    A = O.dense_from_csr(fx.rowptr, fx.col)
    ex = gnnx.Explainer(model=model, adj=A[None], feat=fx.feat[None].astype(np.float64), label=fx.label[None], pred=fx.pred[None],
                        train_idx=list(range(fx.N)), args=args, writer=None, print_training=False, graph_idx=-1)
    for v in (0, 33, 149):
        seed = int(fx.gold["n%d_seed" % v])
        torch.manual_seed(seed)
        masked = ex.explain(v, graph_idx=0, unconstrained=True)
        after = torch.get_rng_state()
        n = len(fx.gold["n%d_nbrs" % v])
        O.draw_m0(n, seed=seed)                                   # the reference's call consumes exactly these n^2 normals
        assert torch.equal(after, torch.get_rng_state())
        _, sub_adj, _, _, _ = ex.extract_neighborhood(v)
        ei, ej = np.nonzero(sub_adj)
        key = "rand_n%d_e30" % v
        assert masked.shape == (n, n) and masked.dtype == np.float64
        assert util.rel_l2(masked[ei, ej], U[key + "_mask"]) <= tol(U[key + "_spread"])
        off = masked.copy(); off[ei, ej] = 0
        assert np.all(off == 0)
        f = os.path.join(str(tmp_path), "masked_adj_rand_base_h20_o20_explainnode_idx_%dgraph_idx_-1.npy" % v)
        assert np.array_equal(np.load(f), masked)
    torch.manual_seed(4)
    grad_u = ex.explain(33, model="grad", unconstrained=True)
    torch.manual_seed(4)
    assert np.array_equal(grad_u, ex.explain(33, model="grad"))
    # print_training: the reference's per-epoch lines
    E = int(U["trace_epochs"])
    ex.print_training = True
    ex.args.num_epochs = E
    capsys.readouterr()
    for v in [int(x) for x in U["trace_rand_nodes"]]:
        torch.manual_seed(int(fx.gold["n%d_seed" % v]))
        ex.explain(v, unconstrained=True)
        text = capsys.readouterr().out
        rows = re.findall(r"epoch:\s+(\d+)\s+; loss:\s+(\S+)\s+; mask density:\s+(\S+)\s+; pred:", text)
        assert len(rows) == E and "finished training in" in text and "Saved adjacency matrix to" in text
        ref = U["trace_rand_n%d" % v]
        got = np.array([[float(r[1]), float(r[2])] for r in rows])
        assert np.all(np.abs(got - ref[:, :2]) <= 1e-5 * np.abs(ref[:, :2])), (v, got, ref[:, :2])


def test_explainer_dropin_graph_mode(tmp_path):
    args = _args(tmp_path, num_epochs=10, dataset="graphs")
    model = _load(gnnx.models.GcnEncoderGraph(14, 20, 20, 2, 3, bn=False, args=args), graph_weights())
    ex = gnnx.Explainer(model=model, adj=torch.tensor(GG["adj"], dtype=torch.float), feat=torch.tensor(GG["feat"]),
                        label=torch.tensor(GG["label"]), pred=GG["pred"], train_idx=[], args=args, writer=None,
                        print_training=False, graph_mode=True, graph_idx=0)
    for g in (0, 4, 7):
        seed = int(GG["g%d_seed" % g])
        torch.manual_seed(seed)
        masked = ex.explain(node_idx=0, graph_idx=g, graph_mode=True, unconstrained=True)
        after = torch.get_rng_state()
        O.draw_m0(NMAX, seed=seed)
        assert torch.equal(after, torch.get_rng_state())
        assert masked.shape == (NMAX, NMAX) and masked.dtype == np.float64
        ei, ej = np.nonzero(GG["adj"][g])
        key = "graphs_g%d_e10" % g
        assert util.rel_l2(masked[ei, ej], U[key + "_mask"]) <= tol(U[key + "_spread"])
        f = os.path.join(str(tmp_path), "masked_adj_graphs_base_h20_o20_explainnode_idx_0graph_idx_0.npy")
        assert np.array_equal(np.load(f), masked)
