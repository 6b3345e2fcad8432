"""GPU (-m gpu): every explainer kernel under non-default hyper-parameters -- learning rate, epochs, Adam betas and eps, loss
coefficients, the step and cosine schedulers, resume under them, the per-handle table cache, the trace limits and the refusals.

  * the UNMODIFIED reference's masks under --lr / --epochs / schedulers (tests/golden/hparams_golden.npz) on the shared-memory kernel,
    its cluster class, the gang and first-generation streaming kernels and explain_graph.cu, within max(1e-4, 3 x spread);
  * the sets H1 / H2 / H0 of tests/test_oracle_hparams.py (betas and eps; loss coefficients; no regularisers) against the torch ports on
    every kernel family, each case also showing that the set moves the port by more than 10 x the tolerance;
  * lr = 0 returns the initial mask; one update (num_epochs = 2) lands within 1e-5 of the fp64 specification."""
import networkx as nx
import numpy as np
import pytest
import torch

import dense_oracle as D
import gnnx
import gnnx_oracle as O
import util
from gnnx import _abi
from test_oracle_att import random_att_model
from test_oracle_hparams import HSETS, case_hparams, golden, gx_over
from test_gpu_wide import _graph_setup, _node_setup

pytestmark = pytest.mark.gpu
GX_ERR_INVALID, GX_ERR_UNSUPPORTED = -1, -3
H = golden()
GG = np.load(util.GOLDEN + "/graphs_golden.npz")
NG, NMAX = int(GG["num_graphs"]), int(GG["max_nodes"])
GW = {k: GG[k] for k in util.WKEYS}
TAGS = [str(t) for t in H["case_tags"]]
NODE_PATHS = ["smem", "cluster2", "cluster4", "gang", "stream1"]
SMEM_CLASSES = 5                              # launch classes 0..4 of the shared-memory kernel; 5 = slabs, 6 = clusters


# ------------------------------------------------------------------------------------ helpers
def to_gx(eng, hp, **extra):
    """engine hyper-parameters of a gnnx_oracle.default_hparams namespace."""
    return eng.make_hparams(num_epochs=hp.num_epochs, lr=hp.lr, beta1=hp.beta1, beta2=hp.beta2, eps=hp.eps, coef_size=hp.size,
                            coef_ent=hp.ent, coef_lap=hp.lap, coef_feat_size=hp.feat_size, opt=_abi.GX_OPT[hp.opt],
                            opt_scheduler=_abi.GX_SCHED[hp.opt_scheduler], opt_decay_step=hp.opt_decay_step,
                            opt_decay_rate=hp.opt_decay_rate, opt_restart=hp.opt_restart, **extra)


def node_path(eng, path):
    """Route the next plan_nodes to a kernel: the shared-memory kernel, its cluster class, the gang or first-generation streaming kernel."""
    if path.startswith("cluster"):
        eng.debug_cluster(int(path[-1]), 1)
    elif path in ("gang", "stream1"):
        eng.debug_force_stream(True)
        eng.debug_gang(0 if path == "gang" else -1)


def fixture_engine(which, path):
    fx = util.load_fixture(which)
    eng = util.make_engine(fx)
    node_path(eng, path)
    return fx, eng


def run_nodes(eng, plan, hp, m0, d):
    out = np.zeros(plan.total_edges, np.float32)
    fm = np.zeros((plan.count, d), np.float32)
    eng.explain_nodes_host(hp, m0, out, fm)
    return out, fm


def run_graphs(eng, gids, hp, dense, d):
    rc = {g: eng.graph_rows_cols(g) for g in gids}
    edge_off = eng.plan_graphs(gids)
    out = np.zeros(int(edge_off[-1]), np.float32)
    fm = np.zeros((len(gids), d), np.float32)
    eng.explain_graphs_host(hp, np.concatenate([dense[g][rc[g]] for g in gids]).astype(np.float32), out, fm)
    return [(out[edge_off[t]:edge_off[t + 1]], fm[t], rc[g]) for t, g in enumerate(gids)]


def fixture_inputs(fx, node, L=3):
    idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(fx.rowptr, fx.col, fx.feat, fx.label, node, L)
    return O.dense_from_csr(srp, scol), X, int(lab[idx]), fx.pred_label[nbrs], idx


def dense_of_edges(plan, t, m0):
    M = np.ones((plan.n(t), plan.n(t)), np.float32)
    r, c = plan.rows_cols_of(t)
    M[r, c] = m0[plan.edge_off[t]:plan.edge_off[t + 1]]
    return M


def graph_m0():
    return {g: O.draw_m0(NMAX, seed=int(GG["g%d_seed" % g])) for g in range(NG)}


# ------------------------------------------------------------------------------------ a. the reference under lr / epochs / schedulers
@pytest.mark.parametrize("path", NODE_PATHS)
@pytest.mark.parametrize("which", ["rand", "syn4", "syn1"])
def test_reference_cases_on_node_kernels(which, path):
    fx, eng = fixture_engine(which, path)
    bad = {}
    for tag in TAGS:
        E, hp = case_hparams(H, tag)
        nodes = [int(v) for v in H["%s_%s_nodes" % (which, tag)]]
        spread = dict(zip(nodes, H["%s_%s_spread" % (which, tag)]))
        plan = eng.plan_nodes(nodes, 3)
        if path == "smem" and tag == TAGS[0]:
            counts, _ = eng.plan_class_counts()
            print("%s launch classes %s" % (which, counts.tolist()))
        out, _ = run_nodes(eng, plan, to_gx(eng, hp), util.golden_m0(fx, plan), fx.feat.shape[1])
        for t, node in enumerate(nodes):
            err = util.rel_l2(out[plan.edge_off[t]:plan.edge_off[t + 1]], H["%s_%s_n%d_mask" % (which, tag, node)])
            tol = max(1e-4, 3 * float(spread[node]))
            if not err <= tol:
                bad[(tag, node)] = (err, tol)
    eng.close()
    assert not bad, bad


def test_reference_batches_cover_every_shared_memory_class():
    seen = np.zeros(7, np.int64)
    for which in ("rand", "syn4", "syn1"):
        fx, eng = fixture_engine(which, "smem")
        eng.plan_nodes([int(v) for v in H[which + "_nodes"]], 3)
        counts, _ = eng.plan_class_counts()
        seen += counts
        eng.close()
    assert (seen[:SMEM_CLASSES] > 0).all(), seen


def test_reference_cases_on_graph_kernel():
    eng = gnnx.Engine(0)
    eng.set_model(GW)
    eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
    dense = graph_m0()
    bad = {}
    for tag in TAGS:
        E, hp = case_hparams(H, tag)
        gids = [int(g) for g in H["graphs_%s_gids" % tag]]
        for (out, _, _), g, s in zip(run_graphs(eng, gids, to_gx(eng, hp), dense, GG["feat"].shape[2]), gids, H["graphs_%s_spread" % tag]):
            err = util.rel_l2(out, H["graphs_%s_g%d_mask" % (tag, g)])
            if not err <= max(1e-4, 3 * float(s)):
                bad[(tag, g)] = (err, max(1e-4, 3 * float(s)))
    eng.close()
    assert not bad, bad


def test_explainer_dropin_lr_and_epochs(tmp_path):
    """Explainer with args.lr = 0.01 and args.num_epochs = 300 reproduces the reference under its torch seeding."""
    from test_gpu_parity import _explainer
    fx = util.load_fixture("syn1")
    ex, _ = _explainer(fx, tmp_path, num_epochs=300, lr=0.01)
    spread = dict(zip((int(v) for v in H["syn1_e300_nodes"]), H["syn1_e300_spread"]))
    for node in spread:
        torch.manual_seed(int(fx.gold["n%d_seed" % node]))
        masked = ex.explain(node, graph_idx=0)
        _, sub_adj, _, _, _ = ex.extract_neighborhood(node)
        ei, ej = np.nonzero(sub_adj)
        assert util.rel_l2(masked[ei, ej], H["syn1_e300_n%d_mask" % node]) <= max(1e-4, 3 * float(spread[node])), node


# ------------------------------------------------------------------------------------ b. H1 / H2 / H0 against the ports
def check_port(got, fm, port, hset, E):
    """got / fm vs port(hp, dtype) -> (mask, feature mask or None): edge mask within max(1e-4, 3 x dis), dis = the port's fp32 / fp64
    distance; feature mask within max(2e-4, 30 x dis) of the fp64 port; and the set moves the port by more than 10 x the tolerance."""
    hp = O.default_hparams(num_epochs=E, **HSETS[hset])
    p32, f32 = port(hp, torch.float)
    p64, f64 = port(hp, torch.float64)
    dis = O.rel_l2(p64, p32)
    tol = max(1e-4, 3 * dis)
    err = O.rel_l2(got, p32)
    assert err <= tol, ("edge mask", err, tol)
    if fm is not None:
        ferr = float(np.abs(np.asarray(fm, np.float64) - f64).max())
        assert ferr <= max(2e-4, 30 * dis), ("feature mask", ferr, max(2e-4, 30 * dis))
    base, _ = port(O.default_hparams(num_epochs=E), torch.float)
    assert O.rel_l2(base, p32) > 10 * tol, ("the set changes nothing", O.rel_l2(base, p32), tol)


def wide_port(A, X, gt, pl, idx, w, M0, graph_mode=False, bn=False):
    return lambda hp, dt: O.explain_dense_torch(A, X, gt, pl, idx, w, M0, hp=hp, graph_mode=graph_mode, bn=bn, dtype=dt, return_feat=True)


def att_port(A, X, gt, pl, idx, w, M0, graph_mode=False, bn=False):
    return lambda hp, dt: O.explain_dense_torch(A, X, gt, pl, idx, w, M0, hp=hp, graph_mode=graph_mode, bn=bn, dtype=dt, return_feat=True)


E_SET = 20


@pytest.mark.parametrize("hset", list(HSETS))
@pytest.mark.parametrize("path", NODE_PATHS)
def test_sets_on_tuned_node_kernels(path, hset):
    fx, eng = fixture_engine("rand", path)
    nodes = [33, 149, 77]
    plan = eng.plan_nodes(nodes, 3)
    m0 = util.golden_m0(fx, plan)
    out, fm = run_nodes(eng, plan, eng.make_hparams(num_epochs=E_SET, **gx_over(hset)), m0, fx.feat.shape[1])
    eng.close()
    for t, node in enumerate(nodes):
        A, X, gt, pl, idx = fixture_inputs(fx, node)
        check_port(plan.dense_of(t, out), fm[t], wide_port(A, X, gt, pl, idx, fx.weights, dense_of_edges(plan, t, m0)), hset, E_SET)


@pytest.mark.parametrize("hset", list(HSETS))
def test_sets_on_graph_kernel(hset):
    eng = gnnx.Engine(0)
    eng.set_model(GW)
    eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
    gids = [0, 4, 7, 10]
    dense = graph_m0()
    res = run_graphs(eng, gids, eng.make_hparams(num_epochs=E_SET, **gx_over(hset)), dense, GG["feat"].shape[2])
    eng.close()
    for (out, fm, rc), g in zip(res, gids):
        Dm = np.zeros((NMAX, NMAX)); Dm[rc] = out
        check_port(Dm, fm, wide_port(GG["adj"][g].astype(np.float64), GG["feat"][g], int(GG["label"][g]), None, 0, GW, dense[g], True), hset, E_SET)


VAR_MODELS = {"L2": (2, False, 20, 20, 10), "bn": (3, True, 20, 20, 10), "wide": (3, False, 20, 20, 300)}   # L, bn, hid, emb, d


@pytest.mark.parametrize("hset", list(HSETS))
@pytest.mark.parametrize("model", list(VAR_MODELS))
def test_sets_on_variant_kernel_nodes(model, hset):
    L, bn, hid, emb, d = VAR_MODELS[model]
    s = _node_setup(40 + L + int(bn), L, bn, hid, emb, d, 3)
    nodes = [0, 7, 23]
    plan = s.eng.plan_nodes(nodes, L)
    dense = [O.draw_m0(plan.n(t), seed=90 + t) for t in range(plan.count)]
    m0 = np.concatenate([dense[t][plan.rows_cols_of(t)] for t in range(plan.count)]).astype(np.float32)
    out, fm = run_nodes(s.eng, plan, s.eng.make_hparams(num_epochs=E_SET, **gx_over(hset)), m0, d)
    s.eng.close()
    for t, node in enumerate(nodes):
        idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(s.rowptr, s.col, s.feat, s.label, node, L)
        port = wide_port(O.dense_from_csr(srp, scol), X, int(lab[idx]), s.pred_label[nbrs], idx, s.w, dense[t], bn=bn)
        check_port(plan.dense_of(t, out), fm[t], port, hset, E_SET)


@pytest.mark.parametrize("hset", list(HSETS))
@pytest.mark.parametrize("model", list(VAR_MODELS))
def test_sets_on_variant_kernel_graphs(model, hset):
    L, bn, hid, emb, d = VAR_MODELS[model]
    adj, feat, label, w, eng = _graph_setup(50 + L + int(bn), L, bn, hid, emb, max(d, 14), 3)
    gids = [1, 5, 9]
    dense = {g: O.draw_m0(NMAX, seed=70 + g) for g in gids}
    res = run_graphs(eng, gids, eng.make_hparams(num_epochs=E_SET, **gx_over(hset)), dense, feat.shape[2])
    eng.close()
    for (out, fm, rc), g in zip(res, gids):
        Dm = np.zeros((NMAX, NMAX)); Dm[rc] = out
        check_port(Dm, fm, wide_port(np.asarray(adj[g], np.float64), feat[g], int(label[g]), None, 0, w, dense[g], True, bn), hset, E_SET)


@pytest.mark.parametrize("hset", list(HSETS))
def test_sets_on_attention_kernel(hset):
    rng = np.random.default_rng(31)
    w = random_att_model(rng, 10, 20, 20, 3, 3)
    att = [w["Wa%d" % l] for l in range(1, 4)]
    # node mode
    rowptr, col = O.csr_from_edges(48, np.array(nx.barabasi_albert_graph(48, 2, seed=31).edges(), dtype=np.int64))
    feat = rng.normal(size=(48, 10)).astype(np.float32)
    label = rng.integers(0, 3, 48).astype(np.int32)
    pred_label = np.argmax(O.model_pred(O.dense_from_csr(rowptr, col), feat, w), 1).astype(np.int32)
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=3, att=att)
    eng.set_graph_csr(rowptr, col, feat, label, pred_label)
    nodes = [0, 7, 23]
    plan = eng.plan_nodes(nodes, 3)
    dense = [O.draw_m0(plan.n(t), seed=60 + t) for t in range(plan.count)]
    m0 = np.concatenate([dense[t][plan.rows_cols_of(t)] for t in range(plan.count)]).astype(np.float32)
    out, fm = run_nodes(eng, plan, eng.make_hparams(num_epochs=E_SET, **gx_over(hset)), m0, 10)
    eng.close()
    for t, node in enumerate(nodes):
        idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(rowptr, col, feat, label, node, 3)
        check_port(plan.dense_of(t, out), fm[t], att_port(O.dense_from_csr(srp, scol), X, int(lab[idx]), pred_label[nbrs], idx, w, dense[t]),
                   hset, E_SET)
    # graph mode
    wg = random_att_model(rng, GG["feat"].shape[2], 20, 20, GW["Wp"].shape[0], 3)
    eng = gnnx.Engine(0)
    eng.set_model(wg, num_layers=3, att=[wg["Wa%d" % l] for l in range(1, 4)])
    eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
    gids = [2, 6, 11]
    dense = graph_m0()
    res = run_graphs(eng, gids, eng.make_hparams(num_epochs=E_SET, **gx_over(hset)), dense, GG["feat"].shape[2])
    eng.close()
    for (out, fm, rc), g in zip(res, gids):
        Dm = np.zeros((NMAX, NMAX)); Dm[rc] = out
        check_port(Dm, fm, att_port(GG["adj"][g].astype(np.float64), GG["feat"][g], int(GG["label"][g]), None, 0, wg, dense[g], True), hset, E_SET)


def _dense_run(graphs, hp_gx, seeds_or_gids, eng, plan=None):
    if graphs:
        m0 = [O.draw_m0(NMAX, seed=int(GG["g%d_seed" % g])) for g in seeds_or_gids]
        edge_off = eng.plan_graphs(seeds_or_gids)
        out = np.zeros(max(int(edge_off[-1]), 1), np.float32)
        eng.explain_graphs_unconstrained(hp_gx, np.concatenate([M.ravel() for M in m0]), out)
        return m0, [out[edge_off[t]:edge_off[t + 1]] for t in range(len(seeds_or_gids))]
    m0 = [O.draw_m0(plan.n(t), seed=seeds_or_gids[t]) for t in range(plan.count)]
    out = np.zeros(max(plan.total_edges, 1), np.float32)
    eng.explain_nodes_unconstrained(hp_gx, np.concatenate([M.ravel() for M in m0]), out)
    return m0, [out[plan.edge_off[t]:plan.edge_off[t + 1]] for t in range(plan.count)]


@pytest.mark.parametrize("hset", list(HSETS))
def test_sets_on_dense_kernel(hset):
    """unconstrained=True: the edge masks against the port within max(1e-4, 3 x its distance to the fp64 closed form)."""
    hp = O.default_hparams(num_epochs=E_SET, **HSETS[hset])
    fx = util.load_fixture("rand")
    eng = util.make_engine(fx)
    nodes = [33, 149]
    plan = eng.plan_nodes(nodes, 3)
    m0, outs = _dense_run(False, to_gx(eng, hp), [int(fx.gold["n%d_seed" % v]) for v in nodes], eng, plan)
    eng.close()
    cases = []
    for t, node in enumerate(nodes):
        A, X, gt, pl, idx = fixture_inputs(fx, node)
        cases.append((outs[t], (A, X, gt, pl, idx, fx.weights, m0[t]), False))
    eng = gnnx.Engine(0)
    eng.set_model(GW)
    eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
    gids = [3, 8]
    m0, outs = _dense_run(True, to_gx(eng, hp), gids, eng)
    eng.close()
    for t, g in enumerate(gids):
        cases.append((outs[t], (GG["adj"][g].astype(np.float64), GG["feat"][g], int(GG["label"][g]), None, 0, GW, m0[t]), True))
    for got, args, graph_mode in cases:
        ei, ej = np.nonzero(args[0])
        port = O.explain_dense_torch(*args, hp=hp, graph_mode=graph_mode, unconstrained=True)[ei, ej]
        cf = D.explain_closed_form(*args, hp=hp, graph_mode=graph_mode)[ei, ej]
        tol = max(1e-4, 3 * O.rel_l2(cf, port))
        assert O.rel_l2(got, port) <= tol, (hset, graph_mode, O.rel_l2(got, port), tol)
        base = O.explain_dense_torch(*args, hp=O.default_hparams(num_epochs=E_SET), graph_mode=graph_mode, unconstrained=True)[ei, ej]
        assert O.rel_l2(base, port) > 10 * tol, (hset, graph_mode)


# ------------------------------------------------------------------------------------ c. lr = 0 and d. one update
def _sym_sigmoid(M):
    S = 1 / (1 + np.exp(-np.asarray(M, np.float64)))
    return (S + S.T) / 2


ALL_NODE_PATHS = NODE_PATHS + ["variant", "wide", "att", "dense"]


def _node_case(path):
    """(engine, plan, dense M0 list, inputs of task t, weights, bn, d) of a small node batch routed to `path`."""
    if path in NODE_PATHS or path == "dense":
        fx, eng = fixture_engine("rand", path if path != "dense" else "smem")
        nodes = [33, 149, 0]
        plan = eng.plan_nodes(nodes, 3)
        dense = [dense_of_edges(plan, t, util.golden_m0(fx, plan)) for t in range(plan.count)]
        return eng, plan, dense, (lambda t: fixture_inputs(fx, nodes[t])), fx.weights, False, fx.feat.shape[1], 3
    if path == "att":
        rng = np.random.default_rng(32)
        w = random_att_model(rng, 10, 20, 20, 3, 3)
        rowptr, col = O.csr_from_edges(48, np.array(nx.barabasi_albert_graph(48, 2, seed=32).edges(), dtype=np.int64))
        feat = rng.normal(size=(48, 10)).astype(np.float32)
        label = rng.integers(0, 3, 48).astype(np.int32)
        pl = np.argmax(O.model_pred(O.dense_from_csr(rowptr, col), feat, w), 1).astype(np.int32)
        eng = gnnx.Engine(0)
        eng.set_model(w, num_layers=3, att=[w["Wa%d" % l] for l in range(1, 4)])
        eng.set_graph_csr(rowptr, col, feat, label, pl)
        s = type("S", (), dict(rowptr=rowptr, col=col, feat=feat, label=label, pred_label=pl, eng=eng, w=w, L=3, bn=False, d=10))
    else:
        L, bn, hid, emb, d = VAR_MODELS["bn" if path == "variant" else "wide"]
        s = _node_setup(80 + d, L, bn, hid, emb, d, 3)
    nodes = [0, 7, 23]
    plan = s.eng.plan_nodes(nodes, s.L)
    dense = [O.draw_m0(plan.n(t), seed=40 + t) for t in range(plan.count)]

    def inputs(t):
        idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(s.rowptr, s.col, s.feat, s.label, nodes[t], s.L)
        return O.dense_from_csr(srp, scol), X, int(lab[idx]), s.pred_label[nbrs], idx
    return s.eng, plan, dense, inputs, s.w, s.bn, s.d, s.L


def _edges_of(plan, dense):
    return np.concatenate([dense[t][plan.rows_cols_of(t)] for t in range(plan.count)]).astype(np.float32)


@pytest.mark.parametrize("path", ALL_NODE_PATHS)
def test_lr_zero_returns_the_initial_mask_nodes(path):
    eng, plan, dense, _, _, _, d, _ = _node_case(path)
    hp = eng.make_hparams(num_epochs=12, lr=0.0, **gx_over("H2"))
    if path == "dense":
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_unconstrained(hp, np.concatenate([M.ravel() for M in dense]), out)
        fm = None
    else:
        out, fm = run_nodes(eng, plan, hp, _edges_of(plan, dense), d)
    eng.close()
    for t in range(plan.count):
        r, c = plan.rows_cols_of(t)
        want = _sym_sigmoid(dense[t])[r, c]
        assert np.abs(out[plan.edge_off[t]:plan.edge_off[t + 1]] - want).max() <= 1e-6, (path, t)
    if fm is not None:
        assert (fm == 0.5).all(), path


@pytest.mark.parametrize("path", ["graph", "variant", "wide", "att", "dense"])
def test_lr_zero_returns_the_initial_mask_graphs(path):
    eng, w, bn, adj, feat, label = _graph_case(path)
    gids = [0, 5, 9]
    dense = graph_m0()
    hp = eng.make_hparams(num_epochs=12, lr=0.0, **gx_over("H2"))
    if path == "dense":
        edge_off = eng.plan_graphs(gids)
        out = np.zeros(int(edge_off[-1]), np.float32)
        eng.explain_graphs_unconstrained(hp, np.concatenate([dense[g].ravel() for g in gids]), out)
        res = [(out[edge_off[t]:edge_off[t + 1]], None, eng.graph_rows_cols(g)) for t, g in enumerate(gids)]
    else:
        res = run_graphs(eng, gids, hp, dense, feat.shape[2])
    eng.close()
    for (out, fm, rc), g in zip(res, gids):
        assert np.abs(out - _sym_sigmoid(dense[g])[rc]).max() <= 1e-6, (path, g)
        if fm is not None:
            assert (fm == 0.5).all(), path


def _graph_case(path):
    if path in ("graph", "dense"):
        eng = gnnx.Engine(0)
        eng.set_model(GW)
        eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
        return eng, GW, False, GG["adj"], GG["feat"], GG["label"]
    if path == "att":
        w = random_att_model(np.random.default_rng(33), GG["feat"].shape[2], 20, 20, GW["Wp"].shape[0], 3)
        eng = gnnx.Engine(0)
        eng.set_model(w, num_layers=3, att=[w["Wa%d" % l] for l in range(1, 4)])
        eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
        return eng, w, False, GG["adj"], GG["feat"], GG["label"]
    L, bn, hid, emb, d = VAR_MODELS["bn" if path == "variant" else "wide"]
    adj, feat, label, w, eng = _graph_setup(90 + d, L, bn, hid, emb, max(d, 14), 3)
    return eng, w, bn, adj, feat, label


@pytest.mark.parametrize("hset", ["H1", "H2"])
@pytest.mark.parametrize("path", ALL_NODE_PATHS)
def test_one_update_matches_fp64_nodes(path, hset):
    eng, plan, dense, inputs, w, bn, d, _ = _node_case(path)
    hp = O.default_hparams(num_epochs=2, **HSETS[hset])
    if path == "dense":
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_unconstrained(to_gx(eng, hp), np.concatenate([M.ravel() for M in dense]), out)
        fm = None
    else:
        out, fm = run_nodes(eng, plan, to_gx(eng, hp), _edges_of(plan, dense), d)
    eng.close()
    for t in range(plan.count):
        args = inputs(t) + (w, dense[t])
        if path == "dense":
            ref, f1 = D.explain_closed_form(*args, hp=hp), None
        elif path == "att":
            ref, f1 = O.explain_dense_torch(*args, hp=hp, dtype=torch.float64, return_feat=True)
        elif path in ("variant", "wide"):
            ref, f1 = O.explain_dense_torch(*args, hp=hp, bn=bn, dtype=torch.float64, return_feat=True)
        else:
            ref = O.explain_closed_form(*args, hp=hp)
            _, st = O.explain_closed_form(*args, hp=O.default_hparams(num_epochs=1, **HSETS[hset]), return_state=True)
            f1 = 1 / (1 + np.exp(-st["F"]))
        r, c = plan.rows_cols_of(t)
        assert O.rel_l2(out[plan.edge_off[t]:plan.edge_off[t + 1]], ref[r, c]) <= 1e-5, (path, t)
        if fm is not None:
            assert np.abs(fm[t] - f1).max() <= 1e-5, (path, t)


@pytest.mark.parametrize("hset", ["H1", "H2"])
@pytest.mark.parametrize("path", ["graph", "variant", "wide", "att", "dense"])
def test_one_update_matches_fp64_graphs(path, hset):
    eng, w, bn, adj, feat, label = _graph_case(path)
    gids = [0, 5, 9]
    dense = graph_m0()
    hp = O.default_hparams(num_epochs=2, **HSETS[hset])
    if path == "dense":
        edge_off = eng.plan_graphs(gids)
        out = np.zeros(int(edge_off[-1]), np.float32)
        eng.explain_graphs_unconstrained(to_gx(eng, hp), np.concatenate([dense[g].ravel() for g in gids]), out)
        res = [(out[edge_off[t]:edge_off[t + 1]], None, eng.graph_rows_cols(g)) for t, g in enumerate(gids)]
    else:
        res = run_graphs(eng, gids, to_gx(eng, hp), dense, feat.shape[2])
    eng.close()
    for (out, fm, rc), g in zip(res, gids):
        args = (np.asarray(adj[g], np.float64), feat[g], int(label[g]), None, 0, w, dense[g])
        if path == "dense":
            ref, f1 = D.explain_closed_form(*args, hp=hp, graph_mode=True), None
        elif path == "att":
            ref, f1 = O.explain_dense_torch(*args, hp=hp, graph_mode=True, dtype=torch.float64, return_feat=True)
        elif path in ("variant", "wide"):
            ref, f1 = O.explain_dense_torch(*args, hp=hp, graph_mode=True, bn=bn, dtype=torch.float64, return_feat=True)
        else:
            ref = O.explain_closed_form(*args, hp=hp, graph_mode=True)
            _, st = O.explain_closed_form(*args, hp=O.default_hparams(num_epochs=1, **HSETS[hset]), graph_mode=True, return_state=True)
            f1 = 1 / (1 + np.exp(-st["F"]))
        assert O.rel_l2(out, ref[rc]) <= 1e-5, (path, g)
        if fm is not None:
            assert np.abs(fm - f1).max() <= 1e-5, (path, g)


# ------------------------------------------------------------------------------------ e. trace columns and limits
TRACE_SETS = {"H2": dict(HSETS["H2"]), "H2_nolap": dict(HSETS["H2"], lap=0.0)}


def _assert_trace(row_of, tr, hp, n, off, what):
    for e in range(len(tr)):
        row = row_of(e)
        ref = tr[e]
        pairs = [(row[_abi.TR_SIZE], ref["size_edges"]), (row[_abi.TR_ENT], ref["ent_edges"]), (row[_abi.TR_LAP], ref["lap"]),
                 (row[_abi.TR_FEAT], ref["feat_size"])]
        if off is not None:
            pairs.append((row[_abi.TR_LOSS_EDGES] + hp.size * off[e, 0] + hp.ent * off[e, 1] / (n * n), ref["loss"]))
        for k, (got, want) in enumerate(pairs):
            assert abs(got - want) <= 2e-5 * abs(want) + 1e-7, (what, e, k, got, want)
    if hp.lap == 0:
        assert all(row_of(e)[_abi.TR_LAP] == 0 for e in range(len(tr)))


@pytest.mark.parametrize("tset", list(TRACE_SETS))
@pytest.mark.parametrize("path", ["smem", "gang", "stream1"])
def test_trace_columns_under_coefficients_nodes(path, tset):
    fx, eng = fixture_engine("rand", path)
    nodes = [33, 149, 77]
    plan = eng.plan_nodes(nodes, 3)
    E = 12
    hp = O.default_hparams(num_epochs=E, **TRACE_SETS[tset])
    m0 = util.golden_m0(fx, plan)
    dense = [dense_of_edges(plan, t, m0) for t in range(plan.count)]
    out = np.zeros(plan.total_edges, np.float32)
    trace = np.zeros((plan.count, E, _abi.GX_TRACE_COLS), np.float32)
    eng.explain_nodes_ex(to_gx(eng, hp), m0, out, trace=trace)
    off = eng.offedge_regularisers(to_gx(eng, hp), np.concatenate([M.ravel() for M in dense]))
    eng.close()
    for t, node in enumerate(nodes):
        A, X, gt, pl, idx = fixture_inputs(fx, node)
        tr = []
        O.explain_dense_torch(A, X, gt, pl, idx, fx.weights, dense[t], hp=hp, trace=tr)
        _assert_trace(lambda e: trace[t, e], tr, hp, plan.n(t), off[t], (path, tset, node))


@pytest.mark.parametrize("tset", list(TRACE_SETS))
def test_trace_columns_under_coefficients_graphs(tset):
    eng = gnnx.Engine(0)
    eng.set_model(GW)
    eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
    gids = [0, 3, 7]
    E = 12
    hp = O.default_hparams(num_epochs=E, **TRACE_SETS[tset])
    dense = graph_m0()
    edge_off = eng.plan_graphs(gids)
    rcs = [eng.graph_rows_cols(g) for g in gids]
    m0 = np.concatenate([dense[g][rc] for g, rc in zip(gids, rcs)]).astype(np.float32)
    out = np.zeros(int(edge_off[-1]), np.float32)
    trace = np.zeros((len(gids), E, _abi.GX_TRACE_COLS), np.float32)
    eng.explain_nodes_ex(to_gx(eng, hp), m0, out, trace=trace, graphs=True)
    eng.close()
    for t, g in enumerate(gids):
        tr = []
        O.explain_dense_torch(GG["adj"][g].astype(np.float64), GG["feat"][g], int(GG["label"][g]), None, 0, GW, dense[g], hp=hp, graph_mode=True, trace=tr)
        _assert_trace(lambda e: trace[t, e], tr, hp, NMAX, None, ("graph", tset, g))


def test_trace_epoch_limits():
    fx, eng = fixture_engine("rand", "smem")
    nodes = [149, 33]
    plan = eng.plan_nodes(nodes, 3)
    m0 = util.golden_m0(fx, plan)
    dense = np.concatenate([dense_of_edges(plan, t, m0).ravel() for t in range(plan.count)])

    def trace_of(E):
        out = np.zeros(plan.total_edges, np.float32)
        tr = np.zeros((plan.count, E, _abi.GX_TRACE_COLS), np.float32)
        eng.explain_nodes_ex(eng.make_hparams(num_epochs=E, **gx_over("H2")), m0, out, trace=tr)
        return tr
    long, short = trace_of(1536), trace_of(100)
    assert long.shape[1] == 1536 and np.isfinite(short).all()
    assert np.array_equal(long[:, :100], short)
    with pytest.raises(_abi.GnnxError) as e:
        trace_of(1537)
    assert e.value.status == GX_ERR_UNSUPPORTED
    off = eng.offedge_regularisers(eng.make_hparams(num_epochs=3072, **gx_over("H2")), dense)
    assert off.shape == (plan.count, 3072, 2)
    assert np.array_equal(off[:, :100], eng.offedge_regularisers(eng.make_hparams(num_epochs=100, **gx_over("H2")), dense))
    with pytest.raises(_abi.GnnxError) as e:
        eng.offedge_regularisers(eng.make_hparams(num_epochs=3073), dense)
    assert e.value.status == GX_ERR_INVALID
    eng.close()


# ------------------------------------------------------------------------------------ f. resume under schedulers
SCHEDS = {"step": dict(opt_scheduler=_abi.GX_SCHED["step"], opt_decay_step=5, opt_decay_rate=0.5),   # boundaries 15, 20, 25 in the 2nd call
          "cos": dict(opt_scheduler=_abi.GX_SCHED["cos"], opt_restart=8)}                           # T_max 8 < 30 epochs


@pytest.mark.parametrize("sched", list(SCHEDS))
@pytest.mark.parametrize("path", ["smem", "gang", "stream1", "graph"])
def test_resume_under_schedulers_is_bit_identical(path, sched):
    E, E1 = 30, 13
    if path == "graph":
        eng = gnnx.Engine(0)
        eng.set_model(GW)
        eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
        gids = [0, 3, 7]
        edge_off = eng.plan_graphs(gids)
        dense = graph_m0()
        m0 = np.concatenate([dense[g][eng.graph_rows_cols(g)] for g in gids]).astype(np.float32)
        te, count, d = int(edge_off[-1]), len(gids), GG["feat"].shape[2]
    else:
        fx, eng = fixture_engine("rand", path)
        plan = eng.plan_nodes([33, 149, 0], 3)
        m0 = util.golden_m0(fx, plan)
        te, count, d = plan.total_edges, plan.count, fx.feat.shape[1]
    graphs = path == "graph"
    full = np.zeros(te, np.float32); fm_full = np.zeros((count, d), np.float32)
    eng.explain_nodes_ex(eng.make_hparams(num_epochs=E, **SCHEDS[sched]), m0, full, fm_full, graphs=graphs)
    so = dict(M=np.zeros(te, np.float32), m=np.zeros(te, np.float32), v=np.zeros(te, np.float32), feat=np.zeros((count, 3, d), np.float32))
    part = np.zeros(te, np.float32)
    eng.explain_nodes_ex(eng.make_hparams(num_epochs=E1, **SCHEDS[sched]), m0, part, state_out=so, graphs=graphs)
    rest = np.zeros(te, np.float32); fm = np.zeros((count, d), np.float32)
    eng.explain_nodes_ex(eng.make_hparams(num_epochs=E - E1 + 1, init=_abi.GX_INIT_STATE, start_step=E1 - 1, **SCHEDS[sched]), so["M"], rest,
                         fm, state_in=dict(m=so["m"], v=so["v"], feat=so["feat"]), graphs=graphs)
    # the same split without the scheduler lands elsewhere: the second call did run the scheduled rates
    plain = np.zeros(te, np.float32)
    eng.explain_nodes_ex(eng.make_hparams(num_epochs=E - E1 + 1, init=_abi.GX_INIT_STATE, start_step=E1 - 1), so["M"], plain,
                         state_in=dict(m=so["m"], v=so["v"], feat=so["feat"]), graphs=graphs)
    eng.close()
    assert np.array_equal(rest, full) and np.array_equal(fm, fm_full)
    assert util.rel_l2(plain, full) > 1e-3


# ------------------------------------------------------------------------------------ g. the table cache of one handle
def test_table_cache_follows_every_setting_on_one_handle():
    fx = util.load_fixture("rand")
    nodes = [33, 149, 0]
    d = fx.feat.shape[1]
    A = dict(num_epochs=20, lr=0.05, opt_scheduler=_abi.GX_SCHED["step"], opt_decay_step=4, opt_decay_rate=0.5)
    B = dict(A, beta2=0.99)
    A2 = dict(A, opt_decay_rate=0.7)
    C = dict(num_epochs=20, opt_scheduler=_abi.GX_SCHED["cos"], opt_restart=6, beta1=0.8)

    def node_call(eng, hp, state=None):
        eng.set_graph_csr(fx.rowptr, fx.col, fx.feat, fx.label, fx.pred_label)
        plan = eng.plan_nodes(nodes, 3)
        m0 = util.golden_m0(fx, plan)
        out = np.zeros(plan.total_edges, np.float32); fm = np.zeros((plan.count, d), np.float32)
        so = dict(M=np.zeros(plan.total_edges, np.float32), m=np.zeros(plan.total_edges, np.float32),
                  v=np.zeros(plan.total_edges, np.float32), feat=np.zeros((plan.count, 3, d), np.float32))
        if state is None:
            eng.explain_nodes_ex(eng.make_hparams(**hp), m0, out, fm, state_out=so)
        else:
            eng.explain_nodes_ex(eng.make_hparams(init=_abi.GX_INIT_STATE, **hp), state["M"], out, fm,
                                 state_in=dict(m=state["m"], v=state["v"], feat=state["feat"]), state_out=so)
        return out, fm, so

    def graph_call(eng, hp):
        eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
        return tuple(x for r in run_graphs(eng, [1, 4, 8], eng.make_hparams(**hp), graph_m0(), GG["feat"].shape[2]) for x in r[:2])

    def fresh(call, *a):
        eng = gnnx.Engine(0)
        eng.set_model(GW if call is graph_call else fx.weights)
        res = call(eng, *a)
        eng.close()
        return res

    def equal(x, y):
        return all(np.array_equal(a, b) for a, b in zip(x, y))

    eng = gnnx.Engine(0)
    eng.set_model(fx.weights)
    ra = node_call(eng, A)
    st = ra[2]
    seq = [(node_call, (A,)), (node_call, (B,)), (node_call, (A,)), (node_call, (A2,)),
           (node_call, (dict(A, start_step=5), st)), (node_call, (dict(A, start_step=6), st)), (node_call, (A,))]
    got = [node_call(eng, *a) for _, a in seq[1:]]
    eng.set_model(GW)
    gC = graph_call(eng, C)
    eng.set_model(fx.weights)
    last = node_call(eng, A)
    eng.close()
    want = [fresh(c, *a) for c, a in seq[1:]]
    assert equal(ra[:2], fresh(node_call, A)[:2])
    for k, (g, w) in enumerate(zip(got, want)):
        assert equal(g[:2], w[:2]), seq[k + 1][1][0]
    assert equal(gC, fresh(graph_call, C))
    assert equal(last[:2], ra[:2])
    assert not np.array_equal(got[0][0], ra[0]) and not np.array_equal(got[2][0], ra[0])   # beta2 and the decay rate do change the masks
    assert not np.array_equal(got[3][0], got[4][0])                                        # and so does start_step


# ------------------------------------------------------------------------------------ i. refusals
@pytest.mark.parametrize("over", [dict(opt_scheduler=1, opt_decay_step=0), dict(opt_scheduler=2, opt_restart=0), dict(opt=4), dict(opt=-1)],
                         ids=["step_decay0", "cos_restart0", "opt4", "opt-1"])
def test_refuses_invalid_optimiser_settings(over):
    fx, eng = fixture_engine("rand", "smem")
    plan = eng.plan_nodes([33], 3)
    m0 = util.golden_m0(fx, plan)
    out = np.zeros(plan.total_edges, np.float32)
    with pytest.raises(_abi.GnnxError) as e:
        eng.explain_nodes_host(eng.make_hparams(num_epochs=5, **over), m0, out)
    assert e.value.status == GX_ERR_INVALID
    eng.close()
    eng = gnnx.Engine(0)
    eng.set_model(GW)
    eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
    te = int(eng.plan_graphs([0])[-1])
    with pytest.raises(_abi.GnnxError) as e:
        eng.explain_graphs_host(eng.make_hparams(num_epochs=5, **over), np.zeros(te, np.float32), np.zeros(te, np.float32))
    assert e.value.status == GX_ERR_INVALID
    eng.close()
