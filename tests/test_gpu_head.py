"""GPU (-m gpu): models with an MLP prediction head (pred_hidden_dims, models.py:193-207) on the model-variant kernel (explain_var.cu), the
unconstrained kernel (explain_dense.cu) and the model forward (forward.cu), through the C ABI and the drop-in Explainer, node and graph
mode: against the torch port (oracle/gnnx_oracle.explain_dense_torch) in fp32 and fp64."""
import types

import numpy as np
import pytest
import torch

import gnnx
import gnnx_oracle as O
from gnnx import _abi
import util
from test_gpu_deep import GG, _hp, _m0, _ohp, random_model
from test_oracle_head import GOLDEN, case_feat, case_weights, golden_cases

pytestmark = pytest.mark.gpu
GX_ERR_UNSUPPORTED = -3


def head_model(rng, d, hid, emb, C, L, widths, att=False):
    """random_model plus hidden head Linears (out, in), each scaled by 1.5 / sqrt(fan-in), biases N(0, 0.3); Wp / bp the last Linear."""
    w = random_model(rng, d, hid, emb, C, L, att)
    fan = hid * (L - 1) + emb
    head = []
    for h in widths:
        head.append(((rng.normal(size=(h, fan)) * 1.5 / np.sqrt(fan)).astype(np.float32), (rng.normal(size=h) * 0.3).astype(np.float32)))
        fan = h
    w["head"] = head
    w["Wp"] = (rng.normal(size=(C, fan)) * 1.5 / np.sqrt(fan)).astype(np.float32)
    return w


def _set(eng, w, L, bn):
    eng.set_model(w, num_layers=L, bn=bn, att=[w["Wa%d" % l] for l in range(1, L + 1)] if "Wa1" in w else None, head=w["head"])


def _node_setup(seed, L, bn, att, hid, emb, d, C, widths, N=48, m=2):
    import networkx as nx
    rng = np.random.default_rng(seed)
    rowptr, col = O.csr_from_edges(N, np.array(nx.barabasi_albert_graph(N, m, seed=seed).edges(), dtype=np.int64))
    A = O.dense_from_csr(rowptr, col)
    feat = rng.normal(size=(N, d)).astype(np.float32)
    label = rng.integers(0, C, N).astype(np.int32)
    w = head_model(rng, d, hid, emb, C, L, widths, att)
    pred = O.model_pred(A, feat, w, bn=bn)
    pred_label = np.argmax(pred, 1).astype(np.int32)
    eng = gnnx.Engine(0)
    _set(eng, w, L, bn)
    eng.set_graph_csr(rowptr, col, feat, label, pred_label)
    return types.SimpleNamespace(rowptr=rowptr, col=col, A=A, feat=feat, label=label, w=w, pred=pred, pred_label=pred_label, eng=eng,
                                 L=L, bn=bn, d=d)


def _graph_setup(seed, L, bn, att, hid, emb, d, C, widths):
    rng = np.random.default_rng(seed)
    adj = GG["adj"]
    feat = (rng.normal(size=adj.shape[:2] + (d,)) * (adj.sum(2, keepdims=True) > 0)).astype(np.float32)
    label = np.asarray(GG["label"]) % C
    w = head_model(rng, d, hid, emb, C, L, widths, att)
    eng = gnnx.Engine(0)
    _set(eng, w, L, bn)
    eng.set_graph_batch(adj, feat, label)
    return adj, feat, label, w, eng


def _sub(s, node):
    idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(s.rowptr, s.col, s.feat, s.label, node, s.L)
    return O.dense_from_csr(srp, scol), sfeat, slabel[idx], s.pred_label[nbrs], idx


def _check(got, fm, port_args, port_kw):
    """Edge mask within max(1e-4, 3 x the port's fp32 / fp64 distance); feature mask likewise."""
    p32, f32 = O.explain_dense_torch(*port_args, return_feat=True, **port_kw)
    p64, f64 = O.explain_dense_torch(*port_args, return_feat=True, dtype=torch.float64, **port_kw)
    tol = max(1e-4, 3 * O.rel_l2(p64, p32))
    err = O.rel_l2(got, p32)
    assert err <= tol, ("edge mask", err, tol)
    if fm is not None:
        ftol = max(1e-4, 3 * float(np.abs(f64 - f32).max()))
        ferr = float(np.abs(fm - f32).max())
        assert ferr <= ftol, ("feature mask", ferr, ftol)


# seed, L, bn, att, hid, emb, d, C, head widths, opt, scheduler.  Heads: widths 1 / 7 / 50 / 256, 1 .. 4 hidden layers; the small ones
# (C (PD + 1) + .. <= 2048 words) staged in shared memory, the others read through L2.  d = 300: the wide path; 200 wide: the row-block path.
CASES = [
    (1, 3, False, False, 20, 20, 10, 4, [50], "adam", "none"),
    (2, 2, True, False, 64, 64, 16, 2, [7, 1], "sgd", "step"),
    (3, 5, False, False, 20, 20, 12, 40, [256, 50, 7], "rmsprop", "cos"),
    (4, 7, True, False, 20, 20, 14, 3, [7], "adagrad", "none"),
    (5, 3, False, True, 20, 20, 8, 3, [20], "adam", "none"),
    (6, 3, False, False, 40, 40, 300, 3, [50], "adam", "step"),
    (7, 3, True, False, 200, 200, 10, 5, [256, 256, 7, 50], "adam", "cos"),
    (8, 2, False, False, 64, 64, 20, 2, [1], "sgd", "none"),
]


def _case_id(c):
    return "s%d_L%d%s%s_h%d_d%d_C%d_head%s_%s_%s" % (c[0], c[1], "_bn" if c[2] else "", "_att" if c[3] else "", c[4], c[6], c[7],
                                                    "-".join(map(str, c[8])), c[9], c[10])


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_head_nodes_match_port(case):
    seed, L, bn, att, hid, emb, d, C, widths, opt, sched = case
    s = _node_setup(seed, L, bn, att, hid, emb, d, C, widths)
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


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_head_graphs_match_port(case):
    seed, L, bn, att, hid, emb, d, C, widths, opt, sched = case
    adj, feat, label, w, eng = _graph_setup(seed + 20, L, bn, att, hid, emb, d, C, widths)
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
        _check(Dm, fm[t], (np.asarray(adj[g], np.float64), feat[g], int(label[g]), None, 0, w, dense[g]),
               dict(hp=_ohp(E, opt, sched), bn=bn, graph_mode=True))


@pytest.mark.parametrize("graph", [False, True], ids=["nodes", "graphs"])
def test_head_one_update_matches_fp64_port(graph):
    """num_epochs = 2: one update; edge and feature masks within 1e-5 of the fp64 port."""
    hp = O.default_hparams(num_epochs=2)
    if not graph:
        s = _node_setup(31, 4, True, False, 20, 20, 16, 4, [50, 7])
        nodes = list(range(0, 48, 5))
        plan = s.eng.plan_nodes(nodes, 4)
        m0, dense = _m0(plan, 70)
        out = np.zeros(plan.total_edges, np.float32)
        fm = np.zeros((plan.count, 16), np.float32)
        s.eng.explain_nodes_host(s.eng.make_hparams(num_epochs=2), m0, out, fm)
        s.eng.close()
        for t, node in enumerate(nodes):
            A, X, gt, pl, idx = _sub(s, node)
            ref, f1 = O.explain_dense_torch(A, X, gt, pl, idx, s.w, dense[t], hp, bn=True, dtype=torch.float64, return_feat=True)
            assert O.rel_l2(plan.dense_of(t, out), ref) <= 1e-5, node
            assert np.abs(fm[t] - f1).max() <= 1e-5, node
        return
    adj, feat, label, w, eng = _graph_setup(41, 4, True, False, 20, 20, 16, 3, [50, 7])
    gids = list(range(12))
    n = adj.shape[1]
    dense = {g: O.draw_m0(n, seed=900 + g) for g in gids}
    rc = {g: eng.graph_rows_cols(g) for g in gids}
    edge_off = eng.plan_graphs(gids)
    out = np.zeros(int(edge_off[-1]), np.float32)
    fm = np.zeros((len(gids), 16), np.float32)
    eng.explain_graphs_host(eng.make_hparams(num_epochs=2), np.concatenate([dense[g][rc[g]] for g in gids]).astype(np.float32), out, fm)
    eng.close()
    for t, g in enumerate(gids):
        ref, f1 = O.explain_dense_torch(np.asarray(adj[g], np.float64), feat[g], int(label[g]), None, 0, w, dense[g], hp, graph_mode=True,
                                        bn=True, dtype=torch.float64, return_feat=True)
        assert O.rel_l2(out[edge_off[t]:edge_off[t + 1]], ref[rc[g]]) <= 1e-5, g
        assert np.abs(fm[t] - f1).max() <= 1e-5, g


@pytest.mark.parametrize("widths", [[50], [8]], ids=["head50_l2", "head8_smem"])
def test_head_unconstrained_matches_port(widths):
    """unconstrained=True (explain_dense.cu) with a head, node and graph mode, against the port: a head block read through L2 ([50]) and
    one staged in shared memory ([8] on PD = 60: 8 x 61 + 3 x 9 = 515 words <= GX_WP_SMEM_MAX)."""
    E = 10
    s = _node_setup(51, 3, True, False, 20, 20, 10, 3, widths)
    nodes = [3, 20]
    plan = s.eng.plan_nodes(nodes, 3)
    m0 = [O.draw_m0(plan.n(t), seed=40 + t) for t in range(plan.count)]
    out = np.zeros(plan.total_edges, np.float32)
    s.eng.explain_nodes_unconstrained(s.eng.make_hparams(num_epochs=E), np.concatenate([M.reshape(-1) for M in m0]).astype(np.float32), out)
    s.eng.close()
    for t, v in enumerate(nodes):
        A, X, gt, pl, idx = _sub(s, v)
        _check(plan.dense_of(t, out), None, (A, X, gt, pl, idx, s.w, m0[t]), dict(hp=O.default_hparams(num_epochs=E), bn=True, unconstrained=True))
    adj, feat, label, w, eng = _graph_setup(52, 4, False, False, 24, 16, 10, 2, [32, 16] if widths == [50] else widths)
    gids = [2, 7]
    n = adj.shape[1]
    m0 = [O.draw_m0(n, seed=60 + g) for g in gids]
    rc = {g: eng.graph_rows_cols(g) for g in gids}
    edge_off = eng.plan_graphs(gids)
    out = np.zeros(int(edge_off[-1]), np.float32)
    eng.explain_graphs_unconstrained(eng.make_hparams(num_epochs=E), np.concatenate([M.reshape(-1) for M in m0]).astype(np.float32), out)
    eng.close()
    for t, g in enumerate(gids):
        Dm = np.zeros((n, n))
        Dm[rc[g]] = out[edge_off[t]:edge_off[t + 1]]
        _check(Dm, None, (np.asarray(adj[g], np.float64), feat[g], int(label[g]), None, 0, w, m0[t]),
               dict(hp=O.default_hparams(num_epochs=E), graph_mode=True, unconstrained=True))


@pytest.mark.parametrize("L,bn,att,hid,emb,d,widths", [(3, False, False, 20, 20, 10, [50]), (7, True, False, 256, 256, 12, [256]),
                                                        (3, False, True, 20, 20, 8, [20, 7]), (2, True, False, 64, 48, 300, [1, 7, 50, 256])])
def test_head_model_forward_matches_port(L, bn, att, hid, emb, d, widths):
    """gx_model_forward of a head model: the head's logits for all N nodes."""
    s = _node_setup(70 + L, L, bn, att, hid, emb, d, 4, widths, N=300, m=3)
    got = s.eng.model_forward()
    s.eng.close()
    assert np.abs(got - s.pred).max() <= 2e-5 * max(1.0, np.abs(s.pred).max())


def test_head_large_subgraph_deterministic_and_order_free():
    """A hub whose 4-hop set has more than 1500 nodes, against the port; then Philox-initialised reruns are bit-identical, whatever
    the order of the batch."""
    s = _node_setup(81, 4, True, False, 20, 20, 12, 3, [50], N=2000, m=2)
    hub = int(np.argmax(np.diff(s.rowptr)))
    plan = s.eng.plan_nodes([hub], 4)
    assert plan.n(0) > 1500
    m0, dense = _m0(plan, 9)
    out = np.zeros(plan.total_edges, np.float32)
    fm = np.zeros((1, 12), np.float32)
    s.eng.explain_nodes_host(s.eng.make_hparams(num_epochs=5), m0, out, fm)
    A, X, gt, pl, idx = _sub(s, hub)
    _check(plan.dense_of(0, out), fm[0], (A, X, gt, pl, idx, s.w, dense[0]), dict(hp=O.default_hparams(num_epochs=5), bn=True))
    nodes = [3, 17, hub, 120, 999]
    hp = s.eng.make_hparams(num_epochs=30, init=_abi.GX_INIT_PHILOX, seed=5)
    res = {}
    for order in (nodes, nodes[::-1], nodes):
        plan = s.eng.plan_nodes(order, 4)
        out = np.zeros(plan.total_edges, np.float32)
        fm = np.zeros((plan.count, 12), np.float32)
        s.eng.explain_nodes_host(hp, None, out, fm)
        for t, node in enumerate(order):
            got = np.concatenate([out[plan.edge_off[t]:plan.edge_off[t + 1]], fm[t]])
            if node in res:
                assert np.array_equal(res[node], got), node
            res[node] = got
    s.eng.close()
    adj, feat, label, w, eng = _graph_setup(82, 3, False, False, 20, 20, 14, 3, [256, 7])
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


def test_head_refusals():
    s = _node_setup(61, 3, False, False, 20, 20, 10, 3, [50])
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
                                            state_in=dict(m=np.zeros(te, np.float32), v=np.zeros(te, np.float32)))]
    for call in calls:
        with pytest.raises(_abi.GnnxError) as e:
            call()
        assert e.value.status == GX_ERR_UNSUPPORTED
    w = s.w
    wide = dict(w, head=[(np.zeros((257, 60), np.float32), np.zeros(257, np.float32))], Wp=np.zeros((3, 257), np.float32))
    with pytest.raises(_abi.GnnxError) as e:
        _set(s.eng, wide, 3, False)
    assert e.value.status == GX_ERR_UNSUPPORTED and "GX_MAX_WIDTH" in str(e.value), str(e.value)
    # the C entry point itself, past GX_MAX_HEAD_LAYERS (Engine.set_model refuses before calling it)
    import ctypes as C
    lib = _abi.lib()
    dims = _abi.GxModelDims(10, 20, 20, 3, 3, 0)
    Ws = [np.ascontiguousarray(w["W%d" % l]) for l in (1, 2, 3)]
    wp = (C.c_void_p * 3)(*[x.ctypes.data for x in Ws])
    k = _abi.GX_MAX_HEAD_LAYERS + 1
    widths = np.full(k, 4, np.int32)
    hw = [np.zeros((4, 60), np.float32)] + [np.zeros((4, 4), np.float32)] * (k - 1) + [np.zeros((3, 4), np.float32)]
    hb = [np.zeros(4, np.float32)] * k + [np.zeros(3, np.float32)]
    rc = lib.gx_set_model_head(s.eng._h, C.byref(dims), wp, None, None, k, widths.ctypes.data_as(C.POINTER(C.c_int32)),
                               (C.c_void_p * (k + 1))(*[x.ctypes.data for x in hw]), (C.c_void_p * (k + 1))(*[x.ctypes.data for x in hb]))
    assert rc == GX_ERR_UNSUPPORTED
    assert "GX_MAX_HEAD_LAYERS" in lib.gx_last_error().decode()
    with pytest.raises(NotImplementedError, match="hidden layers"):
        _set(s.eng, dict(w, head=[(np.zeros((4, 60), np.float32), np.zeros(4, np.float32))] + [(np.zeros((4, 4), np.float32),
                                                                                                np.zeros(4, np.float32))] * (k - 1),
                         Wp=np.zeros((3, 4), np.float32)), 3, False)
    s.eng.close()


def _explainer(tmp_path, graph_mode, print_training):
    """The drop-in Explainer on a gnnx.models model with pred_hidden_dims=[50] (torch's init), node or graph mode, pred computed on the
    device."""
    args = types.SimpleNamespace(num_gc_layers=3, num_epochs=20, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                 mask_bias=False, gpu=False, bias=True, bn=True, method="base", dataset="graphs" if graph_mode else "syn1",
                                 bmname=None, hidden_dim=20, output_dim=20, name_suffix="", explainer_suffix="", logdir=str(tmp_path))
    torch.manual_seed(3)
    if graph_mode:
        adj, feat = GG["adj"], GG["feat"].astype(np.float32)
        label = np.asarray(GG["label"]) % 2
        model = gnnx.models.GcnEncoderGraph(feat.shape[2], 20, 20, 2, 3, pred_hidden_dims=[50], bn=True, args=args)
        return gnnx.Explainer(model=model, adj=torch.tensor(adj, dtype=torch.float), feat=torch.tensor(feat), label=torch.tensor(label),
                              pred=None, train_idx=[], args=args, writer=None, print_training=print_training, graph_mode=True, graph_idx=0)
    s = _node_setup(91, 3, True, False, 20, 20, 10, 4, [50])
    s.eng.close()
    model = gnnx.models.GcnEncoderNode(10, 20, 20, 4, 3, pred_hidden_dims=[50], bn=True, args=args)
    return gnnx.Explainer(model=model, adj=torch.tensor(s.A[None], dtype=torch.float), feat=torch.tensor(s.feat[None]),
                          label=torch.tensor(s.label[None]), pred=None, train_idx=[], args=args, writer=None, print_training=print_training,
                          graph_mode=False, graph_idx=0)


@pytest.mark.parametrize("graph_mode", [False, True], ids=["nodes", "graphs"])
def test_head_drop_in_explainer(tmp_path, capsys, graph_mode):
    """A notice with print_training, the masks and .npy files of a silent run, model='grad' refused before any RNG is drawn."""
    quiet = _explainer(tmp_path / "quiet", graph_mode, False)
    loud = _explainer(tmp_path / "loud", graph_mode, True)
    capsys.readouterr()
    got = []
    for ex in (quiet, loud):
        torch.manual_seed(4)
        got.append(ex.explain(0, graph_idx=3, graph_mode=True) if graph_mode else ex.explain(7, graph_idx=0))
    assert "trace is not built for models with an MLP prediction head" in capsys.readouterr().out
    assert np.array_equal(got[0], got[1])
    fa = sorted(p.name for p in (tmp_path / "quiet").glob("*.npy"))
    fb = sorted(p.name for p in (tmp_path / "loud").glob("*.npy"))
    assert fa == fb and fa
    for f in fa:
        assert np.array_equal(np.load(tmp_path / "quiet" / f), np.load(tmp_path / "loud" / f))
    if not graph_mode:
        state = torch.get_rng_state()
        with pytest.raises(NotImplementedError, match="MLP prediction head"):
            loud.explain(7, graph_idx=0, model="grad")
        assert torch.equal(torch.get_rng_state(), state)


def test_head_sharded_explain_matches_explain_nodes(tmp_path):
    """gnnx.dist on a head model (one rank, gloo, the torch all-gather): the packed masks of explain_nodes_sharded equal
    Explainer.explain_nodes under the same torch seed."""
    import socket
    import torch.distributed as dist
    from gnnx import dist as gdist
    ex = _explainer(tmp_path, False, False)
    args = ex.args
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
    for t, (node, Dn) in enumerate(zip(nodes, dense)):
        _, sub_adj, _, _, _ = ex.extract_neighborhood(node, 0)
        ei, ej = np.nonzero(sub_adj)
        assert np.array_equal(values[offsets[t]:offsets[t + 1]], Dn[ei, ej].astype(np.float32)), node


# ---------------------------------------------------------------------------------------------------------- the unmodified reference
def _golden_engine(case):
    w, L, bn = case_weights(case), int(GOLDEN[case + "_L"]), bool(GOLDEN[case + "_bn"])
    eng = gnnx.Engine(0)
    _set(eng, w, L, bn)
    return eng, L


@pytest.mark.parametrize("case", golden_cases(0))
def test_head_matches_reference_nodes(case):
    """Every node of tests/golden/head_golden.npz within max(1e-4, 3 x the reference's own spread)."""
    eng, L = _golden_engine(case)
    fx, feat = case_feat(case)
    eng.set_graph_csr(fx.rowptr, fx.col, feat, fx.label, np.argmax(GOLDEN[case + "_pred"], 1).astype(np.int32))
    nodes = [int(v) for v in GOLDEN[case + "_nodes"]]
    plan = eng.plan_nodes(nodes, L)
    hp = _hp(eng, int(GOLDEN[case + "_epochs"]), str(GOLDEN[case + "_opt"]))
    out = np.zeros(plan.total_edges, np.float32)
    if int(GOLDEN[case + "_unc"]):
        m0 = [O.draw_m0(plan.n(t), seed=int(GOLDEN["%s_n%d_seed" % (case, v)])).reshape(-1) for t, v in enumerate(nodes)]
        eng.explain_nodes_unconstrained(hp, np.concatenate(m0).astype(np.float32), out)
    else:
        m0 = np.empty(plan.total_edges, np.float32)
        for t, node in enumerate(nodes):
            r, c = plan.rows_cols_of(t)
            m0[plan.edge_off[t]:plan.edge_off[t + 1]] = O.draw_m0(plan.n(t), seed=int(GOLDEN["%s_n%d_seed" % (case, node)]))[r, c]
        eng.explain_nodes_host(hp, m0, out)
    eng.close()
    for t, node in enumerate(nodes):
        key = "%s_n%d" % (case, node)
        assert np.array_equal(plan.neighbors_of(t), GOLDEN[key + "_nbrs"])
        got = out[plan.edge_off[t]:plan.edge_off[t + 1]]
        assert O.rel_l2(got, GOLDEN[key + "_mask"]) <= max(1e-4, 3 * float(GOLDEN[key + "_spread"])), key


@pytest.mark.parametrize("case", golden_cases(1))
def test_head_matches_reference_graphs(case):
    eng, L = _golden_engine(case)
    eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
    G = int(GG["num_graphs"])
    n = int(GG["max_nodes"])
    gids = list(range(G))
    rc = {g: eng.graph_rows_cols(g) for g in gids}
    edge_off = eng.plan_graphs(gids)
    hp = _hp(eng, int(GOLDEN[case + "_epochs"]), str(GOLDEN[case + "_opt"]))
    out = np.zeros(int(edge_off[-1]), np.float32)
    dense = [O.draw_m0(n, seed=int(GG["g%d_seed" % g])) for g in gids]
    if int(GOLDEN[case + "_unc"]):
        eng.explain_graphs_unconstrained(hp, np.concatenate([M.reshape(-1) for M in dense]).astype(np.float32), out)
    else:
        eng.explain_graphs_host(hp, np.concatenate([dense[g][rc[g]] for g in gids]).astype(np.float32), out)
    eng.close()
    for t, g in enumerate(gids):
        key = "%s_g%d" % (case, g)
        ei, ej = np.nonzero(GG["adj"][g])
        assert np.array_equal(rc[g][0], ei) and np.array_equal(rc[g][1], ej)
        assert O.rel_l2(out[edge_off[t]:edge_off[t + 1]], GOLDEN[key + "_mask"]) <= max(1e-4, 3 * float(GOLDEN[key + "_spread"])), key


@pytest.mark.parametrize("case", golden_cases(0))
def test_head_model_forward_matches_reference_pred(case):
    """gx_model_forward on the rand graph reproduces the reference model's pred within 2e-5."""
    eng, L = _golden_engine(case)
    fx, feat = case_feat(case)
    eng.set_graph_csr(fx.rowptr, fx.col, feat, fx.label, np.zeros(len(fx.label), np.int32))
    got = eng.model_forward()
    eng.close()
    want = GOLDEN[case + "_pred"]
    assert np.abs(got - want).max() <= 2e-5 * max(1.0, np.abs(want).max())
