"""GPU (-m gpu): one engine handle across many calls, and the engine on streams other than the legacy default stream.

Plan lifetime (a table): every call that can change a plan's inputs or buffers, then every consumer of the node and the graph plan.  The
consumers are probed with an argument the library refuses after its plan check and before any device work (num_epochs = 0,
threshold_num = 0): "no plan" means the plan was dropped, the argument's own message that it was kept.  A call that keeps the plan
also runs the real consumer, bit-identical to a fresh handle.

One session: ~25 steps on one engine, large batches, then small ones, then large ones again, so that workspaces grown by an earlier step
hold stale, larger contents: node and graph mode, every kernel family and debug knob, each step bit-identical to the same step on a
fresh engine and the first, last and variant steps against the reference goldens.

Streams: the engine on a torch stream behind a queued sleep and an asynchronous copy (gx_set_stream), the drop-in (Explainer, gnnx.dist)
under `with torch.cuda.stream(side)`, and Engine.densify_device after plan_nodes(fetch=False)."""
import ctypes as C
import socket
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist

import gnnx
import gnnx_oracle as O
import util
from gnnx import _abi
from gnnx import dist as gdist
from test_gpu_wide import _node_setup, random_model
from test_oracle_att import random_att_model

pytestmark = pytest.mark.gpu
GX_ERR_INVALID = -1
GIDS = [0, 3, 5, 9, 11]
EPOCHS = 20


@pytest.fixture(scope="module")
def syn1():
    return util.load_fixture("syn1")


@pytest.fixture(scope="module")
def gg():
    return np.load(util.GOLDEN + "/graphs_golden.npz")


def _m0(plan, fx=None, seed=0):
    """M0 at the plan's edge slots: the golden draw of a node that has one, a seeded N(1, 2/n) draw otherwise."""
    m0 = np.empty(plan.total_edges, np.float32)
    for t, node in enumerate(plan.nodes):
        key = "n%d_m0" % node
        if fx is not None and key in fx.gold.files:
            m0[plan.edge_off[t]:plan.edge_off[t + 1]] = fx.gold[key]
        else:
            r, c = plan.rows_cols_of(t)
            m0[plan.edge_off[t]:plan.edge_off[t + 1]] = O.draw_m0(plan.n(t), seed=seed + int(node))[r, c]
    return m0


def _graph_m0(eng, gids, seed=0):
    """Seeded (max_nodes, max_nodes) draws of the listed graphs: (edge-slot M0 in plan order, the dense draws concatenated)."""
    n = eng.batch_n
    dense = [O.draw_m0(n, seed=seed + int(g)) for g in gids]
    return (np.concatenate([D[eng.graph_rows_cols(int(g))] for D, g in zip(dense, gids)]).astype(np.float32),
            np.concatenate([D.reshape(-1) for D in dense]).astype(np.float32))


def _same(a, b, what=""):
    """Bit-identical results: tuples / lists / dicts of arrays or tensors, NaN where NaN."""
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for k in a:
            _same(a[k], b[k], "%s.%s" % (what, k))
    elif isinstance(a, (tuple, list)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, "%s[%d]" % (what, i))
    else:
        x = a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
        y = b.cpu().numpy() if torch.is_tensor(b) else np.asarray(b)
        assert x.dtype == y.dtype and x.shape == y.shape, (what, x.dtype, y.dtype, x.shape, y.shape)
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), what


def _batch(fx, gg):
    """The graphs fixture's adjacency with syn1-wide (d = 10) features and labels below syn1's class count: one model serves both modes."""
    rng = np.random.default_rng(2)
    adj = gg["adj"]
    feat = (rng.normal(size=adj.shape[:2] + (fx.feat.shape[1],)) * (adj.sum(2, keepdims=True) > 0)).astype(np.float32)
    return adj, feat, np.asarray(gg["label"]) % fx.weights["Wp"].shape[0]


# ------------------------------------------------------------------------------------------------ a. plan lifetime
def _probe(eng, graph):
    """{consumer: True (the plan is still accepted) / False ("no plan")} without launching anything on a stale plan."""
    lib, h = eng._lib, eng._h
    hp0 = eng.make_hparams(num_epochs=0)
    f = np.zeros(1 << 20, np.float32)
    d = np.zeros(1 << 20, np.float64)
    i = np.zeros(1 << 20, np.int32)
    p = lambda a: a.ctypes.data
    io = _abi.GxExplainIo()
    io.m0_edges = p(f); io.edge_mask = p(f)
    if graph:
        refused = {
            "explain_graphs": lambda: lib.gx_explain_graphs(h, C.byref(hp0), _abi.GX_HOST, p(f), p(f), None),
            "explain_graphs_ex": lambda: lib.gx_explain_graphs_ex(h, C.byref(hp0), _abi.GX_HOST, C.byref(io)),
            "explain_graphs_unconstrained": lambda: lib.gx_explain_graphs_unconstrained(h, C.byref(hp0), _abi.GX_HOST, p(f), p(f), None, None, None),
            "offedge_regularisers_graphs": lambda: lib.gx_offedge_regularisers_graphs(h, C.byref(hp0), _abi.GX_HOST, p(f), p(d)),
        }
        real = {}
    else:
        refused = {
            "explain_nodes": lambda: lib.gx_explain_nodes(h, C.byref(hp0), _abi.GX_HOST, p(f), p(f), None),
            "explain_nodes_ex": lambda: lib.gx_explain_nodes_ex(h, C.byref(hp0), _abi.GX_HOST, C.byref(io)),
            "explain_nodes_unconstrained": lambda: lib.gx_explain_nodes_unconstrained(h, C.byref(hp0), _abi.GX_HOST, p(f), p(f), None, None, None),
            "offedge_regularisers": lambda: lib.gx_offedge_regularisers(h, C.byref(hp0), _abi.GX_HOST, p(f), p(d)),
            "denoise_topk": lambda: lib.gx_denoise_topk(h, _abi.GX_HOST, p(f), 0, 4, p(f), p(i), p(i), p(f)),
            "denoise_topk_edges": lambda: lib.gx_denoise_topk_edges(h, _abi.GX_HOST, p(f), 0, 4, p(f), p(i), p(i), p(f)),
        }
        # no argument refused after the plan check: the real call, safe either way (host state only, or a node plan, whose
        # invalidation the refused probes above already cover)
        real = {
            "plan_fetch": lambda: lib.gx_plan_fetch(h, p(np.zeros(eng._plan_sizes[0] + 1, np.int64)), None, None, None, None, None),
            "plan_class_counts": lambda: lib.gx_plan_class_counts(h, p(i), p(i), p(i)),
            "grad_nodes": lambda: lib.gx_grad_nodes(h, _abi.GX_HOST, p(f)),
            "densify": lambda: lib.gx_densify(h, _abi.GX_HOST, p(f), p(d)),
        }
    out = {}
    for name, call in list(refused.items()) + list(real.items()):
        rc = call()
        msg = lib.gx_last_error().decode()
        if rc != _abi.GX_OK and "no plan" in msg:
            out[name] = False
            continue
        if name in refused:
            assert rc == GX_ERR_INVALID and ("num_epochs" in msg or "threshold_num" in msg), (name, rc, msg)
        else:
            assert rc == _abi.GX_OK, (name, rc, msg)
        out[name] = True
    return out


def _table_setup(fx, batch, graph):
    eng = util.make_engine(fx)
    eng.set_graph_batch(*batch)
    plan = eng.plan_graphs(GIDS) if graph else eng.plan_nodes(fx.nodes[:6], 3)
    return eng, plan


def _consume(eng, fx, plan, graph):
    """The real consumer: the planned batch explained (EPOCHS epochs), with its feature masks."""
    hp = eng.make_hparams(num_epochs=EPOCHS)
    if graph:
        m0, _ = _graph_m0(eng, GIDS, seed=40)
        out = np.zeros(int(plan[-1]), np.float32)
        fm = np.zeros((len(GIDS), fx.feat.shape[1]), np.float32)
        eng.explain_graphs_host(hp, m0, out, fm)
    else:
        out = np.zeros(plan.total_edges, np.float32)
        fm = np.zeros((plan.count, fx.feat.shape[1]), np.float32)
        eng.explain_nodes_host(hp, _m0(plan, fx), out, fm)
    return out, fm


def _att_weights(fx):
    w = random_att_model(np.random.default_rng(5), fx.feat.shape[1], 20, 20, fx.weights["Wp"].shape[0], 3)
    return w, [w["Wa%d" % l] for l in (1, 2, 3)]


def _head_weights(fx):
    rng = np.random.default_rng(6)
    C = fx.weights["Wp"].shape[0]
    head = [((rng.normal(size=(16, 60)) * 0.2).astype(np.float32), (rng.normal(size=16) * 0.3).astype(np.float32))]
    return dict(fx.weights, Wp=(rng.normal(size=(C, 16)) * 0.3).astype(np.float32)), head


# name -> (the call, keeps a node plan, keeps a graph plan)
MUTATORS = {
    "set_model": (lambda e, fx, b: e.set_model(fx.weights), False, False),
    "set_model_variant": (lambda e, fx, b: e.set_model(fx.weights, bn=True), False, False),
    "set_model_att": (lambda e, fx, b: e.set_model(_att_weights(fx)[0], att=_att_weights(fx)[1]), False, False),
    "set_model_head": (lambda e, fx, b: e.set_model(_head_weights(fx)[0], head=_head_weights(fx)[1]), False, False),
    "set_graph_csr": (lambda e, fx, b: e.set_graph_csr(fx.rowptr, fx.col, fx.feat, fx.label, fx.pred_label), False, True),
    "set_graph_batch_csr": (lambda e, fx, b: e.set_graph_batch(*b), True, False),
    "count_nodes": (lambda e, fx, b: e.count_nodes(fx.nodes[:40], 3), False, False),
    "plan_nodes": (lambda e, fx, b: e.plan_nodes(fx.nodes[:6], 3), True, False),
    "plan_graphs": (lambda e, fx, b: e.plan_graphs(GIDS), False, True),
    "debug_set_cluster": (lambda e, fx, b: e.debug_cluster(1, 0), False, True),
    "debug_force_stream": (lambda e, fx, b: e.debug_force_stream(False), False, True),
    "model_forward": (lambda e, fx, b: e.model_forward(), True, True),
    "neighborhood_rows": (lambda e, fx, b: e.neighborhood_rows(fx.nodes[:40], 3), True, True),
    "count_graphs": (lambda e, fx, b: e.count_graphs(list(range(12))), True, True),
    "densify_graphs": (lambda e, fx, b: e.densify_graphs_host(GIDS, np.ones(int(e.count_graphs(GIDS)[1].sum()), np.float32)), True, True),
    "set_stream": (lambda e, fx, b: e.set_stream(torch.cuda.current_stream().cuda_stream), True, True),
    "debug_set_gang": (lambda e, fx, b: e.debug_gang(0), True, True),
    "debug_ieee_edge": (lambda e, fx, b: e.debug_ieee_edge(False), True, True),
    "explain": (None, True, True),     # the mode's own explain call, run twice
}


@pytest.fixture(scope="module")
def fresh_consumers(syn1, gg):
    res = {}
    for graph in (False, True):
        eng, plan = _table_setup(syn1, _batch(syn1, gg), graph)
        try:
            res[graph] = _consume(eng, syn1, plan, graph)
        finally:
            eng.close()
    return res


@pytest.mark.parametrize("graph", [False, True], ids=["node_plan", "graph_plan"])
@pytest.mark.parametrize("mutator", list(MUTATORS))
def test_plan_lifetime(syn1, gg, fresh_consumers, mutator, graph):
    call, keeps_node, keeps_graph = MUTATORS[mutator]
    keeps = keeps_graph if graph else keeps_node
    batch = _batch(syn1, gg)
    eng, plan = _table_setup(syn1, batch, graph)
    try:
        assert all(_probe(eng, graph).values())
        if call is None:
            _consume(eng, syn1, plan, graph)
        else:
            call(eng, syn1, batch)
        got = _probe(eng, graph)
        assert got == {k: keeps for k in got}, (mutator, got)
        if keeps:
            _same(_consume(eng, syn1, plan, graph), fresh_consumers[graph], mutator)
    finally:
        eng.close()


def test_graph_plan_of_another_model_is_dropped(syn1, gg):
    """A graph plan made under a variant model (no shared-memory footprints) must not reach the tuned kernel after gx_set_model, nor a
    plan of one input width a model of another width; planning again checks the width."""
    eng = util.make_engine(syn1)
    try:
        eng.set_graph_batch(*_batch(syn1, gg))
        eng.set_model(syn1.weights, bn=True)
        eng.plan_graphs(GIDS)
        assert all(_probe(eng, True).values())
        eng.set_model(syn1.weights)
        assert not any(_probe(eng, True).values())
        eng.plan_graphs(GIDS)
        eng.set_model(random_model(np.random.default_rng(1), 14, 20, 20, 4, 3))
        assert not any(_probe(eng, True).values())
        with pytest.raises(_abi.GnnxError, match="feat_dim"):
            eng.plan_graphs(GIDS)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ b. one session
def _explain(eng, nodes, L=3, epochs=EPOCHS, fx=None, feat=True, **hp_over):
    plan = eng.plan_nodes(nodes, L)
    hp = eng.make_hparams(num_epochs=epochs, **hp_over)
    out = np.zeros(plan.total_edges, np.float32)
    fm = np.zeros((plan.count, eng.input_dim), np.float32) if feat else None
    eng.explain_nodes_host(hp, _m0(plan, fx, seed=7), out, fm)
    return (out, fm) if feat else (out,)


def _session_steps(fx, fx4, gg, var):
    """[(name, setup(eng), run(eng) -> results)]: setup is what the step needs on a fresh engine, applied on the session engine too (it
    replaces the model / graph / knobs of the step before; plans are made by run)."""
    all_nodes = list(range(fx.N))
    syn1 = lambda e: (e.set_model(fx.weights), e.set_graph_csr(fx.rowptr, fx.col, fx.feat, fx.label, fx.pred_label))
    syn4 = lambda e: (e.set_model(fx4.weights), e.set_graph_csr(fx4.rowptr, fx4.col, fx4.feat, fx4.label, fx4.pred_label))
    rng = np.random.default_rng(9)
    d, C = fx.feat.shape[1], fx.weights["Wp"].shape[0]
    pad32 = random_model(rng, d, 24, 24, C, 3)
    bn4 = random_model(rng, d, 20, 20, C, 4)
    att_w, att = _att_weights(fx)
    head_w, head = _head_weights(fx)
    w256 = random_model(rng, d, 256, 256, C, 3)
    wide = _node_setup(31, 3, False, 20, 20, 300, 3)
    wide.eng.close()
    nodes = fx.nodes[:24]
    mask_of_700 = {}

    def all700(e):
        out, fm = _explain(e, all_nodes, epochs=100, fx=fx)
        mask_of_700.setdefault("mask", out)
        return out, fm

    def trace_state(e):
        plan = e.plan_nodes(all_nodes, 3)
        hp = e.make_hparams(num_epochs=100)
        out = np.zeros(plan.total_edges, np.float32)
        tr = np.zeros((plan.count, 100, _abi.GX_TRACE_COLS), np.float32)
        tp = np.zeros((plan.count, 100, C), np.float32)
        st = {k: np.zeros(plan.total_edges, np.float32) for k in ("M", "m", "v")}
        st["feat"] = np.zeros((plan.count, 3, d), np.float32)
        e.explain_nodes_ex(hp, _m0(plan, fx, seed=7), out, trace=tr, trace_pred=tp, state_out=st)
        return out, tr, tp, st

    def grad_post(e):
        plan = e.plan_nodes(all_nodes, 3)
        g = np.zeros(plan.total_edges, np.float32)
        e.grad_nodes_host(g)
        mask = mask_of_700["mask"]
        total = int(np.sum(np.diff(plan.node_off) ** 2))
        return (g,) + e.denoise_topk(mask, 20) + e.denoise_topk_edges(mask, 20) + (e.densify_host(mask, total),)

    def forward_rows_count(e):
        return (e.model_forward(), e.neighborhood_rows(nodes, 3)) + e.count_nodes(all_nodes, 3)

    def unconstrained(e):
        plan = e.plan_nodes(fx.nodes[:12], 3)
        dense = np.concatenate([O.draw_m0(plan.n(t), seed=70 + t).reshape(-1) for t in range(plan.count)]).astype(np.float32)
        out = np.zeros(plan.total_edges, np.float32)
        md = np.zeros(len(dense), np.float32)
        e.explain_nodes_unconstrained(e.make_hparams(num_epochs=EPOCHS), dense, out, md)
        return out, md

    gset = lambda e: (e.set_model({k: gg[k] for k in util.WKEYS}), e.set_graph_batch(gg["adj"], gg["feat"], gg["label"]))
    all_g = list(range(int(gg["num_graphs"])))

    def graphs_tuned(e):
        eo = e.plan_graphs(all_g)
        out = np.zeros(int(eo[-1]), np.float32)
        fm = np.zeros((len(all_g), gg["feat"].shape[2]), np.float32)
        e.explain_graphs_host(e.make_hparams(num_epochs=100), np.concatenate([gg["g%d_m0" % g] for g in all_g]), out, fm)
        return eo, out, fm

    def graphs_trace(e):
        eo = e.plan_graphs(GIDS)
        m0, dense = _graph_m0(e, GIDS, seed=50)
        out = np.zeros(int(eo[-1]), np.float32)
        tr = np.zeros((len(GIDS), 30, _abi.GX_TRACE_COLS), np.float32)
        tp = np.zeros((len(GIDS), 30, 2), np.float32)
        hp = e.make_hparams(num_epochs=30)
        e.explain_nodes_ex(hp, m0, out, trace=tr, trace_pred=tp, graphs=True)
        return out, tr, tp, e.offedge_regularisers_graphs(hp, dense)

    def graphs_unconstrained(e):
        eo = e.plan_graphs(GIDS[::-1])
        _, dense = _graph_m0(e, GIDS[::-1], seed=60)
        out = np.zeros(int(eo[-1]), np.float32)
        md = np.zeros(len(dense), np.float32)
        e.explain_graphs_unconstrained(e.make_hparams(num_epochs=EPOCHS), dense, out, md)
        return out, md

    def graphs_variant(e):
        eo = e.plan_graphs(all_g)
        m0, _ = _graph_m0(e, all_g, seed=80)
        out = np.zeros(int(eo[-1]), np.float32)
        e.explain_graphs_host(e.make_hparams(num_epochs=EPOCHS, opt=_abi.GX_OPT["rmsprop"]), m0, out)
        return (out, e.densify_graphs_host(all_g[::-1], out[::-1].copy())) + e.count_graphs(all_g)

    def variant_golden(e):
        plan = e.plan_nodes(var.nodes, 3)
        m0 = np.concatenate([var.g["bn_n%d_m0" % n] for n in var.nodes]).astype(np.float32)
        out = np.zeros(plan.total_edges, np.float32)
        e.explain_nodes_host(e.make_hparams(num_epochs=var.epochs), m0, out)
        return plan.edge_off, out

    def device_700(e):
        plan = e.plan_nodes(all_nodes, 3, fetch=False)
        ref = gnnx.Engine(e.device)      # the plan's M0 needs the canonical description (a fetched plan of the same nodes)
        try:
            syn1(ref)
            ref_plan = ref.plan_nodes(all_nodes, 3)
            m0 = _m0(ref_plan, fx, seed=7)
            dense_700 = int(np.sum(np.diff(ref_plan.node_off) ** 2))
        finally:
            ref.close()
        mask = e.explain_nodes_device(e.make_hparams(num_epochs=100), torch.from_numpy(m0).cuda())
        assert e._dense_total() == dense_700      # the size densify_device allocates, checked before the library writes into it
        return mask, e.densify_device(mask)

    def setting(model, graph=None, L=3, bn=False, att_=None, head_=None):
        def f(e):
            e.set_model(model, num_layers=L, bn=bn, att=att_, head=head_)
            g = graph or fx
            e.set_graph_csr(g.rowptr, g.col, g.feat, g.label, g.pred_label)
        return f

    def knobbed(gang=None, stream=None, cluster=None):
        def f(e):
            syn1(e)
            if stream is not None:
                e.debug_force_stream(stream)
            if gang is not None:
                e.debug_gang(gang)
            if cluster is not None:
                e.debug_cluster(cluster, 0)
        return f

    off = knobbed(gang=0, stream=False, cluster=1)
    return [
        ("syn1_700", syn1, all700),
        ("syn1_700_trace_state", syn1, trace_state),
        ("syn1_grad_denoise_densify", syn1, grad_post),
        ("syn4_51", syn4, lambda e: _explain(e, fx4.nodes, epochs=100, fx=fx4)),
        ("syn4_one_node", syn4, lambda e: _explain(e, fx4.nodes[7:8], fx=fx4)),
        ("forced_gang", knobbed(gang=3, stream=True), lambda e: _explain(e, nodes, fx=fx)),
        ("knobs_off_1", off, lambda e: _explain(e, nodes[:5], fx=fx)),
        ("forced_stream1", knobbed(gang=-1, stream=True), lambda e: _explain(e, nodes, fx=fx)),
        ("knobs_off_2", off, lambda e: _explain(e, nodes[5:9], fx=fx)),
        ("forced_cluster4", knobbed(cluster=4), lambda e: _explain(e, nodes, fx=fx)),
        ("knobs_off_3", off, lambda e: _explain(e, nodes, fx=fx)),
        ("pad32", setting(pad32), lambda e: _explain(e, nodes, fx=fx)),
        ("bn_L4", setting(bn4, L=4, bn=True), lambda e: _explain(e, nodes[:10], L=4, feat=False)),
        ("rmsprop_default_model", syn1, lambda e: _explain(e, nodes, fx=fx, feat=False, opt=_abi.GX_OPT["rmsprop"])),
        ("attention", setting(att_w, att_=att), lambda e: _explain(e, nodes[:10], fx=fx, feat=False)),
        ("mlp_head", setting(head_w, head_=head), lambda e: _explain(e, nodes[:10], fx=fx, feat=False)),
        ("d300", setting(wide.w, graph=types.SimpleNamespace(rowptr=wide.rowptr, col=wide.col, feat=wide.feat, label=wide.label,
                                                              pred_label=wide.pred_label)), lambda e: _explain(e, [0, 7, 23, 47], feat=False)),
        ("width256", setting(w256), lambda e: _explain(e, nodes[:6], fx=fx, feat=False)),
        ("variant_golden_bn", lambda e: (e.set_model(var.w, bn=True), e.set_graph_csr(var.rowptr, var.col, var.feat, var.label, var.pred_label)),
         variant_golden),
        ("forward_rows_count", syn1, forward_rows_count),
        ("unconstrained_nodes", syn1, unconstrained),
        ("graphs_tuned", gset, graphs_tuned),
        ("graphs_trace_offedge", gset, graphs_trace),
        ("graphs_unconstrained", gset, graphs_unconstrained),
        ("graphs_variant_densify_count", lambda e: (gset(e), e.set_model({k: gg[k] for k in util.WKEYS}, bn=True)), graphs_variant),
        ("syn1_700_device", syn1, device_700),
    ]


def test_one_session_against_fresh_engines(syn1, gg):
    fx4 = util.load_fixture("syn4")
    g = np.load(util.GOLDEN + "/variants_golden.npz")
    rowptr, col = O.csr_from_edges(int(g["N"]), g["edges"])
    var = types.SimpleNamespace(g=g, w={k[3:]: g[k] for k in g.files if k.startswith("bn_W") or k.startswith("bn_b")}, rowptr=rowptr, col=col,
                                feat=g["feat"].astype(np.float32), label=g["label"].astype(np.int32),
                                pred_label=np.argmax(g["bn_pred"], 1).astype(np.int32), nodes=[int(x) for x in g["bn_nodes"]],
                                epochs=int(g["num_epochs"]))
    steps = _session_steps(syn1, fx4, gg, var)
    session = gnnx.Engine(0)
    results = {}
    try:
        for name, setup, run in steps:
            setup(session)
            results[name] = run(session)
            fresh = gnnx.Engine(0)
            try:
                setup(fresh)
                want = run(fresh)
            finally:
                fresh.close()
            _same(results[name], want, name)
    finally:
        session.close()
    # the session never compares two wrong runs: the first and last syn1 steps, the graph step and the variant step against the goldens
    plan_nodes = list(range(syn1.N))
    ref = util.make_engine(syn1)
    try:
        plan = ref.plan_nodes(plan_nodes, 3)
    finally:
        ref.close()
    for key, mask in (("syn1_700", results["syn1_700"][0]), ("syn1_700_device", results["syn1_700_device"][0].cpu().numpy())):
        errs = {n: util.rel_l2(mask[plan.edge_off[n]:plan.edge_off[n + 1]], syn1.gold["n%d_mask" % n]) for n in syn1.nodes}
        util.assert_per_node(errs, "syn1", 100)
    dense = results["syn1_700_device"][1].cpu().numpy()
    offs = np.concatenate([[0], np.cumsum(np.diff(plan.node_off) ** 2)])
    for n in syn1.nodes[:10]:
        assert np.array_equal(dense[offs[n]:offs[n + 1]].reshape(plan.n(n), plan.n(n)), plan.dense_of(n, results["syn1_700"][0]))
    eo, out, fm = results["graphs_tuned"]
    errs = [util.rel_l2(out[eo[t]:eo[t + 1]], gg["g%d_mask_e100" % t]) for t in range(int(gg["num_graphs"]))]
    assert max(errs) <= 1e-4, errs
    w = {k: gg[k] for k in util.WKEYS}
    for t in (1, 9):
        A = gg["adj"][t]
        r, c = np.nonzero(A)
        util.check_graph_masks(A, gg["feat"][t], gg["label"][t], w, _dense_m0(A, gg["g%d_m0" % t]), 100, out[eo[t]:eo[t + 1]], fm[t], (r, c))
    eo, out = results["variant_golden_bn"]
    for t, n in enumerate(var.nodes):
        assert util.rel_l2(out[eo[t]:eo[t + 1]], g["bn_n%d_mask" % n]) <= 1e-4, n


def _dense_m0(A, m0_edges):
    """The golden graph M0 at the adjacency's slots (row-major), zero elsewhere: the oracle only reads the edge entries."""
    D = np.zeros(A.shape, np.float32)
    D[np.nonzero(A)] = m0_edges
    return D


# ------------------------------------------------------------------------------------------------ c. the engine on a caller stream
def test_engine_on_a_caller_stream(syn1, gg):
    """gx_set_stream(s): the library's device-buffer calls are ordered behind a sleep and an asynchronous M0 copy queued on s, and
    return the GX_HOST results of a fresh engine on the default stream, bit for bit; then set_stream(0) on the same handle."""
    nodes = syn1.nodes[:40]
    gw = {k: gg[k] for k in util.WKEYS}
    ref = util.make_engine(syn1)
    try:
        plan = ref.plan_nodes(nodes, 3)
        m0 = _m0(plan, syn1)
        hp = ref.make_hparams(num_epochs=EPOCHS)
        want_mask = np.zeros(plan.total_edges, np.float32)
        ref.explain_nodes_host(hp, m0, want_mask)
        total = int(np.sum(np.diff(plan.node_off) ** 2))
        want_node = (want_mask, ref.densify_host(want_mask, total)) + ref.denoise_topk_edges(want_mask, 20)
        ref.set_model(gw)
        ref.set_graph_batch(gg["adj"], gg["feat"], gg["label"])
        eo = ref.plan_graphs(GIDS)
        gm0 = np.concatenate([gg["g%d_m0" % g] for g in GIDS])
        want_g = np.zeros(int(eo[-1]), np.float32)
        ref.explain_graphs_host(hp, gm0, want_g)
        want_graph = (want_g, ref.densify_graphs_host(GIDS, want_g))
    finally:
        ref.close()
    pinned, gpinned = torch.from_numpy(m0).pin_memory(), torch.from_numpy(gm0).pin_memory()
    eng = util.make_engine(syn1)
    try:
        eng.set_graph_batch(gg["adj"], gg["feat"], gg["label"])
        side = torch.cuda.Stream()
        for s in (side, torch.cuda.default_stream()):
            eng.set_model(syn1.weights)
            eng.set_stream(s.cuda_stream)
            eng.plan_nodes(nodes, 3)
            with torch.cuda.stream(s):
                m0_dev = torch.empty(len(m0), dtype=torch.float32, device="cuda")
                torch.cuda._sleep(200_000_000)
                m0_dev.copy_(pinned, non_blocking=True)
                mask = eng.explain_nodes_device(hp, m0_dev)
                got = (mask, eng.densify_device(mask)) + eng.denoise_topk_edges(mask, 20)
                got = tuple(x.cpu() for x in got)
            _same(got, want_node, "nodes on %s" % s)
            eng.set_model(gw)
            eng.plan_graphs(GIDS)
            with torch.cuda.stream(s):
                gm0_dev = torch.empty(len(gm0), dtype=torch.float32, device="cuda")
                torch.cuda._sleep(200_000_000)
                gm0_dev.copy_(gpinned, non_blocking=True)
                out = eng.explain_graphs_device(hp, gm0_dev)
                got = tuple(x.cpu() for x in (out, eng.densify_graphs_device(GIDS, out)))
            _same(got, want_graph, "graphs on %s" % s)
        eng.set_stream(0)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ d. the drop-in under a side stream
def _args(tmp_path, fx, init, **over):
    a = dict(num_gc_layers=3, num_epochs=EPOCHS, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid", mask_bias=False, gpu=False,
             bias=True, method="base", dataset=fx.name, bmname=None, hidden_dim=20, output_dim=20, name_suffix="", explainer_suffix="",
             logdir=str(tmp_path), gnnx_init=init, gnnx_seed=5)
    a.update(over)
    return types.SimpleNamespace(**a)


def _node_explainer(fx, args):
    model = gnnx.models.GcnEncoderNode(fx.feat.shape[1], 20, 20, fx.weights["Wp"].shape[0], 3, bn=False, args=args)
    sd = {"conv_first.weight": fx.weights["W1"], "conv_first.bias": fx.weights["b1"], "conv_block.0.weight": fx.weights["W2"],
          "conv_block.0.bias": fx.weights["b2"], "conv_last.weight": fx.weights["W3"], "conv_last.bias": fx.weights["b3"],
          "pred_model.weight": fx.weights["Wp"], "pred_model.bias": fx.weights["bp"]}
    model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    A = O.dense_from_csr(fx.rowptr, fx.col)
    return gnnx.Explainer(model=model, adj=A[None], feat=fx.feat[None], label=fx.label[None], pred=fx.pred[None], train_idx=[], args=args,
                          writer=None, print_training=False, graph_idx=-1)


def _graph_explainer(gg, args):
    torch.manual_seed(17)
    model = gnnx.models.GcnEncoderGraph(gg["feat"].shape[2], 20, 20, 2, 3, args=args)
    w = {k: gg[k] for k in util.WKEYS}
    sd = {"conv_first.weight": w["W1"], "conv_first.bias": w["b1"], "conv_block.0.weight": w["W2"], "conv_block.0.bias": w["b2"],
          "conv_last.weight": w["W3"], "conv_last.bias": w["b3"], "pred_model.weight": w["Wp"], "pred_model.bias": w["bp"]}
    model.load_state_dict({k: torch.tensor(np.asarray(v)) for k, v in sd.items()})
    return gnnx.Explainer(model=model, adj=torch.tensor(gg["adj"], dtype=torch.float), feat=torch.tensor(np.asarray(gg["feat"], np.float32)),
                          label=torch.tensor(np.asarray(gg["label"])), pred=None, train_idx=[], args=args, writer=None, print_training=False,
                          graph_mode=True, graph_idx=0)


def _on(stream, fn):
    """fn() under `with torch.cuda.stream(stream)` (None: the default stream), its results copied to the host on that stream."""
    torch.manual_seed(3)
    if stream is None:
        res = fn()
    else:
        with torch.cuda.stream(stream):
            res = fn()
            res = [x.cpu() if torch.is_tensor(x) else np.array(x, copy=True) for x in res]
    return [x.cpu() if torch.is_tensor(x) else np.array(x, copy=True) for x in res]


@pytest.mark.parametrize("copy", [True, False], ids=["copy", "shared_buffer"])
@pytest.mark.parametrize("init", ["device", "torch"])
def test_dropin_explain_nodes_on_a_side_stream(syn1, tmp_path, init, copy):
    """Explainer.explain_nodes (device densify, pinned host copy) inside `with torch.cuda.stream(side)`: the same bits as on the default
    stream.  The side stream runs first, into memory no earlier call has filled."""
    ex = _node_explainer(syn1, _args(tmp_path, syn1, init))
    try:
        side = torch.cuda.Stream()
        nodes = list(range(0, syn1.N, 3))
        got = _on(side, lambda: ex.explain_nodes(nodes, save=False, copy=copy))
        want = _on(None, lambda: ex.explain_nodes(nodes, save=False, copy=copy))
        _same(got, want, "explain_nodes")
    finally:
        ex.engine.close()


@pytest.mark.parametrize("init", ["device", "torch"])
def test_dropin_explain_nodes_topk_on_a_side_stream(syn1, tmp_path, init):
    ex = _node_explainer(syn1, _args(tmp_path, syn1, init))
    try:
        side = torch.cuda.Stream()
        nodes = list(range(0, syn1.N, 2))
        got = _on(side, lambda: ex.explain_nodes_topk(nodes, chunk_size=100))
        want = _on(None, lambda: ex.explain_nodes_topk(nodes, chunk_size=100))
        _same(got, want, "explain_nodes_topk")
    finally:
        ex.engine.close()


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def test_dropin_sharded_on_a_side_stream(syn1, gg, tmp_path):
    """gnnx.dist.explain_nodes_sharded, explain_nodes_topk_sharded and explain_graphs_sharded(dense=True) on a one-rank group, through gloo
    and through the engine's own communicator, inside `with torch.cuda.stream(side)`: the same bits as on the default stream."""
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % _free_port(), rank=0, world_size=1)
    try:
        ex = _node_explainer(syn1, _args(tmp_path, syn1, "torch"))
        gex = _graph_explainer(gg, _args(tmp_path, syn1, "torch", dataset="graphs"))
        nodes = list(range(1, syn1.N, 3))
        gids = [4, 1, 9, 1, 0, 11, 6]
        side = torch.cuda.Stream()
        try:
            for use_engine_comm in (False, True):
                calls = {
                    "nodes": lambda: gdist.explain_nodes_sharded(ex, nodes, use_engine_comm=use_engine_comm)[:2],
                    "topk": lambda: gdist.explain_nodes_topk_sharded(ex, nodes, chunk_size=100, use_engine_comm=use_engine_comm)[:4],
                    "graphs": lambda: (lambda r: (r[0], r[1], r[3]))(gdist.explain_graphs_sharded(gex, gids, use_engine_comm=use_engine_comm,
                                                                                                      dense=True)),
                }
                for name, fn in calls.items():
                    got = _on(side, fn)
                    want = _on(None, fn)
                    _same(got, want, (name, use_engine_comm))
        finally:
            ex.engine.close()
            gex.engine.close()
    finally:
        dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------ e. densify_device without a fetched plan
def test_densify_device_after_plan_without_fetch(syn1):
    """plan_nodes(fetch=False) of a larger batch than the last fetched plan: densify_device sizes its output from the library's current
    plan.  The size is asserted before any library call writes into it."""
    small, big = syn1.nodes[:5], syn1.nodes[:60]
    ref = util.make_engine(syn1)
    try:
        plan = ref.plan_nodes(big, 3)
        m0 = _m0(plan, syn1)
        hp = ref.make_hparams(num_epochs=EPOCHS)
        want = np.zeros(plan.total_edges, np.float32)
        ref.explain_nodes_host(hp, m0, want)
        total = int(np.sum(np.diff(plan.node_off) ** 2))
        want_dense = ref.densify_host(want, total)
    finally:
        ref.close()
    eng = util.make_engine(syn1)
    try:
        eng.plan_nodes(small, 3)
        assert eng.plan_nodes(big, 3, fetch=False) is None
        assert eng._dense_total() == total
        mask = eng.explain_nodes_device(hp, torch.from_numpy(m0).cuda())
        dense = eng.densify_device(mask)
        assert dense.numel() == total
        _same((mask.cpu(), dense.cpu()), (want, want_dense))
    finally:
        eng.close()
