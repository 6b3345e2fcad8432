"""GPU (-m gpu): every explainer kernel's first-step gradients dL/dM (every directed slot) and dL/dF (every feature), element by element,
against fp64 torch autograd of the reference's loss (tests/mask_grad_oracle.py) at spread-out masks.

Readout.
  * Tuned kernels (explain_node.cu in every launch class and the cluster class, explain_gang.cu, explain_stream.cu with its outer pairs,
    explain_graph.cu; Adam only): two epochs from GX_INIT_STATE with beta1 = 0 and zero moments.  The one update sets exp_avg = g exactly,
    so adam_m_out is the kernel's g of every slot and feat_state_out[:, 1] its dL/dF; adam_v_out must be (1 - beta2) g^2 at the same
    slot.  M is drawn per directed slot ~ N(0, 1.5^2) and F ~ N(0, 1.5^2) (feat_state_in), so S and sigmoid(F) spread over (0.05, 0.95)
    and a backward that reads the wrong slot, the transposed entry or another feature's sigmoid gets different numbers.
  * Variant and dense kernels (explain_var.cu, explain_dense.cu; no optimiser-state output): two epochs of SGD, whose first step is
    P -= lr g.  M0 is symmetric, so g_ij = g_ji and the returned mask is sigmoid(M0 - lr g): g = (M0 - logit(mask)) / lr in fp64.  lr is
    set from the oracle's largest |g| and a second call at 1e3 x lr reads the elements with |lr g| < 1e-3.  F starts at 0 on this path
    (it has no state input), so every feature's first-step sigmoid is 0.5; gF = -logit(feat_mask) / lr_F from calls of their own.

Comparison, per element class (node mode: pairs by the hop levels of their endpoints, pairs touching the explained node; graph mode:
edges, non-edges and rows without edges of the dense mask; features):
    |g - g64| <= max(1e-5 scale_c, 5e-6 scale_task, 3 max_c |g32 - g64|, readout resolution),   scale_c = max_c |g64|,
and, wherever |g64| >= 1e-2 scale_c, |g - g64| <= max(2e-4 |g64|, the same task, fp32 and readout terms) (an element of a fresh syn4 run measured
1.1e-4).  On the 3xTF32 products of inputs wider than 128 the scale-relative bound is 3e-5.  g32 is the same oracle in float32.  Points
within 2 fp32 ulps of a ReLU kink or of a max-pool tie are redrawn.  Every test asserts the route it claims."""
import os
import types

import networkx as nx
import numpy as np
import pytest
import torch

import gnnx
from gnnx import _abi
import gnnx_oracle as O
import kernel_spec as KS
import mask_grad_oracle as MG
import util
from test_gpu_graph_shapes import _batch, _tree
from test_gpu_slab_shapes import _ba_case, _weights

pytestmark = pytest.mark.gpu

SMEM, SLAB, CLUSTER = 5, 5, 6         # launch classes 0..4: explain_node.cu; 5: the slab kernels; 6: the cluster class
KINK = 2 * 2.0 ** -23                 # redraw a point whose smallest relative ReLU input is below 2 fp32 ulps
SGD = _abi.GX_OPT["sgd"]
HP = O.default_hparams()
B2 = float(np.float32(1) - np.float32(0.999))


def _logit(p):
    p = np.asarray(p, np.float64)
    return np.log(p) - np.log1p(-p)


# ------------------------------------------------------------------------------------------------ problems and the oracle
class Problem:
    """One task (node or graph) with its oracle.  model: dict(bn, unconstrained) flags of mask_grads (the weights carry the model)."""

    def __init__(self, A, X, gt, pl, idx, w, graph_mode, **model):
        self.A, self.X, self.gt, self.pl, self.idx, self.w = np.asarray(A, np.float64), np.asarray(X), int(gt), pl, int(idx), w
        self.graph_mode = graph_mode
        self.model = {**dict(bn=False, unconstrained=False), **model}
        self.n, self.d = self.A.shape[0], self.X.shape[1]

    def grads(self, M, F):
        """(g64, g32) namespaces, or None when the point is too close to a ReLU kink or a pool tie."""
        kw = dict(graph_mode=self.graph_mode, **self.model)
        args = (self.A, self.X, self.gt, self.pl, self.idx, self.w, M, F, HP)
        g64 = MG.mask_grads(*args, dtype=torch.float64, **kw)
        if g64.kink < KINK or g64.ties:
            return None
        return g64, MG.mask_grads(*args, dtype=torch.float32, **kw)

    def classes(self, rows, cols):
        """{class name: boolean selector} over the slots (rows, cols)."""
        if self.graph_mode:
            edge = self.A[rows, cols] > 0
            live = self.A.sum(1) > 0
            out = {"edge": edge, "non_edge": ~edge & live[rows] & live[cols], "edgeless_row": ~live[rows] | ~live[cols]}
        else:
            rp, col = _csr(self.A)
            lvl = KS.hop_distances(rp, col, self.idx, self.n)
            lvl = np.where(lvl < 0, 9, lvl)
            lo, hi = np.minimum(lvl[rows], lvl[cols]), np.maximum(lvl[rows], lvl[cols])
            root = (rows == self.idx) | (cols == self.idx)
            loop = rows == cols
            out = {"root": root & ~loop, "loop": loop}
            for a in range(10):
                for b in range(a, 10):
                    sel = (lo == a) & (hi == b) & ~root & ~loop
                    if sel.any():
                        out["h%d%d" % (a, min(b, 9))] = sel
        return {k: v for k, v in out.items() if v.any()}


def _csr(A):
    rows, cols = np.nonzero(A)
    rp = np.zeros(A.shape[0] + 1, np.int64)
    np.add.at(rp, rows + 1, 1)
    return np.cumsum(rp), cols


def check(label, got, g64, g32, classes, res=None, floor=1e-5):
    """The per-class rule of the module docstring.  res: per-element readout resolution (SGD path), None on the Adam readout.  floor:
    the scale-relative bound, 3e-5 on the 3xTF32 products of inputs wider than 128 (TF32 hi / lo operands carry 21 bits, not 24)."""
    got, g64, g32 = (np.asarray(a, np.float64) for a in (got, g64, g32))
    res = np.zeros_like(g64) if res is None else res
    worst = {}
    # the kernels' sums carry the rounding of the task's largest terms into every class, also into small ones (a pair class of 6
    # elements at the explained node measured 3e-6 of the task's largest |g| where its own largest is 20x smaller)
    top = max((np.abs(g64[sel]).max() for sel in classes.values()), default=0.0)
    for name, sel in classes.items():
        scale = np.abs(g64[sel]).max()
        dev32 = 3 * np.abs(g32[sel] - g64[sel]).max()
        tol = np.maximum(max(floor * scale, 5e-6 * top, dev32), res[sel])
        err = np.abs(got[sel] - g64[sel])
        bad = err > tol
        assert not bad.any(), (label, name, "abs", int(bad.sum()), int(sel.sum()), float(err[bad].max()), float(tol[bad].min()), float(scale))
        big = np.abs(g64[sel]) >= 1e-2 * scale
        if big.any():
            rtol = np.maximum(np.maximum(20 * floor * np.abs(g64[sel][big]), max(5e-6 * top, dev32)), res[sel][big])
            bad = err[big] > rtol
            assert not bad.any(), (label, name, "rel", float((err[big] / np.abs(g64[sel][big])).max()), int(bad.sum()), int(big.sum()))
            worst[name] = float((err[big] / np.abs(g64[sel][big])).max())
    return worst


# ------------------------------------------------------------------------------------------------ tuned kernels: the Adam readout
def _node_problem(cs, plan, t, L=3):
    nbrs = plan.neighbors_of(t)
    idx = int(plan.node_idx_new[t])
    rp, col = plan.csr_of(t)
    A = O.dense_from_csr(rp, col)
    return Problem(A, cs.feat[nbrs], cs.label[nbrs][idx], cs.pred_label[nbrs], idx, cs.weights, False)


def _draw(prob, rows, cols, seed, sym=False):
    """(M dense (n, n) float32, F (d,) float32) at a point away from kinks and ties: M ~ N(0, 1.5^2) per slot (symmetric with sym), F ~
    N(0, 1.5^2) (zero with sym: the SGD path starts at F = 0)."""
    for k in range(8):
        rng = np.random.default_rng(seed + 7919 * k)
        M = rng.normal(0, 1.5, (prob.n, prob.n)).astype(np.float32)
        if sym:
            M = np.triu(M) + np.triu(M, 1).T
        F = np.zeros(prob.d, np.float32) if sym else rng.normal(0, 1.5, prob.d).astype(np.float32)
        g = prob.grads(M, F)
        if g is not None:
            return M, F, g
    raise AssertionError("no point away from ReLU kinks / pool ties in 8 draws")


def run_state(eng, plan_count, edge_off, rcs, probs, d, seed, graphs=False, trace=False, m0_init=None):
    """Adam readout of every task: -> {t: (g_slots, gF, g64, g32, rows, cols)}.  m0_init: GX_INIT_M0 at the given packed M0 instead."""
    te = int(edge_off[-1])
    M = np.zeros(te, np.float32)
    feat = np.zeros((plan_count, 3, d), np.float32)
    pts = []
    for t in range(plan_count):
        rows, cols = rcs[t]
        Md, F, g = _draw(probs[t], rows, cols, seed + 31 * t)
        if m0_init is not None:
            Md = np.zeros_like(Md); Md[rows, cols] = m0_init[edge_off[t]:edge_off[t + 1]]
            F = np.zeros_like(F)
            g = probs[t].grads(Md, F)
            assert g is not None, t
        M[edge_off[t]:edge_off[t + 1]] = Md[rows, cols]
        feat[t, 0] = F
        pts.append(g)
    so = dict(M=np.zeros(te, np.float32), m=np.zeros(te, np.float32), v=np.zeros(te, np.float32), feat=np.zeros((plan_count, 3, d), np.float32))
    out = np.zeros(max(te, 1), np.float32)
    tr = np.zeros((plan_count, 2, _abi.GX_TRACE_COLS), np.float32) if trace else None
    if m0_init is None:
        hp = eng.make_hparams(num_epochs=2, init=_abi.GX_INIT_STATE, beta1=0.0)
        eng.explain_nodes_ex(hp, M, out, trace=tr, state_in=dict(m=np.zeros(te, np.float32), v=np.zeros(te, np.float32), feat=feat),
                             state_out=so, graphs=graphs)
    else:
        eng.explain_nodes_ex(eng.make_hparams(num_epochs=2, beta1=0.0), M, out, trace=tr, state_out=so, graphs=graphs)
    # a state write to the wrong slot: exp_avg_sq must be (1 - beta2) g^2 where exp_avg is g
    m, v = so["m"][:te], so["v"][:te]
    assert np.allclose(v, np.float32(B2) * m * m, rtol=1e-6, atol=0), "adam_v_out is not (1 - beta2) g^2 at adam_m_out's slots"
    fm, fv = so["feat"][:, 1], so["feat"][:, 2]
    assert np.allclose(fv, np.float32(B2) * fm * fm, rtol=1e-6, atol=0)
    return {t: (m[edge_off[t]:edge_off[t + 1]], fm[t], pts[t][0], pts[t][1], *rcs[t]) for t in range(plan_count)}, so


def check_tasks(label, res, probs):
    worst = {}
    for t, (g, gF, g64, g32, rows, cols) in res.items():
        p = probs[t]
        w = check((label, t, "M"), g, g64.gM[rows, cols], g32.gM[rows, cols], p.classes(rows, cols))
        w.update(check((label, t, "F"), gF, g64.gF, g32.gF, {"feat": np.ones(p.d, bool)}))
        for k, e in w.items():
            worst[k] = max(worst.get(k, 0.0), e)
    print(label, "worst relative error per class:", {k: "%.1e" % e for k, e in sorted(worst.items())})
    return worst


def _node_engine(cs, generic=None, L=3, bn=False, **model):
    old = os.environ.get("GNNX_NODE_GENERIC")
    if generic is not None:
        os.environ["GNNX_NODE_GENERIC"] = "1" if generic else "0"
    try:
        eng = gnnx.Engine(0)
    finally:
        if generic is not None:
            if old is None:
                del os.environ["GNNX_NODE_GENERIC"]
            else:
                os.environ["GNNX_NODE_GENERIC"] = old
    eng.set_model(cs.weights, num_layers=L, bn=bn, **model)
    eng.set_graph_csr(cs.rowptr, cs.col, cs.feat, cs.label, cs.pred_label)
    return eng


def _node_state_run(label, cs, eng, nodes, seed, trace=False, m0_init=None):
    plan = eng.plan_nodes(nodes, 3)
    probs = [_node_problem(cs, plan, t) for t in range(plan.count)]
    rcs = [plan.rows_cols_of(t) for t in range(plan.count)]
    d = cs.feat.shape[1]
    res, so = run_state(eng, plan.count, plan.edge_off, rcs, probs, d, seed, trace=trace,
                        m0_init=None if m0_init is None else m0_init(plan))
    check_tasks(label, res, probs)
    return plan, res


def _classes_of(eng, nodes):
    out = {}
    for v in nodes:
        eng.plan_nodes([v], 3)
        out[v] = int(np.argmax(eng.plan_class_counts()[0]))
    return out


@pytest.mark.parametrize("generic,trace", [(0, False), (1, False), (0, True)], ids=["narrow", "generic", "narrow_trace"])
def test_node_smem_classes(generic, trace):
    """The fixtures' golden nodes (syn1 / syn4 / rand): every launch class 0..4 of explain_node.cu, narrow and generic instantiations,
    with and without a trace."""
    seen = set()
    for which in ("syn1", "syn4", "rand"):
        fx = util.load_fixture(which)
        eng = _node_engine(fx, generic)
        cls = _classes_of(eng, fx.nodes)
        seen |= set(cls.values())
        plan = eng.plan_nodes(fx.nodes, 3)
        counts, csz = eng.plan_class_counts()
        assert counts[SMEM:].sum() == 0 and csz == 1, counts
        _node_state_run((which, generic, trace), fx, eng, fx.nodes, 100 + generic, trace=trace)
        eng.close()
    assert seen >= set(range(SMEM)), sorted(seen)


def test_node_from_reference_m0():
    """GX_INIT_M0 at the reference's own draw (the IEEE sigmoid of the first S): the load path of a fresh explanation."""
    fx = util.load_fixture("syn4")
    eng = util.make_engine(fx)
    _node_state_run("syn4_m0", fx, eng, fx.nodes, 7, m0_init=lambda plan: util.golden_m0(fx, plan))
    eng.close()


@pytest.mark.parametrize("cs_size", [2, 4])
def test_node_cluster_class(cs_size):
    fx = util.load_fixture("syn1")
    eng = util.make_engine(fx)
    nodes = fx.nodes[:6]
    eng.debug_cluster(cs_size, 1)
    eng.plan_nodes(nodes, 3)
    counts, csz = eng.plan_class_counts()
    assert counts[CLUSTER] == len(nodes) and csz == cs_size, (counts, csz)
    _node_state_run(("cluster", cs_size), fx, eng, nodes, 200 + cs_size)
    eng.close()


def _hub_ba(seed=3, N=700, hub_deg=600, d=16, C=4, hid=20, emb=20):
    """BA(N, 2) plus a hub adjacent to hub_deg pool nodes: its row has more than 512 induced edges in every 3-hop neighbourhood."""
    rng = np.random.default_rng(seed)
    edges = [tuple(e) for e in nx.barabasi_albert_graph(N, 2, seed=seed).edges()]
    edges += [(N, int(p)) for p in rng.choice(N, hub_deg, replace=False)]
    rowptr, col = O.csr_from_edges(N + 1, np.array(edges, np.int64))
    feat = rng.normal(size=(N + 1, d)).astype(np.float32)
    return types.SimpleNamespace(N=N + 1, rowptr=rowptr, col=col, feat=feat, label=rng.integers(0, C, N + 1).astype(np.int32),
                                 pred_label=rng.integers(0, C, N + 1).astype(np.int32), weights=_weights(rng, d, C, hid, emb), L=3,
                                 bn=False, hub=N)


SLAB_CASES = {   # (seed, N, hid, emb, d, C)
    "h24e17_d1_C2": (71, 40, 24, 17, 1, 2), "h24e17_d33_C22": (72, 48, 24, 17, 33, 22),
    "h32e32_d128_C2": (73, 44, 32, 32, 128, 2), "h32e32_d33_C22": (74, 52, 32, 32, 33, 22), "h20e20_d128_C22": (75, 46, 20, 20, 128, 22),
}


@pytest.mark.parametrize("case", list(SLAB_CASES))
def test_node_slab_kernels(case):
    """BA cases forced into the slab class: gang sizes 0 (automatic) and 3 (explain_gang.cu) and -1 (explain_stream.cu, its outer pairs),
    each against the oracle; the gang and stream1 bits differ where both kernels really ran (explain_stream.cu for every setting at padded
    width 32 with d = 128)."""
    seed, N, hid, emb, d, C = SLAB_CASES[case]
    cs = _ba_case(seed, N, 2, d, C, hid, emb)
    nodes = list(range(0, N, N // 4))[:4]
    got = {}
    for gang in (0, 3, -1):
        eng = _node_engine(cs)
        eng.debug_force_stream(True)
        eng.debug_gang(gang)
        eng.plan_nodes(nodes, 3)
        assert eng.plan_class_counts()[0][SLAB] == len(nodes)
        _, res = _node_state_run((case, gang), cs, eng, nodes, seed)
        got[gang] = np.concatenate([res[t][0] for t in sorted(res)])
        eng.close()
    assert np.array_equal(got[0], got[3])
    gang_runs = not (max(hid, emb) > 24 and d == 128)
    assert np.array_equal(got[0], got[-1]) != gang_runs, "expected %s" % ("explain_gang.cu" if gang_runs else "explain_stream.cu")


@pytest.mark.parametrize("gang", [0, 3, -1], ids=["gang0", "gang3", "stream1"])
def test_node_hub_row_over_512(gang):
    cs = _hub_ba()
    eng = _node_engine(cs)
    eng.debug_force_stream(True)
    eng.debug_gang(gang)
    nodes = [cs.hub, 5]
    plan = eng.plan_nodes(nodes, 3)
    assert eng.plan_class_counts()[0][SLAB] == len(nodes)
    assert max(np.diff(plan.csr_of(t)[0]).max() for t in range(plan.count)) > 512
    _node_state_run(("hub", gang), cs, eng, nodes, 300)
    eng.close()


def test_node_self_loops():
    """Neighbourhoods of a graph with self loops (and a node whose only edge is its loop): the plan drops the diagonal, as the reference's
    diag_mask does, and every other slot keeps its gradient."""
    from test_gpu_grad import _loop_case
    cs = _loop_case()
    eng = _node_engine(cs)
    nodes = cs.looped[:4] + [cs.iso]
    plan = eng.plan_nodes(nodes, 3)
    assert all(cs.loops[plan.neighbors_of(t)].any() for t in range(plan.count))
    assert not any((lambda r, c: (r == c).any())(*plan.rows_cols_of(t)) for t in range(plan.count))
    _node_state_run("loops", cs, eng, nodes, 400)
    eng.close()


# ------------------------------------------------------------------------------------------------ graph mode, tuned kernel
def _graph_engine(w, adj, feat, label, L=3, bn=False, **model):
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bn, **model)
    eng.set_graph_batch(adj, feat, label)
    return eng


def _graph_problems(eng, w, adj, feat, label, gids, **model):
    return [Problem(adj[g], feat[g], label[g], None, 0, w, True, **model) for g in gids], [eng.graph_rows_cols(g) for g in gids]


@pytest.mark.parametrize("case", ["classes", "h24e17_d128"])
def test_graph_tuned_kernel(case):
    """explain_graph.cu: one graph per footprint class 0..5 (BA(n, 2) at n = 6 .. 300, d = 14) or a 24/17 model at d = 128, padded rows
    and an edge-less row in every graph."""
    from test_gpu_graph_variants import _random_model
    rng = np.random.default_rng(11 if case == "classes" else 12)
    if case == "classes":
        sizes, n, d, hid, emb = [6, 15, 30, 50, 90, 300], 320, 14, 20, 20
        parts = [nx.to_numpy_array(nx.barabasi_albert_graph(s, 2, seed=1)).astype(np.uint8) for s in sizes]
    else:
        sizes, n, d, hid, emb = [20, 33], 40, 128, 24, 17
        parts = [_tree(rng, s, 4) for s in sizes]
    adj = _batch([(1, p) for p in parts], n)          # row 0 and the rows past the graph: no edges
    feat = rng.normal(size=(len(sizes), n, d)).astype(np.float32)
    label = rng.integers(0, 2, len(sizes))
    w = _random_model(rng, 3, False, hid, emb, d, 2, "normal")
    eng = _graph_engine(w, adj, feat, label)
    gids = list(range(len(sizes)))
    eo = eng.plan_graphs(gids)
    probs, rcs = _graph_problems(eng, w, adj, feat, label, gids)
    res, _ = run_state(eng, len(gids), eo, rcs, probs, d, 500, graphs=True)
    _, end = eng.last_class_ms()
    ran = [c for c in range(6) if end[c] >= 0]
    if case == "classes":
        assert ran == list(range(6)), ran
    else:
        assert ran, ran
    check_tasks(("graph", case), res, probs)
    eng.close()


# ------------------------------------------------------------------------------------------------ variant and dense kernels: SGD readout
def _sgd_read(call, M0s, g64s, lr_scale=1.0):
    """g of every element from two SGD calls (lr from max |g64|, then 1e3 x lr for |lr g| < 1e-3): call(lr) -> list of fp32 masks at the
    same elements as M0s (fp64 arrays).  Returns (g, resolution) lists."""
    gmax = max(np.abs(g).max() for g in g64s)
    lr = lr_scale / gmax
    outs = {}
    for k, f in ((0, 1.0), (1, 1e3)):
        masks = call(lr * f)
        outs[k] = [(np.asarray(mk, np.float64), lr * f) for mk in masks]
    gs, ress = [], []
    for t, (M0, g64) in enumerate(zip(M0s, g64s)):
        pick = np.abs(lr * g64) < 1e-3
        g = np.empty_like(g64); res = np.empty_like(g64)
        for k, sel in ((0, ~pick), (1, pick)):
            mk, l = outs[k][t]
            mk = mk[sel]
            M1 = np.float32(M0[sel]) - np.float32(l) * np.float32(g64[sel])
            g[sel] = (M0[sel] - _logit(mk)) / l
            # 4 ulps of the returned sigmoid and 2 of M1, in M units, over lr
            res[sel] = (4 * np.spacing(np.float32(mk)) / np.maximum(mk * (1 - mk), 1e-30) + 2 * np.spacing(np.abs(M1))) / l
        gs.append(g); ress.append(res)
    return gs, ress


def _variant_check(label, probs, rcs, call, seed, floor=1e-5):
    """probs / rcs per task; call(M0 list, lr) -> (fp32 masks at the compared elements, fp32 feature masks or None) per task."""
    pts = [_draw(p, *rc, seed + 13 * t, sym=True) for t, (p, rc) in enumerate(zip(probs, rcs))]
    M0s = [M for M, _, _ in pts]
    g64 = [g[0].gM[r, c] for (_, _, g), (r, c) in zip(pts, rcs)]
    g32 = [g[1].gM[r, c] for (_, _, g), (r, c) in zip(pts, rcs)]
    gs, ress = _sgd_read(lambda lr: call(M0s, lr)[0], [M.astype(np.float64)[r, c] for M, (r, c) in zip(M0s, rcs)], g64)
    for t, p in enumerate(probs):
        check((label, t, "M"), gs[t], g64[t], g32[t], p.classes(*rcs[t]), ress[t], floor)
    if call(M0s, 0.0)[1] is None:
        return
    gF64 = [g[0].gF for _, _, g in pts]
    gF32 = [g[1].gF for _, _, g in pts]
    gF, resF = _sgd_read(lambda lr: call(M0s, lr)[1], [np.zeros_like(g) for g in gF64], gF64)
    for t, p in enumerate(probs):
        check((label, t, "F"), gF[t], gF64[t], gF32[t], {"feat": np.ones(p.d, bool)}, resF[t], floor)


def _head(rng, PD, dims):
    out, width = [], PD
    for h in dims:
        out.append(((rng.normal(size=(h, width)) * np.sqrt(2.0 / width)).astype(np.float32), (rng.normal(size=h) * 0.3).astype(np.float32)))
        width = h
    return out


def _model(tag, seed, d_default=10):
    """(weights, L, bn, set_model keywords, mask_grads flags, d) of a variant case."""
    spec = dict(default=(3, False, 20, 20, d_default), L2=(2, False, 20, 20, d_default), L5=(5, False, 20, 20, d_default),
                L7=(7, False, 20, 20, d_default), bn=(3, True, 20, 20, d_default), w64_48=(3, False, 64, 48, d_default),
                w128=(3, False, 128, 128, d_default), w200_256=(3, False, 200, 256, d_default), d129=(3, False, 20, 20, 129),
                d1433=(3, False, 20, 20, 1433), att_L3_bn=(3, True, 20, 20, d_default), head50=(3, False, 20, 20, d_default),
                head256_7=(3, True, 20, 20, d_default))[tag]
    L, bn, hid, emb, d = spec
    rng = np.random.default_rng(seed)
    C = 4
    w = _weights(rng, d, C, hid, emb, L)
    kw, flags = {}, dict(bn=bn)
    if tag == "att_L3_bn":
        from test_oracle_att import random_att_model
        w = random_att_model(rng, d, hid, emb, C, L)
        kw["att"] = [w["Wa%d" % (l + 1)] for l in range(L)]
    if tag.startswith("head"):
        dims = [50] if tag == "head50" else [256, 7]
        head = _head(rng, hid * (L - 1) + emb, dims)
        w["head"] = head
        w["Wp"] = (rng.normal(size=(C, dims[-1])) * 0.5).astype(np.float32)
        kw["head"] = head
    return w, L, bn, kw, flags, d


VAR_TAGS = ["default", "L2", "L5", "L7", "bn", "w64_48", "w128", "w200_256", "d129", "d1433", "att_L3_bn", "head50", "head256_7"]


@pytest.mark.parametrize("tag", VAR_TAGS)
def test_variant_kernel_nodes(tag):
    w, L, bn, kw, flags, d = _model(tag, 900 + VAR_TAGS.index(tag))
    cs = _ba_case(60 + VAR_TAGS.index(tag), 60, 2, d, 4, 20, 20)
    cs.weights = w
    eng = _node_engine(cs, L=L, bn=bn, **kw)
    nodes = [0, 17, 42]
    plan = eng.plan_nodes(nodes, L)
    # a model variant plans every task into the slab class of the variant kernel; the default model is planned for the tuned kernels,
    # and an optimiser other than Adam sends the whole batch to explain_var.cu instead (node_mode.cu)
    assert eng.plan_class_counts()[0][SLAB] == (0 if tag == "default" else len(nodes))
    probs, rcs = [], []
    for t in range(plan.count):
        nbrs = plan.neighbors_of(t); idx = int(plan.node_idx_new[t])
        probs.append(Problem(O.dense_from_csr(*plan.csr_of(t)), cs.feat[nbrs], cs.label[nbrs][idx], cs.pred_label[nbrs], idx, w, False,
                             **flags))
        rcs.append(plan.rows_cols_of(t))
    _node_variant(("var_node", tag), eng, plan, probs, rcs, d, 910)
    eng.close()


def _node_variant(label, eng, plan, probs, rcs, d, seed):
    floor = 3e-5 if d > 128 else 1e-5
    def call(M0s, lr):
        m0 = np.concatenate([M[r, c] for M, (r, c) in zip(M0s, rcs)]).astype(np.float32)
        out = np.zeros(plan.total_edges, np.float32)
        fm = np.zeros((plan.count, d), np.float32)
        eng.explain_nodes_host(eng.make_hparams(num_epochs=2, lr=lr, opt=SGD), m0, out, fm)
        return [out[plan.edge_off[t]:plan.edge_off[t + 1]] for t in range(plan.count)], list(fm)

    _variant_check(label, probs, rcs, call, seed, floor)


def test_variant_kernel_hub_subgraph():
    """A subgraph of more than 1500 nodes on the variant kernel (the default model under SGD)."""
    cs = _ba_case(91, 2500, 2, 10, 4, 20, 20)
    hub = int(np.argmax(np.diff(cs.rowptr)))
    eng = _node_engine(cs)
    plan = eng.plan_nodes([hub], 3)
    assert 1500 < plan.n(0) <= 2200 and eng.plan_class_counts()[0][SLAB] == 1, plan.n(0)
    nbrs = plan.neighbors_of(0); idx = int(plan.node_idx_new[0])
    probs = [Problem(O.dense_from_csr(*plan.csr_of(0)), cs.feat[nbrs], cs.label[nbrs][idx], cs.pred_label[nbrs], idx, cs.weights, False)]
    _node_variant("var_hub", eng, plan, probs, [plan.rows_cols_of(0)], 10, 920)
    eng.close()


@pytest.mark.parametrize("tag", VAR_TAGS)
def test_variant_kernel_graphs(tag):
    w, L, bn, kw, flags, d = _model(tag, 950 + VAR_TAGS.index(tag))
    rng = np.random.default_rng(960 + VAR_TAGS.index(tag))
    n = 40
    adj = _batch([(1, _tree(rng, 25, 4)), (3, _tree(rng, 33, 6))], n)
    feat = rng.normal(size=(2, n, d)).astype(np.float32)
    label = np.array([1, 3])
    eng = _graph_engine(w, adj, feat, label, L=L, bn=bn, **kw)
    gids = [0, 1]
    eo = eng.plan_graphs(gids)
    probs, rcs = _graph_problems(eng, w, adj, feat, label, gids, **flags)

    def call(M0s, lr):
        m0 = np.concatenate([M[r, c] for M, (r, c) in zip(M0s, rcs)]).astype(np.float32)
        out = np.zeros(int(eo[-1]), np.float32)
        fm = np.zeros((len(gids), d), np.float32)
        eng.explain_graphs_host(eng.make_hparams(num_epochs=2, lr=lr, opt=SGD), m0, out, fm)
        return [out[eo[t]:eo[t + 1]] for t in range(len(gids))], list(fm)

    _variant_check(("var_graph", tag), probs, rcs, call, 970, 3e-5 if d > 128 else 1e-5)
    eng.close()


# ------------------------------------------------------------------------------------------------ dense kernel (unconstrained=True)
def _dense_rc(n):
    r, c = np.nonzero(1 - np.eye(n))
    return r, c


@pytest.mark.parametrize("model", ["default", "bn", "head50"])
@pytest.mark.parametrize("size", [37, 100, 1100])
def test_dense_kernel_nodes(model, size):
    """explain_dense.cu, node mode: every off-diagonal entry of the dense mask (the diagonal is masked out of the forward)."""
    w, L, bn, kw, flags, d = _model(model, 1000 + size)
    N = 1500
    cs = _ba_case(7, N, 2, d, 4, 20, 20)                     # 3-hop neighbourhoods from 22 to about 1200 nodes
    cs.weights = w
    eng = _node_engine(cs, L=L, bn=bn, **kw)
    n_all, _ = eng.count_nodes(np.arange(N, dtype=np.int32), 3)
    cand = np.nonzero((n_all % 16 != 0) & (np.abs(n_all - size) <= size // 8 + 3))[0]
    assert len(cand), (size, np.sort(n_all)[-5:])
    node = int(cand[np.argmin(np.abs(n_all[cand] - size))])
    plan = eng.plan_nodes([node], 3)
    n = plan.n(0)
    assert n % 16 and n % 32, n
    nbrs = plan.neighbors_of(0); idx = int(plan.node_idx_new[0])
    probs = [Problem(O.dense_from_csr(*plan.csr_of(0)), cs.feat[nbrs], cs.label[nbrs][idx], cs.pred_label[nbrs], idx, w, False,
                     unconstrained=True, **flags)]
    rc = _dense_rc(n)

    def call(M0s, lr):
        md = np.zeros(n * n, np.float32)
        eng.explain_nodes_unconstrained(eng.make_hparams(num_epochs=2, lr=lr, opt=SGD), M0s[0].reshape(-1),
                                        np.zeros(plan.total_edges, np.float32), md)
        return [md.reshape(n, n)[rc]], None

    _variant_check(("dense_node", model, n), probs, [rc], call, 1100)
    eng.close()


@pytest.mark.parametrize("model", ["default", "bn", "head50"])
@pytest.mark.parametrize("n", [37, 101])
def test_dense_kernel_graphs(model, n):
    w, L, bn, kw, flags, d = _model(model, 1200 + n)
    rng = np.random.default_rng(1200 + n)
    adj = _batch([(2, _tree(rng, n - 6, 5))], n)
    feat = rng.normal(size=(1, n, d)).astype(np.float32)
    label = np.array([2])
    eng = _graph_engine(w, adj, feat, label, L=L, bn=bn, **kw)
    eng.plan_graphs([0])
    probs = [Problem(adj[0], feat[0], label[0], None, 0, w, True, unconstrained=True, **flags)]
    rc = _dense_rc(n)

    def call(M0s, lr):
        md = np.zeros(n * n, np.float32)
        eng.explain_graphs_unconstrained(eng.make_hparams(num_epochs=2, lr=lr, opt=SGD), M0s[0].reshape(-1),
                                         np.zeros(max(int(adj.sum()), 1), np.float32), md)
        return [md.reshape(n, n)[rc]], None

    _variant_check(("dense_graph", model, n), probs, [rc], call, 1300)
    eng.close()
