"""GPU (-m gpu): the WHOLE mask of the unconstrained kernel (explain_dense.cu), mask_dense of gx_explain_{nodes,graphs}_unconstrained,
entry by entry.  The edge slots are a few percent of its n^2 entries; the rest (non-edges inside the k-hop rows, graph mode's padding
and isolated rows) move too and feed the next forward.  Checked per entry class (dense_oracle.entry_classes):
  * shapes across every tile edge of the 16 x 32 tensor-core tiles (n = 2 .. 4096, max_nodes = 2 .. 4096), input widths and models
    whose concatenated width K = d + hid (L - 1) + emb leaves every remainder mod 8, after 1, 2 and 5 updates, against the fp64
    closed form;
  * every optimiser and scheduler and two hyper-parameter sets, after 5 updates against the closed form and after 30 epochs against
    the line-by-line port; per epoch, the trace's size / entropy / feat-size sums (all n^2 entries, the diagonal included, and the
    feature mask) against the closed form's;
  * the unmodified reference's full masks (tests/golden/unconstrained_full_golden.npz) at 10 and 30 epochs."""
import os

import numpy as np
import pytest
import torch

import gnnx
from gnnx import _abi
import dense_oracle as D
import gnnx_oracle as O
import util
from test_gpu_unconstrained import _args, _bench, _load, _random_model, graph_engine, graph_weights, run, run_graphs, run_nodes

pytestmark = pytest.mark.gpu
UF = np.load(os.path.join(util.GOLDEN, "unconstrained_full_golden.npz"))
GG = np.load(os.path.join(util.GOLDEN, "graphs_golden.npz"))
NMAX = int(GG["max_nodes"])


# ------------------------------------------------------------------------------------ models, hyper-parameters
MODELS = {"m20": dict(hid=20, emb=20, L=3), "m16x12": dict(hid=16, emb=12, L=3), "bn64x48": dict(hid=64, emb=48, L=3, bn=True),
          "L2w128x96": dict(hid=128, emb=96, L=2), "L4": dict(hid=20, emb=20, L=4), "L6": dict(hid=20, emb=20, L=6),
          "head": dict(hid=20, emb=20, L=3, head=(24, 10))}


def make_model(name, d, C, seed):
    c = MODELS[name]
    rng = np.random.default_rng(seed)
    W = _random_model(rng, d, c["hid"], c["emb"], C, c["L"])
    if "head" in c:   # pred_model = Linear(PD, 24), ReLU, Linear(24, 10), ReLU, Linear(10, C)
        width, head = c["hid"] * (c["L"] - 1) + c["emb"], []
        for h in c["head"]:
            head.append(((rng.normal(size=(h, width)) * 0.4).astype(np.float32), (rng.normal(size=h) * 0.4).astype(np.float32)))
            width = h
        W["head"] = head
        W["Wp"] = (rng.normal(size=(C, width)) * 0.4).astype(np.float32)
    return W, c["L"], c.get("bn", False)


def set_model(eng, W, L, bn):
    eng.set_model({k: v for k, v in W.items() if k != "head"}, num_layers=L, bn=bn, head=W.get("head"))


HSETS = {"H1": dict(beta1=0.5, beta2=0.99, eps=1e-3), "H2": dict(size=0.05, ent=0.3, lap=4.0, feat_size=0.2)}
GX_NAMES = dict(beta1="beta1", beta2="beta2", eps="eps", size="coef_size", ent="coef_ent", lap="coef_lap", feat_size="coef_feat_size")


def hparams(eng, E, opt="adam", sched="none", hset=None):
    """(gx_hparams, oracle hparams) of one run: StepLR halves the rate every 3 epochs, cosine restarts after 4 (both inside a 5-update
    run)."""
    over = dict(opt=opt, opt_scheduler=sched, opt_decay_step=3, opt_decay_rate=0.5, opt_restart=4, **HSETS.get(hset, {}))
    gx = dict(opt=_abi.GX_OPT[opt], opt_scheduler=_abi.GX_SCHED[sched], opt_decay_step=3, opt_decay_rate=0.5, opt_restart=4)
    gx.update({GX_NAMES[k]: v for k, v in HSETS.get(hset, {}).items()})
    return eng.make_hparams(num_epochs=E, **gx), O.default_hparams(num_epochs=E, **over)


# ------------------------------------------------------------------------------------ graphs with a known k-hop set
def path(k):
    return O.csr_from_edges(k, np.array([[i, i + 1] for i in range(k - 1)], np.int64)), 0


def spider(legs):
    """A centre with legs of the given lengths (a star when every leg is 1); node 0 is the centre."""
    edges, nxt = [], 1
    for ln in legs:
        prev = 0
        for _ in range(ln):
            edges.append([prev, nxt]); prev = nxt; nxt += 1
    return O.csr_from_edges(nxt, np.array(edges, np.int64)), 0


def ba(N, m, seed, node):
    rowptr, col = _bench().make_ba_csr(N, m, seed)
    return (rowptr, col), node


# (n, d, model, optimiser-scheduler, K mod 8, graph builder); K = d + hid (L - 1) + emb, the columns of the pair product dZc Hc^T
NODE_CASES = [
    (2, 3, "m20", "adam-none", 7, lambda: path(2)),
    (3, 1, "m20", "sgd-none", 5, lambda: path(3)),
    (15, 8, "m16x12", "rmsprop-none", 4, lambda: spider([1] * 14)),
    (16, 9, "m20", "adagrad-none", 5, lambda: spider([3] * 5)),
    (17, 3, "bn64x48", "adam-step", 3, lambda: spider([3] * 5 + [1])),
    (31, 128, "L2w128x96", "adam-none", 0, lambda: ba(300, 1, 0, 16)),
    (32, 8, "L4", "adam-cos", 0, lambda: ba(300, 1, 0, 281)),
    (33, 9, "L6", "sgd-none", 1, lambda: ba(300, 1, 8, 261)),
    (48, 8, "head", "adam-none", 4, lambda: spider([3] * 15 + [2])),
    (49, 1, "m20", "rmsprop-cos", 5, lambda: ba(300, 1, 0, 60)),
    (4095, 3, "m20", "sgd-none", 7, lambda: spider([1] * 4094)),
    (4096, 9, "m16x12", "sgd-step", 5, lambda: spider([3] * 1365)),
]
# (max_nodes, d, model, optimiser-scheduler, K mod 8, [real nodes per graph]): each graph is a BA tree over all but its last real node,
# which is isolated, and padding rows up to max_nodes (max_nodes = 2: one edge, nothing else fits).  max_nodes = 4096 runs a model
# variant: gx_plan_graphs sizes the default model's graphs for the shared-memory graph kernel, which cannot hold 3000 nodes.
GRAPH_CASES = [
    (2, 3, "m20", "adam-none", 7, [2]),
    (16, 8, "bn64x48", "sgd-none", 0, [13, 9]),
    (17, 1, "L4", "rmsprop-none", 1, [15, 16]),
    (33, 9, "head", "adagrad-none", 5, [30, 21]),
    (100, 128, "L2w128x96", "sgd-step", 0, [97, 64]),
    (4096, 3, "L4", "sgd-cos", 3, [3000]),
]
# The n = 4096 cases and max_nodes = 100 run SGD, whose step is linear in the gradient.  Adam, RMSprop and Adagrad take a first step of about lr * sign(g):
# an entry whose gradient is within rounding of zero lands anywhere in (-lr, lr).  Among the 4094 centre-row entries of a 4095-node star
# the smallest |g| is 4e-7, and there fp32-grade gradients (the kernel's and the port's alike) cannot fix the sign-like step to 1e-5.


def k_concat(W, L):
    """K of the pair product from the weights themselves."""
    return W["W1"].shape[0] + sum(W["W%d" % l].shape[1] for l in range(1, L + 1))


def _id(c, what):
    return "%s%d-d%d-%s-%s" % (what, c[0], c[1], c[2], c[3])


def run_graphs_n(eng, gids, hp, m0_list, n, **kw):
    """run_graphs for a batch of max_nodes = n."""
    edge_off = eng.plan_graphs(gids)
    return edge_off, run(eng, hp, m0_list, len(gids), [n] * len(gids), edge_off[-1], graphs=True, **kw)


def assert_no_sign_tie(tr, opt, A):
    """Adam, RMSprop and Adagrad move an entry by about lr * sign(g) on their first update, so an entry whose fp64 gradient is within
    rounding of zero is ambiguous: the case's draw must have none (|g| >= 1e-6 off the diagonal)."""
    if opt != "sgd":
        off = ~np.eye(len(A), dtype=bool)
        assert np.abs(tr[0]["gM"][off]).min() >= 1e-6, "a near-tie in the first update: redraw the case"


def updates_of(n):
    """Update counts compared: the fp64 closed form at n = 4096 costs seconds per epoch on the CPU."""
    return (1, 2) if n > 1024 else (1, 2, 5)


# ------------------------------------------------------------------------------------ the oracles on one task
class Task:
    """One dense problem: A (n, n), X, gt, y (node mode), idx, W, L, bn, M0, graph_mode."""

    def __init__(self, A, X, gt, y, idx, W, L, bn, M0, graph_mode):
        self.A, self.X, self.gt, self.y, self.idx, self.W, self.L, self.bn, self.M0, self.graph = A, X, gt, y, idx, W, L, bn, M0, graph_mode

    def closed_form(self, hp):
        """The fp64 closed form over hp.num_epochs epochs: per epoch its dense mask and regulariser sums (dense_oracle trace)."""
        tr = []
        D.explain_closed_form(self.A, self.X, self.gt, self.y, self.idx, self.W, self.M0, hp=hp, graph_mode=self.graph, bn=self.bn,
                              full=True, trace=tr)
        return tr

    def port(self, hp):
        """The fp32 line-by-line port's whole mask after hp.num_epochs - 1 updates."""
        return O.explain_dense_torch(self.A, self.X, self.gt, self.y, self.idx, self.W, self.M0, hp=hp, graph_mode=self.graph, bn=self.bn,
                                     full=True, unconstrained=True)


def compare_to_closed_form(gpu, cf, port, A, what, bad, report):
    """Every off-diagonal entry within max(1e-5 x class max, 3 x the class's fp32-port distance from the fp64 closed form), and the
    class's rel-L2 within max(1e-5, 3 x the port's); the diagonal is exactly zero and the mask symmetric."""
    if not (np.all(np.diag(gpu) == 0) and np.array_equal(gpu, gpu.T)):
        bad[what + ":diag/sym"] = True
    for c, (r, k) in D.entry_classes(A).items():
        g, x, p = gpu[r, k].astype(np.float64), cf[r, k], port[r, k]
        tol = max(1e-5 * np.abs(x).max(), 3.0 * np.abs(p - x).max())
        err = np.abs(g - x).max()
        rl, rl_tol = O.rel_l2(g, x), max(1e-5, 3.0 * O.rel_l2(p, x))
        w = int(np.abs(g - x).argmax())
        report.append("%s %s: %d entries, max |err| %.2e at (%d, %d) (tol %.2e), rel-L2 %.2e (tol %.2e)"
                      % (what, c, len(r), err, r[w], k[w], tol, rl, rl_tol))
        if not (err <= tol and rl <= rl_tol):
            bad["%s:%s" % (what, c)] = (err, tol, rl, rl_tol)


# ------------------------------------------------------------------------------------ (2) shape sweep, node mode
@pytest.mark.parametrize("case", NODE_CASES, ids=[_id(c, "n") for c in NODE_CASES])
def test_node_shapes_match_closed_form(case):
    n, d, model, optsched, k8, build = case
    opt, sched = optsched.split("-")
    W, L, bn = make_model(model, d, 3, seed=n)
    (rowptr, col), node = build()
    N = len(rowptr) - 1
    rng = np.random.default_rng(1000 + n)
    feat = rng.normal(size=(N, d)).astype(np.float32)
    label = rng.integers(0, 3, N).astype(np.int32)
    pl = rng.integers(0, 3, N).astype(np.int32)
    eng = gnnx.Engine(0)
    set_model(eng, W, L, bn)
    eng.set_graph_csr(rowptr, col, feat, label, pl)
    plan = eng.plan_nodes([node], L)
    # the regime the case exists for: the builder's L-hop set has exactly n rows (n mod 16 / 32 the tile tails), K mod 8 the K tail
    assert (plan.n(0), plan.n(0) % 16, plan.n(0) % 32, feat.shape[1], k_concat(W, L) % 8) == (n, n % 16, n % 32, d, k8)
    idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(rowptr, col, feat, label, node, L)
    A = O.dense_from_csr(srp, scol)
    assert np.array_equal(plan.neighbors_of(0), nbrs)
    M0 = O.draw_m0(n, seed={32: 232}.get(n, n))   # n = 32 redrawn off a first-update near-tie (assert_no_sign_tie)
    task = Task(A, X, int(lab[idx]), pl[nbrs], idx, W, L, bn, M0, False)
    U = updates_of(n)
    tr = task.closed_form(hparams(eng, max(U) + 1, opt, sched)[1])
    assert_no_sign_tie(tr, opt, A)
    bad, report = {}, []
    for u in U:
        hp, hp_o = hparams(eng, u + 1, opt, sched)
        out, md, _, _ = run_nodes(eng, plan, hp, [M0], dense=True)
        r, c = plan.rows_cols_of(0)
        if not np.array_equal(md[0][r, c], out[:plan.total_edges]):      # the returned edge slots are the dense mask's, bit for bit
            bad["u%d:edge slots" % u] = True
        compare_to_closed_form(md[0], tr[u]["a"], task.port(hp_o), A, "u%d" % u, bad, report)
    eng.close()
    print("\n".join(report))
    assert not bad, bad


# ------------------------------------------------------------------------------------ (2) shape sweep, graph mode
SEED_OF = {17: 317, 33: 133}   # M0 seeds redrawn off a first-update near-tie (assert_no_sign_tie)


def graph_batch(max_nodes, reals, d, seed):
    """(adj (G, n, n), feat (G, n, d), label): graph g has reals[g] real nodes, a BA tree over all but the last (isolated) one; the
    padding rows have zero features, as the reference's padded batches."""
    G = len(reals)
    adj = np.zeros((G, max_nodes, max_nodes), np.float32)
    feat = np.zeros((G, max_nodes, d), np.float32)
    rng = np.random.default_rng(seed)
    for g, nr in enumerate(reals):
        if nr == 2:
            adj[g, 0, 1] = adj[g, 1, 0] = 1
        else:
            rowptr, col = _bench().make_ba_csr(nr - 1, 1, seed + g)
            rows = np.repeat(np.arange(nr - 1), np.diff(rowptr))
            adj[g, rows, col] = 1
        feat[g, :nr] = rng.normal(size=(nr, d))
    return adj, feat, rng.integers(0, 2, G).astype(np.int64)


@pytest.mark.parametrize("case", GRAPH_CASES, ids=[_id(c, "g") for c in GRAPH_CASES])
def test_graph_shapes_match_closed_form(case):
    mn, d, model, optsched, k8, reals = case
    opt, sched = optsched.split("-")
    W, L, bn = make_model(model, d, 2, seed=mn)
    adj, feat, label = graph_batch(mn, reals, d, seed=mn)
    assert (adj.shape[1], feat.shape[2], k_concat(W, L) % 8) == (mn, d, k8)
    eng = gnnx.Engine(0)
    set_model(eng, W, L, bn)
    eng.set_graph_batch(adj, feat, label)
    gids = list(range(len(reals)))
    M0 = [O.draw_m0(mn, seed=SEED_OF.get(mn, mn) + g) for g in gids]
    tasks = []
    for g in gids:
        A = adj[g].astype(np.float64)
        cls = D.entry_classes(A)
        if mn > 2:   # padding and isolated rows present: the case exercises the "pad" class
            assert "pad" in cls and not A[reals[g] - 1].any() and reals[g] < mn
        tasks.append(Task(A, feat[g], int(label[g]), None, 0, W, L, bn, M0[g], True))
    U = updates_of(mn)
    trs = [t.closed_form(hparams(eng, max(U) + 1, opt, sched)[1]) for t in tasks]
    for t, tr in zip(tasks, trs):
        assert_no_sign_tie(tr, opt, t.A)
    bad, report = {}, []
    for u in U:
        hp, hp_o = hparams(eng, u + 1, opt, sched)
        edge_off, (out, md, _, _) = run_graphs_n(eng, gids, hp, M0, mn, dense=True)
        for t, g in enumerate(gids):
            r, c = eng.graph_rows_cols(g)
            if not np.array_equal(md[t][r, c], out[edge_off[t]:edge_off[t + 1]]):
                bad["g%d u%d:edge slots" % (g, u)] = True
            compare_to_closed_form(md[t], trs[t][u]["a"], tasks[t].port(hp_o), tasks[t].A, "g%d u%d" % (g, u), bad, report)
    eng.close()
    print("\n".join(report))
    assert not bad, bad


# ------------------------------------------------------------------------------------ (3, 4) optimisers, schedulers, the trace
OPT_CASES = ["%s-%s" % (o, s) for o in ("adam", "sgd", "rmsprop", "adagrad") for s in ("none", "step", "cos")] + ["adam-none-H1", "adam-none-H2"]
TRACE_COLS = (("size", _abi.TR_SIZE), ("ent", _abi.TR_ENT), ("feat", _abi.TR_FEAT))


def trace_terms(tr_cf, hp_o, n, d):
    """The trace's TR_SIZE / TR_ENT / TR_FEAT of every epoch from the closed form's sums."""
    return {"size": np.array([hp_o.size * e["size"] for e in tr_cf]), "ent": np.array([hp_o.ent * e["ent"] / (n * n) for e in tr_cf]),
            "feat": np.array([hp_o.feat_size * e["feat"] / d for e in tr_cf])}


def _check_optimiser_task(eng, runner, task, opt, sched, hset, what, bad, report):
    n, d = len(task.A), task.X.shape[1]
    # 5 updates, every entry against the fp64 closed form
    hp, hp_o = hparams(eng, 6, opt, sched, hset)
    tr6 = task.closed_form(hp_o)
    md = runner(hp, dense=True)[1]
    compare_to_closed_form(md[0], tr6[5]["a"], task.port(hp_o), task.A, what + " u5", bad, report)
    # 30 epochs: the whole matrix against the port, per class within max(1e-4, 3 x the closed form's distance from the port)
    hp, hp_o = hparams(eng, 30, opt, sched, hset)
    tr30 = task.closed_form(hp_o)
    port = task.port(hp_o)
    md = runner(hp, dense=True)[1]
    _, md_t, tr, _ = runner(hp, dense=True, trace=True)
    if not np.array_equal(md[0], md_t[0]):
        bad[what + " e30:trace changed mask_dense"] = True
    for c, (r, k) in D.entry_classes(task.A).items():
        spread = O.rel_l2(tr30[29]["a"][r, k], port[r, k])
        err, tol = O.rel_l2(md[0][r, k], port[r, k]), max(1e-4, 3.0 * spread)
        report.append("%s e30 %s: rel-L2 vs port %.2e (tol %.2e)" % (what, c, err, tol))
        if not err <= tol:
            bad["%s e30:%s" % (what, c)] = (err, tol)
    # every epoch's regulariser sums over all n^2 entries (the diagonal's own recurrence included) and the feature mask
    want = trace_terms(tr30, hp_o, n, d)
    for name, col in TRACE_COLS:
        got = tr[0, :, col].astype(np.float64)
        rel = np.abs(got - want[name]) / np.maximum(np.abs(want[name]), 1e-30)
        report.append("%s trace %s: max rel %.2e" % (what, name, rel.max()))
        if not rel.max() <= 1e-5:
            bad["%s trace:%s" % (what, name)] = (int(rel.argmax()), rel.max())


@pytest.mark.parametrize("case", OPT_CASES, ids=["n55-d16-g40-d14-m20-" + c for c in OPT_CASES])
def test_optimisers_full_mask_and_trace(case):
    """rand node 33 (n = 55, 3 hops) and graph 9 of graphs_golden (31 real rows of 40), on their fixture models."""
    parts = case.split("-")
    opt, sched, hset = parts[0], parts[1], parts[2] if len(parts) > 2 else None
    bad, report = {}, []
    fx = util.load_fixture("rand")
    eng = util.make_engine(fx)
    plan = eng.plan_nodes([33], 3)
    idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(fx.rowptr, fx.col, fx.feat, fx.label, 33, 3)
    A = O.dense_from_csr(srp, scol)
    M0 = O.draw_m0(plan.n(0), seed=int(fx.gold["n33_seed"]))
    task = Task(A, X, int(lab[idx]), fx.pred_label[nbrs], idx, fx.weights, 3, False, M0, False)
    _check_optimiser_task(eng, lambda hp, **kw: run_nodes(eng, plan, hp, [M0], **kw), task, opt, sched, hset, "node33", bad, report)
    eng.close()
    eng = graph_engine(graph_weights())
    M0 = O.draw_m0(NMAX, seed=int(GG["g9_seed"]))
    A = GG["adj"][9].astype(np.float64)
    task = Task(A, GG["feat"][9], int(GG["label"][9]), None, 0, graph_weights(), 3, False, M0, True)
    _check_optimiser_task(eng, lambda hp, **kw: run_graphs(eng, [9], hp, [M0], **kw)[1], task, opt, sched, hset, "g9", bad, report)
    eng.close()
    print("\n".join(report))
    assert not bad, bad


# ------------------------------------------------------------------------------------ (5) against the reference's full masks
def ref_tol(key, c):
    return max(1e-4, 3.0 * max(float(UF["%s_spread_%s" % (key, c)]), float(UF["%s_cfdist_%s" % (key, c)])))


@pytest.mark.parametrize("which", ["syn1", "syn4", "rand"])
def test_nodes_full_mask_matches_reference(which):
    fx = util.load_fixture(which)
    eng = util.make_engine(fx)
    nodes = [int(v) for v in UF[which + "_nodes"]]
    plan = eng.plan_nodes(nodes, 3)
    m0 = [O.draw_m0(plan.n(t), seed=int(fx.gold["n%d_seed" % v])) for t, v in enumerate(nodes)]
    bad, report = {}, []
    for E in (int(e) for e in UF["epochs"]):
        out, md, _, _ = run_nodes(eng, plan, eng.make_hparams(num_epochs=E), m0, dense=True)
        for t, v in enumerate(nodes):
            assert np.array_equal(plan.neighbors_of(t), UF["%s_n%d_nbrs" % (which, v)])
            key = "%s_n%d_e%d" % (which, v, E)
            ref = UF[key + "_full"]
            r, c = plan.rows_cols_of(t)
            assert np.array_equal(md[t][r, c], out[plan.edge_off[t]:plan.edge_off[t + 1]])
            A = np.zeros(ref.shape); A[r, c] = 1
            for cl, (i, j) in D.entry_classes(A).items():
                err = O.rel_l2(md[t][i, j], ref[i, j])
                report.append("%s %s: %.2e (tol %.2e)" % (key, cl, err, ref_tol(key, cl)))
                if not err <= ref_tol(key, cl):
                    bad["%s:%s" % (key, cl)] = (err, ref_tol(key, cl))
    eng.close()
    print("\n".join(report))
    assert not bad, bad


def test_graphs_full_mask_matches_reference():
    eng = graph_engine(graph_weights())
    gids = [int(g) for g in UF["graphs"]]
    m0 = [O.draw_m0(NMAX, seed=int(GG["g%d_seed" % g])) for g in gids]
    bad, report = {}, []
    for E in (int(e) for e in UF["epochs"]):
        edge_off, (out, md, _, _) = run_graphs(eng, gids, eng.make_hparams(num_epochs=E), m0, dense=True)
        for t, g in enumerate(gids):
            key = "graphs_g%d_e%d" % (g, E)
            ref = UF[key + "_full"]
            r, c = eng.graph_rows_cols(g)
            assert np.array_equal(md[t][r, c], out[edge_off[t]:edge_off[t + 1]])
            for cl, (i, j) in D.entry_classes(GG["adj"][g]).items():
                err = O.rel_l2(md[t][i, j], ref[i, j])
                report.append("%s %s: %.2e (tol %.2e)" % (key, cl, err, ref_tol(key, cl)))
                if not err <= ref_tol(key, cl):
                    bad["%s:%s" % (key, cl)] = (err, ref_tol(key, cl))
    eng.close()
    print("\n".join(report))
    assert not bad, bad


def test_dropin_matches_reference_full_mask(tmp_path):
    """The drop-in Explainer(..., unconstrained=True) returns the full mask at the sub-adjacency slots and zero elsewhere: one node at
    30 epochs and one graph at 10, against the reference's full matrix."""
    fx = util.load_fixture("rand")
    args = _args(tmp_path)
    model = _load(gnnx.models.GcnEncoderNode(fx.feat.shape[1], 20, 20, 3, 3, bn=False, args=args), fx.weights)
    ex = gnnx.Explainer(model=model, adj=O.dense_from_csr(fx.rowptr, fx.col)[None], feat=fx.feat[None].astype(np.float64),
                        label=fx.label[None], pred=fx.pred[None], train_idx=list(range(fx.N)), args=args, writer=None,
                        print_training=False, graph_idx=-1)
    torch.manual_seed(int(fx.gold["n33_seed"]))
    masked = ex.explain(33, graph_idx=0, unconstrained=True)
    key = "rand_n33_e30"
    ref = UF[key + "_full"]
    _, sub_adj, _, _, _ = ex.extract_neighborhood(33)
    ei, ej = np.nonzero(sub_adj)
    assert masked.shape == ref.shape and np.all(masked[np.asarray(sub_adj) == 0] == 0)
    assert O.rel_l2(masked[ei, ej], ref[ei, ej]) <= ref_tol(key, "edge")
    args = _args(tmp_path, num_epochs=10, dataset="graphs")
    model = _load(gnnx.models.GcnEncoderGraph(14, 20, 20, 2, 3, bn=False, args=args), graph_weights())
    ex = gnnx.Explainer(model=model, adj=torch.tensor(GG["adj"], dtype=torch.float), feat=torch.tensor(GG["feat"]),
                        label=torch.tensor(GG["label"]), pred=GG["pred"], train_idx=[], args=args, writer=None,
                        print_training=False, graph_mode=True, graph_idx=0)
    torch.manual_seed(int(GG["g4_seed"]))
    masked = ex.explain(node_idx=0, graph_idx=4, graph_mode=True, unconstrained=True)
    key = "graphs_g4_e10"
    ref = UF[key + "_full"]
    ei, ej = np.nonzero(GG["adj"][4])
    assert masked.shape == ref.shape and np.all(masked[GG["adj"][4] == 0] == 0)
    assert O.rel_l2(masked[ei, ej], ref[ei, ej]) <= ref_tol(key, "edge")
