"""GPU (-m gpu), one device: every persistent or grid-stride kernel on batches larger than its resident grid, so that CTAs take a second,
third, .. task in the same shared memory, pair slab and k-hop workspace.  Each test asserts the size that puts it past the grid it
computes from the launch constants (host.cuh kNodeClasses, GX_GRID_CAP, the 256-thread variant / dense CTAs, forward.cu's 8 warps).

  * the graphs are disjoint unions of K relabelled copies of small components (induced k-hop subgraphs of fixture nodes, or whole
    graphs).  A constant shift keeps the canonical and the level order, so with GX_INIT_M0 and the same M0 every copy has the same
    arithmetic: every task of the big batch must be bit-identical to copy 0 explained in a chunk where no CTA runs twice;
  * late tasks (the last copies: the queue is largest-first) against the reference goldens, the line-by-line torch port and the fp64
    closed form at the usual bars;
  * the integer and gather kernels (k-hop planner, top-k select, densify, unshard) against numpy / scipy, bit for bit."""
import math
import os
import types

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import gnnx
from gnnx import _abi
import gnnx_oracle as O
import util

pytestmark = pytest.mark.gpu

GRID_CAP = 132 * 8                 # GX_GRID_CAP (gnnx_internal.cuh): CTAs of the grid-stride kernels
SMEM_CTAS = [16, 8, 4, 2, 1]       # CTAs per SM of the shared-memory launch classes 0..4 (host.cuh, kNodeClasses)
SLAB_CTAS = 4                      # CTAs per SM of the variant kernel in node mode at most (api.cu, launch_var_batch)
VAR_THREADS = 256                  # threads of a variant / dense CTA (explain_var_common.cuh): at most 2048 / 256 per SM
FWD_WARPS = 8                      # warps per CTA of gx_model_forward (forward.cu, kFwdThreads = 256)


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ unions of relabelled copies
def component(rowptr, col, feat, label, pred_label, root, k):
    """The induced k-hop subgraph of `root` as a graph of its own (canonical ids), and root's id in it."""
    idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(rowptr, col, feat, label, root, k)
    return types.SimpleNamespace(rowptr=srp, col=scol, feat=np.asarray(sfeat, np.float32), label=np.asarray(slabel, np.int32),
                                 pred_label=np.asarray(pred_label)[nbrs].astype(np.int32), root=int(idx), n=len(nbrs), e=len(scol))


def union(comps, K):
    """K copies of the disjoint union of comps, copy k shifted by k * (nodes of one copy).  Returns the graph and roots (K, len(comps)):
    the global id of every component's root in every copy."""
    sizes = np.array([c.n for c in comps], np.int64)
    off = np.concatenate([[0], np.cumsum(sizes)])
    nb = int(off[-1])
    rp, cols, e0 = [np.zeros(1, np.int64)], [], 0
    for c, o in zip(comps, off):
        rp.append(c.rowptr[1:].astype(np.int64) + e0)
        cols.append(c.col.astype(np.int64) + o)
        e0 += len(c.col)
    rb, cb = np.concatenate(rp), np.concatenate(cols)
    k = np.arange(K, dtype=np.int64)[:, None]
    rowptr = np.concatenate([[0], (rb[1:][None, :] + e0 * k).ravel()]).astype(np.int32)
    col = (cb[None, :] + nb * k).ravel().astype(np.int32)
    cat = lambda a: np.concatenate([getattr(c, a) for c in comps])
    roots = (off[:-1] + np.array([c.root for c in comps]))[None, :] + nb * k
    return types.SimpleNamespace(N=nb * K, rowptr=rowptr, col=col, feat=np.tile(cat("feat"), (K, 1)), label=np.tile(cat("label"), K),
                                 pred_label=np.tile(cat("pred_label"), K), roots=roots.astype(np.int32), K=K)


def engine(g, w, L=3, bn=False, att=None, head=None, generic=False):
    """An engine on graph g.  GNNX_NODE_GENERIC is pinned for its creation: 0 lets inputs no wider than the hidden width take the
    narrow instantiation of the shared-memory kernel, 1 keeps the run-time-shape code for every width."""
    old = os.environ.get("GNNX_NODE_GENERIC")
    os.environ["GNNX_NODE_GENERIC"] = "1" if generic else "0"
    try:
        eng = gnnx.Engine(0)
    finally:
        if old is None:
            del os.environ["GNNX_NODE_GENERIC"]
        else:
            os.environ["GNNX_NODE_GENERIC"] = old
    try:
        eng.set_model(w, num_layers=L, bn=bn, att=att, head=head)
        eng.set_graph_csr(g.rowptr, g.col, g.feat, g.label, g.pred_label)
    except BaseException:
        eng.close()
        raise
    return eng


def graph_engine(w, adj, feat, label, L=3, bn=False):
    eng = gnnx.Engine(0)
    try:
        eng.set_model(w, num_layers=L, bn=bn)
        eng.set_graph_batch(adj, feat, label)
    except BaseException:
        eng.close()
        raise
    return eng


def packed(plan, dense):
    """dense[t] (n_t, n_t) M0 of every planned task -> the packed float32 M0 at the sub-adjacency slots."""
    out = np.empty(plan.total_edges, np.float32)
    for t in range(plan.count):
        r, c = plan.rows_cols_of(t)
        out[plan.edge_off[t]:plan.edge_off[t + 1]] = dense[t][r, c]
    return out


def per_copy(a, K):
    """A packed per-task array of a copy-major batch -> (K, one copy's worth)."""
    return np.asarray(a).reshape(K, -1)


def assert_copies(big, alone, K, what):
    """Every copy's part of `big` has the bits of `alone` (copy 0 explained on its own)."""
    rows = per_copy(big, K)
    ref = np.asarray(alone).reshape(-1)
    bad = [k for k in range(K) if not np.array_equal(rows[k].view(np.uint32), ref.view(np.uint32))]
    assert not bad, (what, "copies differ from the task run alone", bad[:10], len(bad))


def seg(a, off, t):
    return a[off[t]:off[t + 1]]


def port_check(got, fm, args, kw):
    """Edge mask within max(1e-4, 3 x the fp32 / fp64 distance of the torch port), the feature mask likewise."""
    p32, f32 = O.explain_dense_torch(*args, return_feat=True, **kw)
    p64, f64 = O.explain_dense_torch(*args, return_feat=True, dtype=torch.float64, **kw)
    tol = max(1e-4, 3 * O.rel_l2(p64, p32))
    err = O.rel_l2(got, p32)
    assert err <= tol, ("edge mask", err, tol)
    if fm is not None:
        ftol = max(1e-4, 3 * float(np.abs(f64 - f32).max()))
        ferr = float(np.abs(fm - f32).max())
        assert ferr <= ftol, ("feature mask", ferr, ftol)


# ------------------------------------------------------------------------------------------------ k-hop planner beyond its slots
def khop_slots(N, sms):
    """(slots of the k-hop workspace at N nodes, slots before halving): node_mode.cu ensure_slot_ws starts from 8 per SM and halves
    while the workspace exceeds 4 GiB."""
    W = (N + 31) // 32
    per_slot = W * 4 + (W + 1) * 4 + N + (N + 1) * 8 + N * 8 + 64
    slots = sms * 8
    while slots > 1 and per_slot * slots > 4 << 30:
        slots //= 2
    return slots, sms * 8


def reach(A, nodes, k):
    """Rows `nodes` of (A + A^2 + .. + A^k) > 0 (scipy): the root is a member only through a closed walk.  Each step multiplies 0/1
    int32 matrices, so a walk count cannot wrap to zero (a row has fewer than 2^31 entries)."""
    A = A.astype(bool).astype(np.int32)
    R = A[nodes].astype(bool)
    acc = R.copy()
    for _ in range(k - 1):
        R = (R.astype(np.int32) @ A).astype(bool)
        acc = (acc + R).astype(bool)
    return acc.tocsr()


def check_plan(A, nodes, k, plan, cnt):
    """The plan (neighbours, node_idx_new, induced CSR without the diagonal) and count_nodes against scipy, bit for bit."""
    R = reach(A, nodes, k)
    Aoff = A.tolil(copy=True)
    Aoff.setdiag(0)
    Aoff = Aoff.tocsr()
    Aoff.eliminate_zeros()
    n_c, e_c = cnt
    for t, v in enumerate(nodes):
        nb = R.indices[R.indptr[t]:R.indptr[t + 1]]
        nb = np.sort(nb)
        assert np.array_equal(plan.neighbors_of(t), nb), (k, t, v)
        assert int(plan.node_idx_new[t]) == int(np.searchsorted(nb, v)) and nb[plan.node_idx_new[t]] == v, (k, t, v)
        S = Aoff[nb][:, nb].tocsr()
        S.sort_indices()
        rp, col = plan.csr_of(t)
        assert np.array_equal(rp, S.indptr) and np.array_equal(col, S.indices), (k, t, v)
        assert n_c[t] == plan.n(t) == len(nb) and e_c[t] == plan.edge_off[t + 1] - plan.edge_off[t] == S.nnz, (k, t, v)


def test_khop_planner_past_its_slots(sms):
    """Two copies of syn1 with self loops on every 7th node: 1400 nodes through 8 slots per SM at 1 (self loops only), 2, 3 and 7 hops."""
    fx = util.load_fixture("syn1")
    A0 = sp.csr_matrix(O.dense_from_csr(fx.rowptr, fx.col))
    A0 = (A0 + sp.diags((np.arange(fx.N) % 7 == 0).astype(np.float64))).tocsr()
    A = sp.block_diag([A0, A0]).tocsr()
    A.sort_indices()
    N = A.shape[0]
    nodes = np.random.default_rng(0).permutation(N).astype(np.int32)
    assert len(nodes) > khop_slots(N, sms)[0]
    g = types.SimpleNamespace(rowptr=A.indptr.astype(np.int32), col=A.indices.astype(np.int32), feat=np.tile(fx.feat, (2, 1)),
                              label=np.tile(fx.label, 2), pred_label=np.tile(fx.pred_label, 2))
    eng = engine(g, fx.weights)
    try:
        for k in (1, 2, 3, 7):
            R = reach(A, nodes, k)
            rows = eng.neighborhood_rows(nodes, k)
            assert np.array_equal(rows, R.toarray().astype(np.uint8)), k
            n_c, e_c = eng.count_nodes(nodes, k)
            assert np.array_equal(n_c, np.diff(R.indptr)), k
            if k == 1:
                continue
            plan = eng.plan_nodes(nodes, k)
            check_plan(A, nodes, k, plan, (n_c, e_c))
    finally:
        eng.close()


def test_khop_planner_on_a_graph_whose_workspace_halves(sms):
    """A graph large enough that the slot workspace exceeds 4 GiB at 8 slots per SM and halves (N >= 240 k on 132 SMs): 8-node paths,
    a star of 5000 leaves, a triangle in the last bitmap word.  2400 nodes over the id range, including the star's centre and leaves
    (2-hop sets of 5001)."""
    P, star = 8, 5000
    n_paths = 30000
    while khop_slots(n_paths * P + star + 4, sms)[0] == sms * 8:
        n_paths += 1000
    edges = []
    base = np.arange(n_paths, dtype=np.int64)[:, None] * P
    edges.append(np.stack([(base + np.arange(P - 1)).ravel(), (base + np.arange(1, P)).ravel()], 1))
    c0 = n_paths * P
    edges.append(np.stack([np.full(star, c0), c0 + 1 + np.arange(star)], 1))
    t0 = c0 + 1 + star
    N = t0 + 3
    edges.append(np.array([[t0, t0 + 1], [t0 + 1, t0 + 2], [t0, t0 + 2]]))
    rowptr, col = O.csr_from_edges(N, np.concatenate(edges))
    slots, full = khop_slots(N, sms)
    assert slots < full and (N - 1) // 32 == t0 // 32
    A = sp.csr_matrix((np.ones(len(col)), col, rowptr), shape=(N, N))
    rng = np.random.default_rng(1)
    nodes = np.concatenate([rng.choice(c0, 2380, replace=False), [c0, c0 + 1, c0 + star, t0, N - 1],
                            c0 + 1 + rng.choice(star, 15, replace=False)]).astype(np.int32)
    rng.shuffle(nodes)
    assert len(nodes) > 4 * slots
    fx = util.load_fixture("syn1")
    g = types.SimpleNamespace(rowptr=rowptr, col=col, feat=np.zeros((N, fx.feat.shape[1]), np.float32), label=np.zeros(N, np.int32),
                              pred_label=np.zeros(N, np.int32))
    eng = engine(g, fx.weights)
    try:
        for k in (2, 3):
            cnt = eng.count_nodes(nodes, k)
            plan = eng.plan_nodes(nodes, k)
            assert max(plan.n(t) for t in range(plan.count)) == star + 1
            check_plan(A, nodes, k, plan, cnt)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ shared-memory node classes 0..4
_CLASS_CACHE = {}


def class_members():
    """{class: (fixture, [golden nodes])} for the shared-memory classes: each node's class planned alone, the fixture with most nodes."""
    if _CLASS_CACHE:
        return _CLASS_CACHE
    found = {}
    for name in ("syn1", "syn4", "rand"):
        fx = util.load_fixture(name)
        eng = engine(fx, fx.weights)
        try:
            for v in fx.nodes:
                eng.plan_nodes([v], 3)
                c = int(np.argmax(eng.plan_class_counts()[0]))
                found.setdefault(c, {}).setdefault(name, []).append(v)
        finally:
            eng.close()
    for c in range(5):
        name = max(found[c], key=lambda f: len(found[c][f]))
        _CLASS_CACHE[c] = (name, found[c][name])
    return _CLASS_CACHE


def smem_case(c, sms):
    """The union of class c: up to three golden nodes of one fixture (smallest, middle, largest), K copies so that the class holds
    2.5 x its resident grid."""
    name, nodes = class_members()[c]
    fx = util.load_fixture(name)
    comps = {v: component(fx.rowptr, fx.col, fx.feat, fx.label, fx.pred_label, v, 3) for v in nodes}
    nodes = sorted(nodes, key=lambda v: (comps[v].e, v))
    pick = sorted({nodes[0], nodes[len(nodes) // 2], nodes[-1]}, key=nodes.index)
    K = math.ceil(2.5 * sms * SMEM_CTAS[c] / len(pick))
    g = union([comps[v] for v in pick], K)
    return fx, pick, g


def golden_m0(fx, nodes, K):
    return np.tile(np.concatenate([fx.gold["n%d_m0" % v] for v in nodes]).astype(np.float32), K)


def ex_outputs(eng, plan, hp, m0, d, C):
    cnt = plan.count
    o = dict(mask=np.zeros(plan.total_edges, np.float32), feat=np.zeros((cnt, d), np.float32),
             trace=np.zeros((cnt, hp.num_epochs, _abi.GX_TRACE_COLS), np.float32), trace_pred=np.zeros((cnt, hp.num_epochs, C), np.float32))
    so = dict(M=np.zeros(plan.total_edges, np.float32), m=np.zeros(plan.total_edges, np.float32), v=np.zeros(plan.total_edges, np.float32),
              feat=np.zeros((cnt, 3, d), np.float32))
    eng.explain_nodes_ex(hp, m0, o["mask"], o["feat"], trace=o["trace"], trace_pred=o["trace_pred"], state_out=so)
    o.update({"state_" + k: v for k, v in so.items()})
    return o


@pytest.mark.parametrize("c", range(5))
def test_shared_memory_class_past_its_grid(c, sms):
    fx, pick, g = smem_case(c, sms)
    K, d, C = g.K, fx.feat.shape[1], fx.weights["Wp"].shape[0]
    roots = g.roots.ravel()
    eng = engine(g, fx.weights)
    generic = None
    try:
        generic = engine(g, fx.weights, generic=True)
        plan = eng.plan_nodes(roots, 3)
        counts = eng.plan_class_counts()[0]
        assert counts[c] >= 2 * sms * SMEM_CTAS[c] and counts[5:].sum() == 0, (c, counts)
        m0 = golden_m0(fx, pick, K)
        assert len(m0) == plan.total_edges
        hp = eng.make_hparams()
        out = np.zeros(plan.total_edges, np.float32); fm = np.zeros((plan.count, d), np.float32)
        eng.explain_nodes_host(hp, m0, out, fm)
        ex = ex_outputs(eng, plan, hp, m0, d, C)
        grad = np.zeros(plan.total_edges, np.float32)
        eng.grad_nodes_host(grad)
        generic.plan_nodes(roots, 3)
        assert np.array_equal(generic.plan_class_counts()[0], counts)
        gout = np.zeros(plan.total_edges, np.float32); gfm = np.zeros((plan.count, d), np.float32)
        generic.explain_nodes_host(generic.make_hparams(), m0, gout, gfm)
        # copy 0 alone: one task per CTA
        p0 = eng.plan_nodes(g.roots[0], 3)
        assert p0.count <= sms
        m00 = m0[:p0.total_edges]
        a_out = np.zeros(p0.total_edges, np.float32); a_fm = np.zeros((p0.count, d), np.float32)
        eng.explain_nodes_host(hp, m00, a_out, a_fm)
        a_ex = ex_outputs(eng, p0, hp, m00, d, C)
        a_grad = np.zeros(p0.total_edges, np.float32)
        eng.grad_nodes_host(a_grad)
        assert_copies(out, a_out, K, "mask"); assert_copies(fm, a_fm, K, "feature mask")
        for key in ex:
            assert_copies(ex[key], a_ex[key], K, "explain_nodes_ex " + key)
        assert_copies(grad, a_grad, K, "gradient baseline")
        assert_copies(gout, a_out, K, "run-time-shape code"); assert_copies(gfm, a_fm, K, "run-time-shape feature mask")
        # the last copy of every component against the reference golden
        tol = util.node_tolerances(fx.name, 100)
        last = per_copy(out, K)[-1]
        eo = p0.edge_off
        for t, v in enumerate(pick):
            err = util.rel_l2(seg(last, eo, t), fx.gold["n%d_mask" % v])
            assert err <= tol[v], (c, v, err, tol[v])
        # and the last copy of the smallest component against the torch port and the fp64 closed form, 30 epochs
        eng.plan_nodes(roots, 3)
        out30 = np.zeros(plan.total_edges, np.float32); fm30 = np.zeros((plan.count, d), np.float32)
        eng.explain_nodes_host(eng.make_hparams(num_epochs=30), m0, out30, fm30)
    finally:
        eng.close()
        if generic is not None:
            generic.close()
    v = pick[0]
    idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(fx.rowptr, fx.col, fx.feat, fx.label, v, 3)
    Asub = O.dense_from_csr(srp, scol)
    M0 = np.zeros(Asub.shape, np.float32)          # entries off the sub-adjacency never reach an edge value
    M0[np.nonzero(Asub)] = fx.gold["n%d_m0" % v]
    args = (Asub, sfeat, slabel[idx], fx.pred_label[nbrs], idx, fx.weights, M0)
    ref = O.explain_dense_torch(*args, hp=O.default_hparams(num_epochs=30))
    c64 = O.explain_closed_form(*args, hp=O.default_hparams(num_epochs=30))
    dis = O.rel_l2(c64, ref)
    t_last = plan.count - len(pick)
    got = plan.dense_of(t_last, out30)
    assert O.rel_l2(got, ref) <= max(1e-4, 3 * dis), (c, v, O.rel_l2(got, ref), dis)
    _, st = O.explain_closed_form(*args, hp=O.default_hparams(num_epochs=29), return_state=True)
    assert np.abs(fm30[t_last] - 1 / (1 + np.exp(-st["F"]))).max() < max(2e-4, 30 * dis), (c, v)


# ------------------------------------------------------------------------------------------------ variant kernel, node mode
def random_model(rng, d, hid, emb, C, L, att=False, head=None):
    """Weights whose pre-activations stay O(1) at any width; att: Wa1 .. WaL; head: hidden widths of an MLP prediction head."""
    dims = [d] + [hid] * (L - 1) + [emb]
    w = {}
    for l in range(1, L + 1):
        w["W%d" % l] = (rng.normal(size=(dims[l - 1], dims[l])) * 1.5 / np.sqrt(dims[l - 1])).astype(np.float32)
        w["b%d" % l] = (rng.normal(size=dims[l]) * 0.3).astype(np.float32)
        if att:
            w["Wa%d" % l] = (rng.normal(size=(dims[l - 1], dims[l - 1])) / np.sqrt(dims[l - 1])).astype(np.float32)
    fan = hid * (L - 1) + emb
    if head:
        w["head"] = []
        for h in head:
            w["head"].append(((rng.normal(size=(h, fan)) * 1.5 / np.sqrt(fan)).astype(np.float32), (rng.normal(size=h) * 0.3).astype(np.float32)))
            fan = h
    w["Wp"] = (rng.normal(size=(C, fan)) * 0.5).astype(np.float32)
    w["bp"] = (rng.normal(size=C) * 0.3).astype(np.float32)
    return w


# name: seed, L, bn, att, hid, emb, d, C, head widths, optimiser
VAR_CASES = {"bn_L4": (1, 4, True, False, 20, 20, 7, 3, None, "adam"), "att": (2, 3, False, True, 20, 20, 8, 3, None, "adam"),
             "head": (3, 3, False, False, 20, 20, 10, 4, [50], "rmsprop"), "wide_input": (4, 3, False, False, 40, 40, 300, 3, None, "adam"),
             "width_160": (5, 3, True, False, 160, 160, 10, 4, None, "sgd")}
VAR_ROOTS = [0, 7, 23, 47]


@pytest.mark.parametrize("name", list(VAR_CASES))
def test_variant_kernel_node_queue_past_its_grid(name, sms):
    import networkx as nx
    seed, L, bn, att, hid, emb, d, C, head, opt = VAR_CASES[name]
    rng = np.random.default_rng(seed)
    N = 48
    rowptr, col = O.csr_from_edges(N, np.array(nx.barabasi_albert_graph(N, 2, seed=seed).edges(), dtype=np.int64))
    feat = rng.normal(size=(N, d)).astype(np.float32)
    label = rng.integers(0, C, N).astype(np.int32)
    w = random_model(rng, d, hid, emb, C, L, att, head)
    pred_label = np.argmax(O.model_pred(O.dense_from_csr(rowptr, col), feat, w, bn=bn), 1).astype(np.int32)
    comps = [component(rowptr, col, feat, label, pred_label, v, L) for v in VAR_ROOTS]
    K = 520
    g = union(comps, K)
    eng = engine(g, w, L, bn, att=[w["Wa%d" % l] for l in range(1, L + 1)] if att else None, head=w.get("head"))
    try:
        roots = g.roots.ravel()
        plan = eng.plan_nodes(roots, L)
        assert plan.count >= 2 * SLAB_CTAS * sms and eng.plan_class_counts()[0][5] == plan.count
        dense = [O.draw_m0(c.n, seed=100 * seed + i) for i, c in enumerate(comps)]
        p0 = eng.plan_nodes(g.roots[0], L)
        m00 = packed(p0, dense)
        hp = eng.make_hparams(num_epochs=20, opt=_abi.GX_OPT[opt])
        a_out = np.zeros(p0.total_edges, np.float32); a_fm = np.zeros((p0.count, d), np.float32)
        eng.explain_nodes_host(hp, m00, a_out, a_fm)
        eng.plan_nodes(roots, L)
        out = np.zeros(plan.total_edges, np.float32); fm = np.zeros((plan.count, d), np.float32)
        eng.explain_nodes_host(hp, np.tile(m00, K), out, fm)
    finally:
        eng.close()
    assert_copies(out, a_out, K, name); assert_copies(fm, a_fm, K, name + " feature mask")
    last, lfm = per_copy(out, K)[-1], per_copy(fm, K)[-1].reshape(len(comps), d)
    for t, c in enumerate(comps):
        A = O.dense_from_csr(c.rowptr, c.col)
        port_check(p0.dense_of(t, last), lfm[t], (A, c.feat, int(c.label[c.root]), c.pred_label, c.root, w, dense[t]),
                   dict(hp=O.default_hparams(num_epochs=20, opt=opt), bn=bn))


def test_variant_kernel_sgd_on_the_default_model_past_its_grid(sms):
    """--opt sgd on the default model (every task on the variant kernel) against the reference's own SGD masks (opts_golden.npz)."""
    fx = util.load_fixture("rand")
    og = np.load(util.GOLDEN + "/opts_golden.npz")
    nodes = [int(v) for v in og["sgd_nodes"]]
    comps = [component(fx.rowptr, fx.col, fx.feat, fx.label, fx.pred_label, v, 3) for v in nodes]
    K = math.ceil(2.2 * SLAB_CTAS * sms / len(nodes))
    g = union(comps, K)
    eng = engine(g, fx.weights)
    try:
        hp = eng.make_hparams(num_epochs=int(og["num_epochs"]), opt=1)
        p0 = eng.plan_nodes(g.roots[0], 3)
        m00 = np.concatenate([fx.gold["n%d_m0" % v] for v in nodes]).astype(np.float32)
        a_out = np.zeros(p0.total_edges, np.float32)
        eng.explain_nodes_host(hp, m00, a_out)
        plan = eng.plan_nodes(g.roots.ravel(), 3)
        assert plan.count >= 2 * SLAB_CTAS * sms
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_host(hp, np.tile(m00, K), out)
    finally:
        eng.close()
    assert_copies(out, a_out, K, "sgd")
    last = per_copy(out, K)[-1]
    for t, v in enumerate(nodes):
        err = util.rel_l2(seg(last, p0.edge_off, t), og["sgd_n%d_mask" % v])
        assert err <= 1e-4, (v, err)


# ------------------------------------------------------------------------------------------------ unconstrained (explain_dense.cu)
def test_unconstrained_nodes_past_the_grid(sms):
    fx = util.load_fixture("syn1")
    sizes = {v: len(O.khop_walk_set(fx.rowptr, fx.col, v, 3)) for v in fx.nodes}
    nodes = sorted(fx.nodes, key=lambda v: (sizes[v], v))[:4]
    comps = [component(fx.rowptr, fx.col, fx.feat, fx.label, fx.pred_label, v, 3) for v in nodes]
    cap = sms * 2048 // VAR_THREADS
    K = math.ceil(2.1 * cap / len(nodes))
    g = union(comps, K)
    dense = [O.draw_m0(c.n, seed=40 + i) for i, c in enumerate(comps)]
    m00 = np.concatenate([M.ravel() for M in dense]).astype(np.float32)
    nn0 = sum(c.n * c.n for c in comps)
    eng = engine(g, fx.weights)
    try:
        hp = eng.make_hparams(num_epochs=20)
        C = fx.weights["Wp"].shape[0]
        p0 = eng.plan_nodes(g.roots[0], 3)
        a_out = np.zeros(p0.total_edges, np.float32); a_md = np.zeros(nn0, np.float32)
        a_tr = np.zeros((p0.count, 20, _abi.GX_TRACE_COLS), np.float32); a_tp = np.zeros((p0.count, 20, C), np.float32)
        eng.explain_nodes_unconstrained(hp, m00, a_out, a_md, a_tr, a_tp)
        plan = eng.plan_nodes(g.roots.ravel(), 3)
        assert plan.count >= 2 * cap
        out = np.zeros(plan.total_edges, np.float32); md = np.zeros(nn0 * K, np.float32)
        tr = np.zeros((plan.count, 20, _abi.GX_TRACE_COLS), np.float32); tp = np.zeros((plan.count, 20, C), np.float32)
        eng.explain_nodes_unconstrained(hp, np.tile(m00, K), out, md, tr, tp)
    finally:
        eng.close()
    assert_copies(out, a_out, K, "unconstrained mask"); assert_copies(md, a_md, K, "mask_dense")
    assert_copies(tr, a_tr, K, "unconstrained trace"); assert_copies(tp, a_tp, K, "unconstrained trace_pred")
    assert np.isfinite(a_tr).all() and np.abs(a_tr).max() > 0
    last, lmd = per_copy(out, K)[-1], per_copy(md, K)[-1]
    o = 0
    for t, c in enumerate(comps):
        A = O.dense_from_csr(c.rowptr, c.col)
        D = lmd[o:o + c.n * c.n].reshape(c.n, c.n); o += c.n * c.n
        got = p0.dense_of(t, last)
        r, cc = np.nonzero(A)
        assert np.abs(D[r, cc] - got[r, cc]).max() <= 1e-6 and np.all(np.diag(D) == 0)
        port_check(got, None, (A, c.feat, int(c.label[c.root]), c.pred_label, c.root, fx.weights, dense[t]),
                   dict(hp=O.default_hparams(num_epochs=20), unconstrained=True))


# ------------------------------------------------------------------------------------------------ graph mode: variant and dense kernels
def graph_batch(K):
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    G = int(gg["num_graphs"])
    return gg, G, np.tile(gg["adj"], (K, 1, 1)), np.tile(gg["feat"], (K, 1, 1)), np.tile(gg["label"], K)


@pytest.mark.parametrize("tag", ["bn_L4", "rmsprop"])
def test_graph_variant_kernel_past_its_grid(tag, sms):
    gv = np.load(util.GOLDEN + "/graph_variants_golden.npz")
    cap = sms * 2048 // VAR_THREADS
    gg, G, adj, feat, label = graph_batch(math.ceil(2.1 * cap / 12))
    if tag == "rmsprop":
        w, L, bn, over = {k: gg[k] for k in util.WKEYS}, 3, False, dict(opt=2)
    else:
        L = int(gv[tag + "_L"])
        w = {k: gv["%s_%s" % (tag, k)] for k in ["W%d" % l for l in range(1, L + 1)] + ["b%d" % l for l in range(1, L + 1)] + ["Wp", "bp"]}
        bn, over = bool(gv[tag + "_bn"]), {}
    eng = graph_engine(w, adj, feat, label, L, bn)
    E = int(gv["num_epochs"])
    try:
        hp = eng.make_hparams(num_epochs=E, **over)
        m00 = np.concatenate([gg["g%d_m0" % g] for g in range(G)]).astype(np.float32)
        d = feat.shape[2]
        eo0 = eng.plan_graphs(list(range(G)))
        a_out = np.zeros(int(eo0[-1]), np.float32); a_fm = np.zeros((G, d), np.float32)
        eng.explain_graphs_host(hp, m00, a_out, a_fm)
        gids = list(range(adj.shape[0]))
        assert len(gids) >= 2 * cap
        eo = eng.plan_graphs(gids)
        out = np.zeros(int(eo[-1]), np.float32); fm = np.zeros((len(gids), d), np.float32)
        eng.explain_graphs_host(hp, np.tile(m00, len(gids) // G), out, fm)
    finally:
        eng.close()
    K = len(gids) // G
    assert_copies(out, a_out, K, tag); assert_copies(fm, a_fm, K, tag + " feature mask")
    last = per_copy(out, K)[-1]
    for g in range(G):
        err = util.rel_l2(seg(last, eo0, g), gv["%s_g%d_mask" % (tag, g)])
        tol = max(1e-4, 3 * float(gv[tag + "_spread"][g]))
        assert err <= tol, (tag, g, err, tol)


def test_unconstrained_graphs_past_the_grid(sms):
    cap = sms * 2048 // VAR_THREADS
    gg, G, adj, feat, label = graph_batch(math.ceil(2.1 * cap / 12))
    w = {k: gg[k] for k in util.WKEYS}
    n = adj.shape[1]
    dense = [O.draw_m0(n, seed=int(gg["g%d_seed" % g])) for g in range(G)]
    m00 = np.concatenate([M.ravel() for M in dense]).astype(np.float32)
    C = gg["Wp"].shape[0]
    eng = graph_engine(w, adj, feat, label)
    try:
        hp = eng.make_hparams(num_epochs=20)
        eo0 = eng.plan_graphs(list(range(G)))
        a_out = np.zeros(int(eo0[-1]), np.float32); a_md = np.zeros(G * n * n, np.float32)
        a_tr = np.zeros((G, 20, _abi.GX_TRACE_COLS), np.float32); a_tp = np.zeros((G, 20, C), np.float32)
        eng.explain_graphs_unconstrained(hp, m00, a_out, a_md, a_tr, a_tp)
        rc = [eng.graph_rows_cols(g) for g in range(G)]
        gids = list(range(adj.shape[0]))
        assert len(gids) >= 2 * cap
        eo = eng.plan_graphs(gids)
        out = np.zeros(int(eo[-1]), np.float32); md = np.zeros(len(gids) * n * n, np.float32)
        tr = np.zeros((len(gids), 20, _abi.GX_TRACE_COLS), np.float32); tp = np.zeros((len(gids), 20, C), np.float32)
        eng.explain_graphs_unconstrained(hp, np.tile(m00, len(gids) // G), out, md, tr, tp)
    finally:
        eng.close()
    K = len(gids) // G
    assert_copies(out, a_out, K, "unconstrained graphs"); assert_copies(md, a_md, K, "unconstrained graphs mask_dense")
    assert_copies(tr, a_tr, K, "unconstrained graphs trace"); assert_copies(tp, a_tp, K, "unconstrained graphs trace_pred")
    assert np.isfinite(a_tr).all() and np.abs(a_tr).max() > 0
    last, lmd = per_copy(out, K)[-1], per_copy(md, K)[-1].reshape(G, n, n)
    for g in range(0, G, 3):
        got = np.zeros((n, n)); got[rc[g]] = seg(last, eo0, g)
        assert np.abs(lmd[g][rc[g]] - got[rc[g]]).max() <= 1e-6
        port_check(got, None, (np.asarray(gg["adj"][g], np.float64), gg["feat"][g], int(gg["label"][g]), None, 0, w, dense[g]),
                   dict(hp=O.default_hparams(num_epochs=20), graph_mode=True, unconstrained=True))


# ------------------------------------------------------------------------------------------------ grid-stride utility kernels
def syn1_union(K, count=6):
    """K copies of the 3-hop components of syn1's `count` smallest golden nodes."""
    fx = util.load_fixture("syn1")
    sizes = {v: len(O.khop_walk_set(fx.rowptr, fx.col, v, 3)) for v in fx.nodes}
    nodes = sorted(fx.nodes, key=lambda v: (sizes[v], v))[:count]
    comps = [component(fx.rowptr, fx.col, fx.feat, fx.label, fx.pred_label, v, 3) for v in nodes]
    return fx, union(comps, K)


def awkward_values(plan, rng):
    """Random per-task values: zeros, heavy ties on every 5th task, no positive value on every 7th."""
    v = rng.random(plan.total_edges).astype(np.float32)
    v[rng.random(plan.total_edges) < 0.1] = 0.0
    for t in range(0, plan.count, 5):
        s = slice(plan.edge_off[t], plan.edge_off[t + 1])
        v[s] = np.round(v[s] * 8) / 8
    for t in range(3, plan.count, 7):
        v[plan.edge_off[t]:plan.edge_off[t + 1]] = 0.0
    return v


def test_denoise_topk_past_the_grid():
    fx, g = syn1_union(400)
    eng = engine(g, fx.weights)
    try:
        plan = eng.plan_nodes(g.roots.ravel(), 3)
        assert plan.count > 2 * GRID_CAP
        v = awkward_values(plan, np.random.default_rng(3))
        vd = torch.from_numpy(v).cuda()
        rows_cols = [plan.rows_cols_of(t) for t in range(plan.count)]
        for k, cap in ((20, 64), (5, 3)):
            slot_res = eng.denoise_topk(v, k, cap=cap)
            edge_res = [eng.denoise_topk_edges(v, k, cap=cap), [x.cpu().numpy() for x in eng.denoise_topk_edges(vd, k, cap=cap)]]
            thr, cnt, slots, vals = slot_res
            for t in range(plan.count):
                x = seg(v, plan.edge_off, t)
                pos = x[x > 0]
                if len(pos) == 0:
                    assert cnt[t] == 0 and np.isinf(thr[t]) and (slots[t] == -1).all(), (k, t)
                    for e_thr, e_cnt, e_uv, e_vals in edge_res:
                        assert e_cnt[t] == 0 and np.isinf(e_thr[t]) and (e_uv[t] == -1).all() and (e_vals[t] == 0).all(), (k, t)
                    continue
                want_thr = np.sort(pos)[-min(len(pos), 2 * k)]
                keep = np.nonzero(x >= want_thr)[0]
                m = min(len(keep), cap)
                assert thr[t] == want_thr and cnt[t] == len(keep), (k, t)
                assert np.array_equal(slots[t, :m], keep[:m]) and np.array_equal(vals[t, :m], x[keep[:m]]) and (slots[t, m:] == -1).all(), (k, t)
                rows, cols = rows_cols[t]
                keep = np.nonzero((x >= want_thr) & (rows < cols))[0]
                m = min(len(keep), cap)
                nb = plan.neighbors_of(t)
                for e_thr, e_cnt, e_uv, e_vals in edge_res:
                    assert e_thr[t] == want_thr and e_cnt[t] == len(keep), (k, t)
                    assert np.array_equal(e_uv[t, :m], np.stack([nb[rows[keep[:m]]], nb[cols[keep[:m]]]], 1)), (k, t)
                    assert np.array_equal(e_vals[t, :m], x[keep[:m]]) and (e_uv[t, m:] == -1).all() and (e_vals[t, m:] == 0).all(), (k, t)
    finally:
        eng.close()


def test_densify_past_the_grid():
    fx, g = syn1_union(400)
    eng = engine(g, fx.weights)
    try:
        plan = eng.plan_nodes(g.roots.ravel(), 3)
        assert plan.count > 2 * GRID_CAP
        v = np.random.default_rng(4).random(plan.total_edges).astype(np.float32)
        nn = np.diff(plan.node_off).astype(np.int64) ** 2
        dense_off = np.concatenate([[0], np.cumsum(nn)])
        want = np.zeros(int(dense_off[-1]), np.float64)
        want[np.repeat(dense_off[:-1], np.diff(plan.edge_off)) + plan.flat_index()] = v
        host = eng.densify_host(v, int(dense_off[-1]))
        dev = eng.densify_device(torch.from_numpy(v).cuda()).cpu().numpy()
    finally:
        eng.close()
    assert np.array_equal(host, want) and np.array_equal(dev, want)
    for t in (0, plan.count // 2, plan.count - 1):
        assert np.array_equal(host[dense_off[t]:dense_off[t + 1]].reshape(plan.n(t), plan.n(t)), plan.dense_of(t, v))


def test_densify_graphs_past_the_grid():
    gg, G, adj, feat, label = graph_batch(100)
    eng = graph_engine({k: gg[k] for k in util.WKEYS}, adj, feat, label)
    try:
        rng = np.random.default_rng(5)
        gids = rng.integers(0, adj.shape[0], 2 * GRID_CAP + 300).astype(np.int32)     # scrambled, with repeats
        rc = {int(x): eng.graph_rows_cols(int(x)) for x in np.unique(gids)}
        sizes = np.array([len(rc[int(x)][0]) for x in gids])
        vals = rng.random(int(sizes.sum())).astype(np.float32)
        n = adj.shape[1]
        want = np.zeros((len(gids), n, n))
        o = 0
        for i, x in enumerate(gids):
            want[i][rc[int(x)]] = vals[o:o + sizes[i]]; o += sizes[i]
        host = eng.densify_graphs_host(gids, vals)
        dev = eng.densify_graphs_device(gids, torch.from_numpy(vals).cuda()).cpu().numpy()
    finally:
        eng.close()
    assert np.array_equal(host, want) and np.array_equal(dev, want)


def test_unshard_past_the_grid():
    rng = np.random.default_rng(6)
    items = 2 * GRID_CAP + 500
    sizes = rng.integers(0, 40, items).astype(np.int32)
    sizes[::11] = 0
    dst = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    perm = rng.permutation(items)                        # the gathered buffer holds the items in another order, with gaps
    gaps = rng.integers(0, 5, items)
    starts = np.concatenate([[0], np.cumsum(sizes[perm] + gaps)[:-1]])
    src = np.empty(items, np.int64); src[perm] = starts
    gathered = rng.random(int(starts[-1] + sizes[perm[-1]] + gaps[-1]) + 1).astype(np.float32)
    want = np.concatenate([gathered[src[p]:src[p] + sizes[p]] for p in range(items)])
    eng = gnnx.Engine(0)
    try:
        out = torch.full((len(want) + 7,), -1.0, dtype=torch.float32, device="cuda")
        eng.unshard_masks(torch.from_numpy(gathered).cuda(), src, dst, sizes, out)
        eng.sync()
        got = out.cpu().numpy()
    finally:
        eng.close()
    assert np.array_equal(got[:len(want)], want) and (got[len(want):] == -1).all()


def test_explain_nodes_topk_chunks_past_the_grid(tmp_path, sms):
    fx, g = syn1_union(560)
    nodes = g.roots.ravel()
    assert len(nodes) > 3000 > sms
    args = types.SimpleNamespace(num_gc_layers=3, num_epochs=10, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                 mask_bias=False, gpu=False, bias=True, method="base", dataset="syn1", bmname=None, hidden_dim=20,
                                 output_dim=20, name_suffix="", explainer_suffix="", logdir=str(tmp_path), gnnx_init="device", gnnx_seed=5)
    model = gnnx.models.GcnEncoderNode(fx.feat.shape[1], 20, 20, fx.weights["Wp"].shape[0], 3, bn=False, args=args)
    sd = {"conv_first.weight": fx.weights["W1"], "conv_first.bias": fx.weights["b1"], "conv_block.0.weight": fx.weights["W2"],
          "conv_block.0.bias": fx.weights["b2"], "conv_last.weight": fx.weights["W3"], "conv_last.bias": fx.weights["b3"],
          "pred_model.weight": fx.weights["Wp"], "pred_model.bias": fx.weights["bp"]}
    model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    A = sp.csr_matrix((np.ones(len(g.col), np.float32), g.col, g.rowptr), shape=(g.N, g.N))
    ex = gnnx.Explainer(model=model, adj=A, feat=g.feat[None], label=g.label[None], pred=None, train_idx=[], args=args, writer=None,
                        print_training=False, graph_idx=-1)
    res = []
    try:
        for chunk in (sms, 3000, len(nodes)):
            thr, offsets, uv, vals = ex.explain_nodes_topk(nodes, chunk_size=chunk)
            res.append((thr.cpu().numpy(), np.asarray(offsets), uv.cpu().numpy(), vals.cpu().numpy()))
    finally:
        ex.engine.close()
    for r in res[1:]:
        for a, b in zip(r, res[0]):
            assert a.dtype == b.dtype and np.array_equal(a, b)
    assert int(res[0][1][-1]) > 0


# ------------------------------------------------------------------------------------------------ model forward
def test_model_forward_past_the_grid():
    fx = util.load_fixture("syn1")
    K = 16
    comp = types.SimpleNamespace(rowptr=fx.rowptr, col=fx.col, feat=fx.feat.astype(np.float32), label=fx.label.astype(np.int32),
                                 pred_label=fx.pred_label, root=0, n=fx.N, e=len(fx.col))
    g = union([comp], K)
    assert g.N > GRID_CAP * FWD_WARPS
    eng = engine(g, fx.weights)
    try:
        got = eng.model_forward().reshape(K, fx.N, -1)
    finally:
        eng.close()
    assert_copies(got, got[0], K, "logits")
    tol = 2e-5 * max(1.0, np.abs(fx.pred).max())
    assert np.abs(got[-1] - fx.pred).max() <= tol and np.array_equal(np.argmax(got[-1], 1), fx.pred_label)
