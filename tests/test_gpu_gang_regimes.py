"""GPU (-m gpu), one device: explain_gang.cu in the regimes its automatic gang policy picks for large natural subgraphs.

  A. the configs[4] step as `bench.py --workload c5` times it: 132 nodes of BA(100 000, 32), d = 128, 3-hop, 100 epochs, device Philox
     init, masks left on the device.  One gang of every SM takes all 132 tasks in turn in one slab, and the packed plan's offsets cross
     2^31 elements.  Every task against the same node explained alone, a second step against the first, the last task of the queue
     against the fp64 sparse spec, the planner against scipy and the top-k delivery against numpy;
  B. the two regimes between syn1 and configs[4]: one gang with many tasks (BA(40 000, 16)) and a few gangs of tens of CTAs with more
     tasks than gangs (BA(16 000, 8)), at 100 epochs with Philox and at 30 epochs with host M0.

A task's masks do not depend on its batch or its gang size, bit for bit (include/gnnx.h, DESIGN section 10.1).  Every test first asserts
the regime it exists for, from the planner's formula (csrc/node_mode.cu, explain_nodes_impl): a task's working set is 8 B per directed
edge + 240 B per node, as many gangs as fit 5/8 of the L2 with the largest of them, the SMs shared evenly among the gangs."""
import ctypes as C
import os
import sys
import time
import types

import numpy as np
import pytest
import scipy.sparse as sp
import torch
from scipy.sparse.csgraph import dijkstra

import gnnx
import gnnx_oracle as O
import kernel_spec as KS
import util
from gnnx import _abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import bench  # noqa: E402  (make_ba_csr: the c5 workload's graph generator)

pytestmark = pytest.mark.gpu

SLAB = 5                 # launch class of the slab kernels (gx_plan_class_counts)
LONG = 512               # kLongEdges of explain_gang.cu: rows with more induced edges are sliced over a CTA
MAX_GANG = 160           # GX_MAX_GANG (gnnx_internal.cuh)
HOPS, D, HID, C4 = 3, 128, 20, 4
SPEC_EPOCHS = 4


def _sig(x):
    return 1 / (1 + np.exp(-x))


def _device():
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, p.L2_cache_size


def _forward_pred(A, X, W):
    """pred_label of the default 3-layer model on the whole graph: the numpy forward of bench.py's c5 workload, operation for operation."""
    nrm = lambda Y: Y / np.maximum(np.linalg.norm(Y, axis=1, keepdims=True), 1e-12)
    H1 = np.maximum(nrm((A @ X) @ W["W1"] + W["b1"]), 0)
    H2 = np.maximum(nrm((A @ H1) @ W["W2"] + W["b2"]), 0)
    H3 = nrm((A @ H2) @ W["W3"] + W["b3"])
    return np.argmax(np.concatenate([H1, H2, H3], 1) @ W["Wp"].T + W["bp"], 1).astype(np.int32)


def _balls(A, nodes):
    """From the global graph alone, per node: n and E_d of its induced 3-hop ball, and n2 / e1 (the nodes within 2 hops and their
    directed entries: such a row has every neighbour inside the ball, so its induced degree is its degree)."""
    R = np.zeros((A.shape[0], len(nodes)), np.float64)
    R[np.asarray(nodes), np.arange(len(nodes))] = 1.0
    reach = [R]
    for _ in range(HOPS):
        reach.append(((A @ reach[-1]) + reach[-1] > 0).astype(np.float64))
    ball = reach[HOPS]
    deg = np.diff(A.indptr).astype(np.float64)
    as_int = lambda v: np.rint(v).astype(np.int64)
    return types.SimpleNamespace(n=as_int(ball.sum(0)), e_d=as_int((ball * (A @ ball)).sum(0)),
                                 n2=as_int(reach[HOPS - 1].sum(0)), e1=as_int(deg @ reach[HOPS - 1]))


def _gang_policy(n, e_d, sms, l2):
    """(ngangs, gang) the planner picks for a slab class of these tasks with the automatic gang size."""
    ws = max(1, int(np.max(8 * np.asarray(e_d, np.int64) + 240 * np.asarray(n, np.int64))))
    ngangs = max(1, min(min(len(n), sms), (l2 * 5 // 8) // ws))
    return ngangs, max(1, min(sms // ngangs, MAX_GANG))


def _queue(b):
    """Task order of the slab class's work queue: most expensive first by the planner's cost, ties in task order."""
    cost = b.e1 * (D + 2 * HID) + b.n2 * 600 + (b.e_d // 2) * 60
    return sorted(range(len(cost)), key=lambda t: -int(cost[t]))


def _exact_m0(eng, node, seed):
    """The float M0 that GX_INIT_PHILOX draws for `node` (planned alone): the mask parameter a one-epoch run reports before any update."""
    plan = eng.plan_nodes([int(node)], HOPS)
    M = np.zeros(plan.total_edges, np.float32)
    eng.explain_nodes_ex(eng.make_hparams(num_epochs=1, init=_abi.GX_INIT_PHILOX, seed=seed), None,
                         np.zeros(plan.total_edges, np.float32), state_out={"M": M})
    return plan, M


def _spec(plan, t, X, label, pred_label, W, m0, epochs):
    """fp64 sparse edge-list specification of task t of plan: (edge mask, F)."""
    rp, col = plan.csr_of(t)
    nb = plan.neighbors_of(t)
    node = int(plan.nodes[t])
    return KS.explain_pruned_edges_sparse(rp, col, X[nb], int(label[node]), pred_label[nb], int(plan.node_idx_new[t]), W, m0,
                                          num_epochs=epochs, return_F=True)


def _assert_spec(out, fm, ref, what):
    a, F = ref
    err = util.rel_l2(out, a)
    ferr = float(np.abs(np.asarray(fm, np.float64) - _sig(F)).max())
    print("%s: edge mask rel-L2 %.2e, feature mask max-abs %.2e vs the fp64 sparse spec" % (what, err, ferr))
    assert err <= 1e-5 and ferr <= 2e-5, (what, err, ferr)


# ------------------------------------------------------------------------------------------------ A. the configs[4] step
@pytest.fixture(scope="module")
def c5():
    """The inputs of bench.py's c5 workload, built as it builds them, on an engine bound to torch's stream; the batch planned (plan
    fetched to the host) and explained once at 100 epochs with the masks on the device."""
    t0 = time.perf_counter()
    N, m, K = 100000, 32, 132
    rng = np.random.default_rng(0)
    rowptr, col = bench.make_ba_csr(N, m, 0)
    X = rng.normal(size=(N, D)).astype(np.float32)
    label = rng.integers(0, C4, N).astype(np.int32)
    sc = lambda *s_: (rng.normal(size=s_) * 0.3).astype(np.float32)
    W = dict(W1=sc(D, 20), b1=sc(20), W2=sc(20, 20), b2=sc(20), W3=sc(20, 20), b3=sc(20), Wp=sc(C4, 60), bp=sc(C4))
    A = sp.csr_matrix((np.ones(len(col), np.float32), col, rowptr), shape=(N, N))
    pred_label = _forward_pred(A, X, W)
    nodes = np.random.default_rng(1).permutation(N)[:K].astype(np.int32)
    balls = _balls(A, nodes)
    te, tn = int(balls.e_d.sum()), int(balls.n.sum())
    # the plan's arrays (sub_col, icol / cs2is / is2cs, six pair arrays: 28 B per slot; four node arrays), two mask outputs, 1 GB for
    # the slab, the pair slab and the k-hop workspace
    need = 28 * te + 16 * (tn + K) + 2 * 4 * te + (1 << 30)
    free = torch.cuda.mem_get_info(0)[0]
    if free < need:
        pytest.skip("configs[4] batch needs about %.1f GB of device memory, %.1f GB are free" % (need / 1e9, free / 1e9))
    eng = gnnx.Engine(0)
    eng.follow_torch_stream()
    eng.set_model(W)
    eng.set_graph_csr(rowptr, col, X, label, pred_label)
    counts = eng.count_nodes(nodes, HOPS)           # (before the plan: gx_count_nodes shares the handle's task buffer with it)
    hp = eng.make_hparams(num_epochs=100, init=_abi.GX_INIT_PHILOX, seed=99)
    plan = eng.plan_nodes(nodes, HOPS)
    class_counts = eng.plan_class_counts()[0]
    dev = torch.device("cuda", 0)
    out = torch.empty(plan.total_edges, dtype=torch.float32, device=dev)
    fm = torch.empty((K, D), dtype=torch.float32, device=dev)
    eng.explain_nodes_ptr(hp, _abi.GX_DEVICE, 0, out.data_ptr(), fm.data_ptr())
    torch.cuda.synchronize()
    print("configs[4] batch: inputs, plan and the 100-epoch step in %.1f s" % (time.perf_counter() - t0))
    s = types.SimpleNamespace(N=N, K=K, A=A, rowptr=rowptr, col=col, X=X, label=label, W=W, pred_label=pred_label, nodes=nodes,
                              balls=balls, counts=counts, eng=eng, hp=hp, plan=plan, class_counts=class_counts, out=out, fm=fm,
                              batch_planned=True)
    yield s
    eng.close()


def _replan(c5):
    """Put the batch plan back on the handle (tests that plan single nodes take it away)."""
    if not c5.batch_planned:
        c5.eng.plan_nodes(c5.nodes, HOPS, fetch=False)
        c5.batch_planned = True


def test_c5_regime(c5):
    """configs[4] is one gang of every SM taking all 132 tasks in one slab, with the packed offsets past 2^31 elements."""
    sms, l2 = _device()
    b, plan = c5.balls, c5.plan
    n = np.diff(plan.node_off)
    e_d = np.diff(plan.edge_off)
    ngangs, gang = _gang_policy(n, e_d, sms, l2)
    long_rows = sum(int((np.diff(plan.csr_of(t)[0]) > LONG).sum()) for t in range(plan.count))
    print("configs[4]: %d tasks, n %d .. %d, sum E_d %d (3 E_d = %.2f G int32s, 6 x %d pairs = %.2f G int32s), predicted ngangs %d x gang %d, "
          "%d rows over %d edges" % (plan.count, n.min(), n.max(), plan.total_edges, 3 * plan.total_edges / 1e9, plan.total_edges // 2,
                                    6 * (plan.total_edges // 2) / 1e9, ngangs, gang, long_rows, LONG))
    assert c5.class_counts[SLAB] == c5.K and c5.class_counts.sum() == c5.K, c5.class_counts
    assert n.min() >= 90000
    assert 3 * plan.total_edges > 2 ** 31 and 6 * (plan.total_edges // 2) > 2 ** 31
    assert (ngangs, gang) == (1, min(sms, MAX_GANG)) and gang == sms
    assert np.array_equal(n, b.n) and np.array_equal(e_d, b.e_d)


def test_c5_planner_matches_scipy(c5):
    """gx_count_nodes for all 132 nodes, and the plan of the first, the last, the largest and the smallest task (neighbours, sub-CSR,
    the node's position) against scipy's 3-hop ball and induced sub-adjacency, bit for bit."""
    plan, b = c5.plan, c5.balls
    assert np.array_equal(c5.counts[0], b.n) and np.array_equal(c5.counts[1], b.e_d)
    n = np.diff(plan.node_off)
    picks = sorted({0, plan.count - 1, int(np.argmax(n)), int(np.argmin(n))})
    for t in picks:
        node = int(c5.nodes[t])
        ball = np.nonzero(np.isfinite(dijkstra(c5.A, indices=node, unweighted=True, limit=HOPS + 0.5)))[0]
        assert np.array_equal(plan.neighbors_of(t), ball), node
        assert int(plan.node_idx_new[t]) == int(np.searchsorted(ball, node)), node
        sub = c5.A[ball][:, ball].tocsr()
        sub.sort_indices()
        rp, col = plan.csr_of(t)
        assert np.array_equal(rp, sub.indptr) and np.array_equal(col, sub.indices), node
    print("configs[4] planner: counts of %d tasks, plans of tasks %s (n %s) match scipy" % (plan.count, picks, [int(n[t]) for t in picks]))


def test_c5_topk_delivery(c5):
    """gx_denoise_topk and gx_denoise_topk_edges (threshold_num 20) on the device-resident 100-epoch masks of all 132 tasks against numpy
    on each task's slice: the threshold, the count, the kept slots and values, and the row < col half in global ids."""
    _replan(c5)
    eng, plan, K = c5.eng, c5.plan, c5.K
    k, cap, cap_e = 20, 2 * 20 + 16, 20 + 16
    dev = c5.out.device
    thr = torch.empty(K, dtype=torch.float32, device=dev)
    cnt = torch.empty(K, dtype=torch.int32, device=dev)
    slots = torch.empty((K, cap), dtype=torch.int32, device=dev)
    vals = torch.empty((K, cap), dtype=torch.float32, device=dev)
    _abi.check(eng._lib.gx_denoise_topk(eng._h, _abi.GX_DEVICE, C.c_void_p(c5.out.data_ptr()), k, cap, C.c_void_p(thr.data_ptr()),
                                        C.c_void_p(cnt.data_ptr()), C.c_void_p(slots.data_ptr()), C.c_void_p(vals.data_ptr())))
    thr_e, cnt_e, uv, vals_e = eng.denoise_topk_edges(c5.out, k, cap=cap_e)
    torch.cuda.synchronize()
    thr, cnt, slots, vals = (x.cpu().numpy() for x in (thr, cnt, slots, vals))
    thr_e, cnt_e, uv, vals_e = (x.cpu().numpy() for x in (thr_e, cnt_e, uv, vals_e))
    for t in range(K):
        v = c5.out[plan.edge_off[t]:plan.edge_off[t + 1]].cpu().numpy()
        pos = v[v > 0]
        want = min(2 * k, len(pos))
        th = np.partition(pos, len(pos) - want)[len(pos) - want]
        kept = np.nonzero(v >= th)[0]
        node = int(c5.nodes[t])
        assert thr[t] == th and thr_e[t] == th, (node, thr[t], thr_e[t], th)
        assert cnt[t] == len(kept), (node, cnt[t], len(kept))
        m = min(len(kept), cap)
        assert np.array_equal(slots[t, :m], kept[:m]) and (slots[t, m:] == -1).all(), node
        assert np.array_equal(vals[t, :m], v[kept[:m]]), node
        rp, col = plan.csr_of(t)
        rows = np.searchsorted(rp, kept, side="right") - 1
        half = kept[rows < col[kept]]
        hr = np.searchsorted(rp, half, side="right") - 1
        nb = plan.neighbors_of(t)
        assert cnt_e[t] == len(half), (node, cnt_e[t], len(half))
        me = min(len(half), cap_e)
        assert np.array_equal(uv[t, :me, 0], nb[hr[:me]]) and np.array_equal(uv[t, :me, 1], nb[col[half[:me]]]), node
        assert np.array_equal(vals_e[t, :me], v[half[:me]]), node
    print("configs[4] top-k: %d tasks, kept %d .. %d directed slots, %d .. %d edges" % (K, cnt.min(), cnt.max(), cnt_e.min(), cnt_e.max()))


def test_c5_second_step_is_bit_identical(c5):
    """Planning and explaining the batch again on the same handle, as the bench's timed loop does, gives the same bits."""
    eng = c5.eng
    eng.plan_nodes(c5.nodes, HOPS, fetch=False)
    c5.batch_planned = True
    out2 = torch.empty_like(c5.out)
    fm2 = torch.empty_like(c5.fm)
    eng.explain_nodes_ptr(c5.hp, _abi.GX_DEVICE, 0, out2.data_ptr(), fm2.data_ptr())
    torch.cuda.synchronize()
    assert torch.equal(out2, c5.out) and torch.equal(fm2, c5.fm)


def test_c5_batch_is_each_node_alone(c5):
    """Every one of the 132 tasks, taken in turn by one gang in one slab, has the edge and feature masks of its node explained alone on
    the same handle (Philox is keyed by the node id: the same M0)."""
    eng, plan = c5.eng, c5.plan
    e_d = np.diff(plan.edge_off)
    dev = c5.out.device
    o1 = torch.empty(int(e_d.max()), dtype=torch.float32, device=dev)
    f1 = torch.empty((1, D), dtype=torch.float32, device=dev)
    c5.batch_planned = False
    for t, node in enumerate(c5.nodes):
        eng.plan_nodes([int(node)], HOPS, fetch=False)
        assert eng._plan_sizes[2] == e_d[t], int(node)
        eng.explain_nodes_ptr(c5.hp, _abi.GX_DEVICE, 0, o1.data_ptr(), f1.data_ptr())
        same = torch.equal(o1[:e_d[t]], c5.out[plan.edge_off[t]:plan.edge_off[t + 1]]) and torch.equal(f1[0], c5.fm[t])
        assert same, (t, int(node))


def test_c5_last_task_matches_spec(c5):
    """The task the gang takes last (the queue is largest-first: the cheapest task) at 4 epochs of the batch against the fp64 sparse
    spec, started from the exact float M0 the kernel drew."""
    eng, plan, b = c5.eng, c5.plan, c5.balls
    order = _queue(b)
    last = order[-1]
    node = int(c5.nodes[last])
    _replan(c5)
    out4 = torch.empty_like(c5.out)
    fm4 = torch.empty_like(c5.fm)
    eng.explain_nodes_ptr(eng.make_hparams(num_epochs=SPEC_EPOCHS, init=_abi.GX_INIT_PHILOX, seed=99), _abi.GX_DEVICE, 0, out4.data_ptr(),
                          fm4.data_ptr())
    torch.cuda.synchronize()
    got = out4[plan.edge_off[last]:plan.edge_off[last + 1]].cpu().numpy()
    got_f = fm4[last].cpu().numpy()
    del out4, fm4
    p1, M0 = _exact_m0(eng, node, 99)
    c5.batch_planned = False
    assert np.array_equal(p1.neighbors_of(0), plan.neighbors_of(last))
    drift = float(np.abs(M0 - O.philox_m0(99, node, len(M0), p1.n(0))).max())
    t0 = time.perf_counter()
    ref = _spec(plan, last, c5.X, c5.label, c5.pred_label, c5.W, M0, SPEC_EPOCHS)
    print("configs[4] last task: node %d, n %d, E_d %d, queue position %d of %d; kernel M0 vs fp64 Philox max-abs %.1e; spec %.1f s"
          % (node, plan.n(last), len(M0), order.index(last), plan.count, drift, time.perf_counter() - t0))
    _assert_spec(got, got_f, ref, "configs[4] node %d" % node)


# ------------------------------------------------------------------------------------------------ B. the regimes below configs[4]
REGIMES = {   # name: (N, m, tasks, graph seed)
    "one_gang": (40000, 16, 24, 3),
    "few_gangs": (16000, 8, 40, 4),
}


@pytest.fixture(scope="module")
def graphs():
    cache = {}

    def get(name):
        if name not in cache:
            N, m, K, seed = REGIMES[name]
            rng = np.random.default_rng(seed)
            rowptr, col = bench.make_ba_csr(N, m, seed)
            X = rng.normal(size=(N, D)).astype(np.float32)
            label = rng.integers(0, C4, N).astype(np.int32)
            sc = lambda *s_: (rng.normal(size=s_) * 0.5).astype(np.float32)
            W = dict(W1=sc(D, HID), b1=sc(HID), W2=sc(HID, HID), b2=sc(HID), W3=sc(HID, HID), b3=sc(HID), Wp=sc(C4, 3 * HID), bp=sc(C4))
            A = sp.csr_matrix((np.ones(len(col), np.float32), col, rowptr), shape=(N, N))
            nodes = rng.permutation(N)[:K].astype(np.int32)
            cache[name] = types.SimpleNamespace(N=N, rowptr=rowptr, col=col, X=X, label=label, W=W, A=A, nodes=nodes,
                                                pred_label=_forward_pred(A, X, W), balls=_balls(A, nodes))
        return cache[name]
    return get


def _explain_host(eng, hp, m0, E, K):
    out = np.zeros(E, np.float32)
    fm = np.zeros((K, D), np.float32)
    eng.explain_nodes_host(hp, m0, out, fm)
    return out, fm


@pytest.mark.parametrize("init", ["philox", "host_m0"])
@pytest.mark.parametrize("regime", list(REGIMES))
def test_gang_regime_batch_is_alone_and_matches_spec(graphs, regime, init):
    """The automatic gang policy on a batch of large natural subgraphs: every task's masks equal its node explained alone (one gang of
    every SM) bit for bit, at 100 epochs with Philox or at 30 with host M0; the task queued last against the fp64 sparse spec at 4 epochs."""
    g = graphs(regime)
    sms, l2 = _device()
    K = len(g.nodes)
    philox = init == "philox"
    epochs, seed = (100, 7) if philox else (30, 8)
    eng = gnnx.Engine(0)
    eng.set_model(g.W)
    eng.set_graph_csr(g.rowptr, g.col, g.X, g.label, g.pred_label)
    plan = eng.plan_nodes(g.nodes, HOPS)
    counts = eng.plan_class_counts()[0]
    assert counts[SLAB] == K and counts.sum() == K, counts
    n, e_d = np.diff(plan.node_off), np.diff(plan.edge_off)
    assert np.array_equal(n, g.balls.n) and np.array_equal(e_d, g.balls.e_d)
    ngangs, gang = _gang_policy(n, e_d, sms, l2)
    order = _queue(g.balls)
    long_rows = [int((np.diff(plan.csr_of(t)[0]) > LONG).sum()) for t in range(K)]
    reused = order[ngangs:]                   # the tasks a gang takes after its first, in the slab its previous task left behind
    print("%s: %d tasks, n %d .. %d, E_d %d .. %d, predicted ngangs %d x gang %d, rows over %d edges per task %d .. %d (%d in reused slabs)"
          % (regime, K, n.min(), n.max(), e_d.min(), e_d.max(), ngangs, gang, LONG, min(long_rows), max(long_rows),
             sum(long_rows[t] for t in reused)))
    if regime == "one_gang":
        assert ngangs == 1 and gang == min(sms, MAX_GANG) and K >= 16
    else:
        assert 2 <= ngangs <= sms // 10 and gang >= 10 and K >= 2 * ngangs
    assert any(long_rows[t] > 0 for t in reused)
    if philox:
        hp = eng.make_hparams(num_epochs=epochs, init=_abi.GX_INIT_PHILOX, seed=seed)
        m0 = None
    else:
        hp = eng.make_hparams(num_epochs=epochs)
        m0 = _edge_m0(plan, seed)
    t0 = time.perf_counter()
    out, fm = _explain_host(eng, hp, m0, plan.total_edges, K)
    for t, node in enumerate(g.nodes):
        eng.plan_nodes([int(node)], HOPS, fetch=False)
        assert eng._plan_sizes[2] == e_d[t], (regime, t, int(node))
        o1, f1 = _explain_host(eng, hp, None if m0 is None else m0[plan.edge_off[t]:plan.edge_off[t + 1]], int(e_d[t]), 1)
        assert np.array_equal(o1, out[plan.edge_off[t]:plan.edge_off[t + 1]]) and np.array_equal(f1[0], fm[t]), (regime, t, int(node))
    batch_s = time.perf_counter() - t0
    # the task queued last, at 4 epochs of the batch, against the spec from the exact M0
    last = order[-1]
    node = int(g.nodes[last])
    if philox:
        _, M0 = _exact_m0(eng, node, seed)
        hp4 = eng.make_hparams(num_epochs=SPEC_EPOCHS, init=_abi.GX_INIT_PHILOX, seed=seed)
    else:
        M0 = m0[plan.edge_off[last]:plan.edge_off[last + 1]]
        hp4 = eng.make_hparams(num_epochs=SPEC_EPOCHS)
    eng.plan_nodes(g.nodes, HOPS, fetch=False)
    out4, fm4 = _explain_host(eng, hp4, m0, plan.total_edges, K)
    eng.close()
    t1 = time.perf_counter()
    ref = _spec(plan, last, g.X, g.label, g.pred_label, g.W, M0, SPEC_EPOCHS)
    print("%s/%s: batch and %d single-node runs %.1f s; last task node %d (n %d, E_d %d), spec %.1f s"
          % (regime, init, K, batch_s, node, n[last], e_d[last], time.perf_counter() - t1))
    _assert_spec(out4[plan.edge_off[last]:plan.edge_off[last + 1]], fm4[last], ref, "%s/%s node %d" % (regime, init, node))


def _edge_m0(plan, seed):
    """M0 drawn per edge slot with the reference's distribution N(1, gain('relu')^2 * 2 / (n + n)), task by task."""
    rng = np.random.default_rng(seed)
    m0 = np.empty(plan.total_edges, np.float32)
    for t in range(plan.count):
        n = plan.n(t)
        m0[plan.edge_off[t]:plan.edge_off[t + 1]] = rng.normal(1.0, np.sqrt(2.0) * np.sqrt(2.0 / (n + n)), plan.edge_off[t + 1] - plan.edge_off[t])
    return m0
