"""GPU (-m gpu): graph-classification mode (explain_graph.cu, explain_var.cu) where the 12 golden graphs never take it: feature
masks, inputs wider than 32 features (lane groups of 9..32 lanes), more than 32 classes with pred_model read from global memory, every
shared-memory launch class up to the largest graph the tuned kernel accepts, structural edge cases of the max-pool, the benchmarked batch,
one teacher-forced step, and the device Philox init against its host restatement in every kernel.

Edge masks are compared with the line-by-line port at max(1e-4, 3 x rel-L2(fp64 closed form, port)), feature masks with sigmoid(F) of
the fp64 closed form after num_epochs - 1 updates at max(2e-4, 30 x that disagreement) (util.check_graph_masks)."""
import importlib.util
import os
from collections import deque

import networkx as nx
import numpy as np
import pytest
import torch

import gnnx
from gnnx import _abi
import gnnx_oracle as O
import util
from test_gpu_graph_variants import GX_ERR_UNSUPPORTED, _random_model
from test_oracle_graph_variants import dense_m0

pytestmark = pytest.mark.gpu
WP_SMEM_MAX = 2048                          # floats of pred_model + bias the tuned kernel stages in shared memory (GX_WP_SMEM_MAX)
CLASS_CAP_KB = [18, 27, 36, 44, 80, 226]    # largest footprint of each graph launch class (graph_mode.cu)
SMEM_PER_SM_KB = 228                        # H100: shared memory of one SM (each CTA also reserves 1 KB)


def _sig(x):
    return 1.0 / (1.0 + np.exp(-np.asarray(x, np.float64)))


def _ba(n, m=2, seed=1):
    """Barabasi-Albert graph: one family in n (the graph on n nodes is the first n nodes of the graph on n + 1)."""
    return nx.to_numpy_array(nx.barabasi_albert_graph(n, m, seed=seed)).astype(np.uint8)


def _tree(rng, n, extra):
    """Connected graph on n nodes: random recursive tree plus up to `extra` chords."""
    A = np.zeros((n, n), np.uint8)
    for i in range(1, n):
        p = rng.integers(0, i)
        A[i, p] = A[p, i] = 1
    a, b = rng.integers(0, n, extra), rng.integers(0, n, extra)
    ok = a != b
    A[a[ok], b[ok]] = 1
    A[b[ok], a[ok]] = 1
    return A


def _batch(parts, max_nodes):
    """parts: (n,n) adjacencies or (row offset, adjacency) -> the padded (G, max_nodes, max_nodes) batch."""
    adj = np.zeros((len(parts), max_nodes, max_nodes), np.uint8)
    for g, p in enumerate(parts):
        off, a = p if isinstance(p, tuple) else (0, p)
        adj[g, off:off + len(a), off:off + len(a)] = a
    return adj


def _active(A):
    return int((A.sum(1) > 0).sum())


def _layers(A, X, w, M0):
    """Layer outputs of the fp64 forward at M0 (feature mask 0.5): what the readout max-pools."""
    S = _sig(M0)
    a = A * (1 - np.eye(len(A))) * (S + S.T) / 2
    H, out = 0.5 * np.asarray(X, np.float64), []
    for l in range(1, 4):
        Y = a @ H @ w["W%d" % l] + w["b%d" % l]
        Y = Y / np.maximum(np.linalg.norm(Y, axis=1, keepdims=True), 1e-12)
        H = np.maximum(Y, 0) if l < 3 else Y
        out.append(H)
    return out


def _pool_rows(A, X, w, M0):
    """Row every readout feature is max-pooled from (first maximum, as torch.max)."""
    return np.concatenate([H.argmax(0) for H in _layers(A, X, w, M0)])


def _constant_wins_a_pool(A, X, w, M0):
    """Some readout feature pools from a row without edges (the kernel's edge-less constant)."""
    return bool((A.sum(1)[_pool_rows(A, X, w, M0)] == 0).any())


def _constant_beats_every_row(A, X, w, M0):
    """In some readout feature the edge-less constant relu(normalize(b_l)) / normalize(b_3) would exceed every row: a graph without
    edge-less rows must keep it out of the pool."""
    for l, H in enumerate(_layers(A, X, w, M0), 1):
        b = np.asarray(w["b%d" % l], np.float64)
        cst = b / max(np.linalg.norm(b), 1e-12)
        if ((np.maximum(cst, 0) if l < 3 else cst) > H.max(0)).any():
            return True
    return False


def _classes_run(eng):
    """Graph launch classes the engine's last explain call ran (gx_last_class_ms)."""
    _, end = eng.last_class_ms()
    return [c for c in range(6) if end[c] >= 0]


class Batch:
    """A padded graph batch on its own engine (3-layer model: the tuned kernel for widths <= 32)."""

    def __init__(self, w, adj, feat, label):
        self.w, self.adj, self.feat, self.label = w, adj, np.asarray(feat, np.float32), np.asarray(label)
        self.n, self.d = adj.shape[1], self.feat.shape[2]
        self.eng = gnnx.Engine(0)
        self.eng.set_model(w)
        self.eng.set_graph_batch(adj, self.feat, self.label)

    def rc(self, g):
        return self.eng.graph_rows_cols(g)

    def run(self, gids, m0_of, epochs, **over):
        """-> (edge_off, edge masks, feature masks [len(gids), d]); m0_of(g) = dense (n,n) M0 of graph g (None: GX_INIT_PHILOX)."""
        eo = self.eng.plan_graphs(gids)
        m0 = None if m0_of is None else np.concatenate([np.asarray(m0_of(g))[self.rc(g)] for g in gids]).astype(np.float32)
        out = np.zeros(max(int(eo[-1]), 1), np.float32)
        fm = np.zeros((len(gids), self.d), np.float32)
        self.eng.explain_graphs_host(self.eng.make_hparams(num_epochs=epochs, **over), m0, out, fm)
        return eo, out, fm

    def check(self, gids, m0_of, epochs, eo, out, fm):
        for t, g in enumerate(gids):
            util.check_graph_masks(self.adj[g], self.feat[g], self.label[g], self.w, m0_of(g), epochs, out[eo[t]:eo[t + 1]], fm[t],
                                   self.rc(g))

    def close(self):
        self.eng.close()


# ------------------------------------------------------------------------------------------------ A: feature masks, golden graphs
@pytest.mark.parametrize("epochs", [10, 30])
def test_golden_graphs_feature_masks(epochs):
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    b = Batch({k: gg[k] for k in util.WKEYS}, gg["adj"], gg["feat"], gg["label"])
    gids = list(range(int(gg["num_graphs"])))
    m0_of = lambda g: dense_m0(gg, g)
    b.check(gids, m0_of, epochs, *b.run(gids, m0_of, epochs))
    b.close()


# ------------------------------------------------------------------------------------------------ B: lane groups, many classes
# (d, hid, emb, C, bias, lane-group width, pred_model in shared memory).  Group width = max(ceil(d/4), hid/4, emb/4) of the PADDED
# widths (20/20 native, anything else <= 32 padded to 32/32); pred_model stays in shared memory while C (2h+e+1) <= 2048 floats.
B_CASES = [(1, 20, 20, 2, "positive", 5, True), (33, 20, 20, 33, "normal", 9, True), (36, 20, 20, 34, "positive", 9, False),
           (64, 20, 20, 40, "normal", 16, False), (100, 20, 20, 2, "normal", 25, True), (128, 20, 20, 33, "positive", 32, True),
           (1, 24, 17, 21, "normal", 8, True), (33, 24, 17, 22, "positive", 9, False), (36, 24, 17, 40, "normal", 9, False),
           (64, 24, 17, 21, "positive", 16, True), (100, 24, 17, 22, "normal", 25, False), (128, 24, 17, 40, "positive", 32, False)]


@pytest.mark.parametrize("d,hid,emb,C,bias,gw,wp_smem", B_CASES)
def test_wide_inputs_and_many_classes(d, hid, emb, C, bias, gw, wp_smem):
    rng = np.random.default_rng(1000 + 7 * d + C)
    H = 20 if (hid, emb) == (20, 20) else 32
    assert max(-(-d // 4), H // 4) == gw and (C * (3 * H + 1) <= WP_SMEM_MAX) == wp_smem
    w = _random_model(rng, 3, False, hid, emb, d, C, bias)
    n = 64
    adj = _batch([_tree(rng, 30, 5), (10, _tree(rng, 45, 8)), (4, _tree(rng, 60, 10))], n)
    assert [_active(A) for A in adj] == [30, 45, 60]
    feat = rng.normal(size=(3, n, d)).astype(np.float32)
    label = np.array([C - 1, rng.integers(0, C), 0])          # a class >= 32 as the target where C > 32
    b = Batch(w, adj, feat, label)
    m0_of = lambda g: O.draw_m0(n, seed=70 * d + C + g)
    if bias == "positive":
        assert any(_constant_wins_a_pool(adj[g].astype(float), feat[g], w, m0_of(g)) for g in range(3))
    gids = [0, 1, 2]
    b.check(gids, m0_of, 30, *b.run(gids, m0_of, 30))
    b.close()


# ------------------------------------------------------------------------------------------------ C: launch classes
MAXN_C = 448
CLASS_SIZES = [6, 15, 30, 50, 90, 300]     # BA(n, 2) graphs meant for classes 0..5 (d = 14, 20/20); class 5 has > 256 active rows
FAMILY = list(range(320, MAXN_C + 1))      # the same family, searched for the largest graph plan_graphs accepts


@pytest.fixture(scope="module")
def class_batch():
    rng = np.random.default_rng(3)
    sizes = CLASS_SIZES + FAMILY
    adj = _batch([_ba(s) for s in sizes], MAXN_C)
    feat = rng.normal(size=(len(sizes), MAXN_C, 14)).astype(np.float32)
    w = _random_model(rng, 3, False, 20, 20, 14, 2, "normal")
    b = Batch(w, adj, feat, rng.integers(0, 2, len(sizes)))
    b.gid = {s: g for g, s in enumerate(sizes)}
    yield b
    b.close()


def _accepted(b, g):
    try:
        b.eng.plan_graphs([g])
        return True
    except _abi.GnnxError as e:
        assert e.status == GX_ERR_UNSUPPORTED
        return False


def test_every_launch_class_and_the_largest_graph(class_batch):
    b = class_batch
    lo, hi = b.gid[FAMILY[0]], b.gid[FAMILY[-1]]
    assert _accepted(b, lo) and not _accepted(b, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if _accepted(b, mid) else (lo, mid)
    largest = lo
    assert _accepted(b, largest) and not _accepted(b, largest + 1)   # the next size up is refused (GX_ERR_UNSUPPORTED)
    big = b.gid[300]
    assert _active(b.adj[big]) > 256
    A = b.adj[big].astype(float)
    m0_of = lambda g: O.draw_m0(MAXN_C, seed=500 + g)
    rows = _pool_rows(A, b.feat[big], b.w, m0_of(big))
    assert ((rows >= 256) & (A.sum(1)[rows] > 0)).any()             # the max-pool takes features from active rows past 256
    gids = [b.gid[s] for s in CLASS_SIZES] + [largest]
    E = 30
    eo, out, fm = b.run(gids, m0_of, E)
    ran = {}
    for t, g in enumerate(gids):
        eo1, o1, f1 = b.run([g], m0_of, E)
        ran[g] = _classes_run(b.eng)
        assert len(ran[g]) == 1, ran
        assert np.array_equal(o1[:eo1[-1]], out[eo[t]:eo[t + 1]]) and np.array_equal(f1[0], fm[t]), g   # alone == in the mixed batch
    assert [ran[g][0] for g in gids] == [0, 1, 2, 3, 4, 5, 5], ran
    b.check(gids, m0_of, E, eo, out, fm)


def test_trace_and_resume_at_padded_width_32():
    """explain_graph_kernel<32, 32, 128, true>: the per-epoch trace of a 24/17 model (zero-padded to 32) against the port's trace, and
    a run split by the optimiser state == the straight run, bit for bit."""
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    rng = np.random.default_rng(24)
    C = 3
    w = _random_model(rng, 3, False, 24, 17, 14, C, "normal")
    b = Batch(w, gg["adj"], gg["feat"], gg["label"] % C)
    gids = [0, 3, 7]
    m0_of = lambda g: dense_m0(gg, g)
    E, d = 10, b.d
    eo, full, fm_full = b.run(gids, m0_of, E)
    te = int(eo[-1])
    m0 = np.concatenate([m0_of(g)[b.rc(g)] for g in gids]).astype(np.float32)
    trace = np.zeros((len(gids), E, _abi.GX_TRACE_COLS), np.float32)
    pred = np.zeros((len(gids), E, C), np.float32)
    out = np.zeros(te, np.float32)
    b.eng.explain_nodes_ex(b.eng.make_hparams(num_epochs=E), m0, out, trace=trace, trace_pred=pred, graphs=True)
    assert np.array_equal(out, full[:te])
    for t, g in enumerate(gids):
        tr = []
        O.explain_dense_torch(gg["adj"][g].astype(np.float64), gg["feat"][g], int(b.label[g]), None, 0, w, m0_of(g),
                              hp=O.default_hparams(num_epochs=E), graph_mode=True, trace=tr)
        for e in range(E):
            edges = tr[e]["pred_loss"] + tr[e]["size_edges"] + tr[e]["ent_edges"] + tr[e]["lap"] + tr[e]["feat_size"]
            assert abs(trace[t, e, _abi.TR_LOSS_EDGES] - edges) <= 1e-5 * abs(edges), (g, e)
            assert abs(trace[t, e, _abi.TR_DENSITY] - tr[e]["density"]) <= 1e-5
            assert np.abs(pred[t, e] - tr[e]["pred"]).max() <= 1e-5
    so = dict(M=np.zeros(te, np.float32), m=np.zeros(te, np.float32), v=np.zeros(te, np.float32), feat=np.zeros((len(gids), 3, d), np.float32))
    b.eng.explain_nodes_ex(b.eng.make_hparams(num_epochs=4), m0, out, state_out=so, graphs=True)
    rest = np.zeros(te, np.float32)
    fm = np.zeros((len(gids), d), np.float32)
    b.eng.explain_nodes_ex(b.eng.make_hparams(num_epochs=E - 3, init=_abi.GX_INIT_STATE, start_step=3), so["M"], rest, feat_mask_out=fm,
                           state_in=dict(m=so["m"], v=so["v"], feat=so["feat"]), graphs=True)
    assert np.array_equal(rest, full[:te]) and np.array_equal(fm, fm_full)
    b.close()


# ------------------------------------------------------------------------------------------------ D: structure edges
def test_structure_edge_cases():
    rng = np.random.default_rng(31)
    n, d, C = 48, 14, 2
    w = _random_model(rng, 3, False, 20, 20, d, C, "positive")
    star = np.zeros((6, 6), np.uint8)
    star[0, 1:] = star[1:, 0] = 1
    tie = np.zeros((12, 12), np.uint8)
    tie[:6, :6] = star
    tie[6:, 6:] = _tree(rng, 6, 3)
    parts = [_tree(rng, n, 12),            # 0: every row active -- no padding row, so no edge-less constant in the pools
             (6, _tree(rng, 34, 6)),       # 1: rows 0..5 isolated, below the active rows (plan relabelling, lo2gid)
             tie,                          # 2: row 0 is active but all its neighbours have zero features
             np.zeros((n, n), np.uint8),   # 3: no edge at all
             _tree(rng, 30, 4)]            # 4: an ordinary graph
    adj = _batch(parts, n)
    feat = rng.normal(size=(len(parts), n, d)).astype(np.float32)
    feat[2, 1:6] = 0.0
    b = Batch(w, adj, feat, rng.integers(0, C, len(parts)))
    m0_of = lambda g: O.draw_m0(n, seed=60 + g)
    deg = adj.sum(2)
    assert _active(adj[0]) == n and _constant_beats_every_row(adj[0].astype(float), feat[0], w, m0_of(0))
    assert (deg[1, :6] == 0).all() and (deg[1, 6:40] > 0).all()
    A2 = adj[2].astype(float)
    assert deg[2, 0] > 0 and not feat[2][A2[0] > 0].any()
    # row 0 of graph 2: layer-1 aggregate exactly 0, so its value is relu(normalize(b1)) -- the edge-less rows' constant -- and it
    # (the first of the tied rows) wins a layer-1 pool in the reference, where the kernel's strict first maximum keeps the constant;
    # the gradient routed to row 0 meets zero features on every edge, so the two choices must give the same masks
    assert (_pool_rows(A2, feat[2], w, m0_of(2))[:20] == 0).any()
    assert _constant_wins_a_pool(adj[1].astype(float), feat[1], w, m0_of(1))
    gids = [0, 1, 2, 3, 4]
    eo, out, fm = b.run(gids, m0_of, 30)
    assert eo[4] == eo[3]                                         # graph 3 has no edge slot
    b.check(gids, m0_of, 30, eo, out, fm)
    # the edge-less graph changes nothing for its neighbours in the batch
    sub = [0, 1, 2, 4]
    eo2, out2, fm2 = b.run(sub, m0_of, 30)
    for t2, g in enumerate(sub):
        t = gids.index(g)
        assert np.array_equal(out2[eo2[t2]:eo2[t2 + 1]], out[eo[t]:eo[t + 1]]) and np.array_equal(fm2[t2], fm[t]), g
    b.close()


# ------------------------------------------------------------------------------------------------ E: the benchmarked batch
def _bench_module():
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    return bench


def test_benchmarked_graph_batch():
    """bench.py --workload graphs: 4337 graphs, max_nodes 100, GX_INIT_PHILOX seed 7, 100 epochs.  Graphs from every launch class and
    the one graph without a padding row against the CPU oracle from the host Philox M0; a shuffled sub-batch gives the same bits."""
    bench = _bench_module()
    adj, feat, label, W = bench.make_graph_batch()
    G, n = adj.shape[:2]
    seed, E = 7, bench.NUM_EPOCHS
    b = Batch(W, adj, feat, label)
    philox = dict(init=_abi.GX_INIT_PHILOX, seed=seed)
    cls = np.empty(G, np.int64)
    for g in range(G):                        # the class of every graph, run alone (one epoch: the init only)
        b.run([g], None, 1, **philox)
        r = _classes_run(b.eng)
        assert len(r) == 1
        cls[g] = r[0]
    counts = np.bincount(cls, minlength=6)
    assert np.nonzero(counts)[0].tolist() == [0, 1, 2, 3, 4], counts
    assert [g for g in range(G) if _active(adj[g]) == n] == [1279]
    # more graphs than CTAs in some class: at most SMEM_PER_SM_KB / (footprint + 1 KB) CTAs of a class fit an SM, and a class-c graph
    # needs more than the cap of class c - 1, so those CTAs take a second graph from the queue and reuse their pair slab
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert any(counts[c] > sms * (SMEM_PER_SM_KB // (CLASS_CAP_KB[c - 1] + 1)) for c in range(1, 6)), counts
    gids = list(range(G))
    eo, out, fm = b.run(gids, None, E, **philox)

    def m0_of(g):
        r, c = b.rc(g)
        M0 = np.ones((n, n), np.float32)      # off-edge entries never reach the result
        M0[r, c] = O.philox_m0(seed, g, len(r), n)
        return M0

    picks = sorted({1279} | {int(g) for c in range(5) for g in np.nonzero(cls == c)[0][:2]})
    for g in picks:
        util.check_graph_masks(adj[g], feat[g], label[g], W, m0_of(g), E, out[eo[g]:eo[g + 1]], fm[g], b.rc(g))
    sub = np.random.default_rng(0).permutation(G)[:2500].tolist()
    eo2, out2, fm2 = b.run(sub, None, E, **philox)
    for t, g in enumerate(sub):
        assert np.array_equal(out2[eo2[t]:eo2[t + 1]], out[eo[g]:eo[g + 1]]) and np.array_equal(fm2[t], fm[g]), g
    b.close()


# ------------------------------------------------------------------------------------------------ F: teacher forcing
def _d128_batch():
    rng = np.random.default_rng(128)
    n, d = 64, 128
    adj = _batch([(3, _tree(rng, 45, 9))], n)
    w = _random_model(rng, 3, False, 20, 20, d, 3, "normal")
    return Batch(w, adj, rng.normal(size=(1, n, d)).astype(np.float32), [2])


@pytest.mark.parametrize("which", ["class5", "d128"])
def test_teacher_forced_step(which, class_batch):
    """One Adam step from the fp64 closed form's state after 50 updates (M, exp_avg, exp_avg_sq, feature state through state_in,
    GX_INIT_STATE, start_step 50) reproduces its state after 51: a per-step bar that holds where long trajectories drift apart."""
    b = class_batch if which == "class5" else _d128_batch()
    g = b.gid[300] if which == "class5" else 0
    t0 = 50
    A = b.adj[g].astype(np.float64)
    r, c = b.rc(g)
    args = (A, b.feat[g], int(b.label[g]), None, 0, b.w)
    _, s0 = O.explain_closed_form(*args, O.draw_m0(b.n, seed=51), hp=O.default_hparams(num_epochs=t0), graph_mode=True, return_state=True)
    init = dict(m=s0["mM"], v=s0["vM"], feat=np.stack([s0["F"], s0["mF"], s0["vF"]]), step=t0)
    _, s1 = O.explain_closed_form(*args, s0["M"], hp=O.default_hparams(num_epochs=1), graph_mode=True, return_state=True, init_state=init)
    S1 = _sig(s1["M"])
    mask1 = ((S1 + S1.T) / 2)[r, c]
    te = int(b.eng.plan_graphs([g])[-1])
    f32 = lambda x: np.ascontiguousarray(x, np.float32)
    out, sF = np.zeros(te, np.float32), np.zeros((1, b.d), np.float32)
    so = dict(M=np.zeros(te, np.float32), m=np.zeros(te, np.float32), v=np.zeros(te, np.float32), feat=np.zeros((1, 3, b.d), np.float32))
    b.eng.explain_nodes_ex(b.eng.make_hparams(num_epochs=2, init=_abi.GX_INIT_STATE, start_step=t0), f32(s0["M"][r, c]), out,
                           feat_mask_out=sF, state_in=dict(m=f32(s0["mM"][r, c]), v=f32(s0["vM"][r, c]), feat=f32(init["feat"][None])),
                           state_out=so, graphs=True)
    if which == "class5":
        assert _classes_run(b.eng) == [5] and _active(A) > 256
    else:
        assert b.d == 128
        b.close()
    assert util.rel_l2(out, mask1) <= 1e-5 and util.rel_l2(so["M"], s1["M"][r, c]) <= 1e-5, (util.rel_l2(out, mask1), util.rel_l2(so["M"], s1["M"][r, c]))
    assert np.abs(sF[0] - _sig(s1["F"])).max() <= 1e-5


# ------------------------------------------------------------------------------------------------ G: Philox in the node kernels
def _dist_from(rp, col, src):
    dist = -np.ones(len(rp) - 1, np.int64)
    dist[src] = 0
    q = deque([src])
    while q:
        u = q.popleft()
        for v in col[rp[u]:rp[u + 1]]:
            if dist[v] < 0:
                dist[v] = dist[u] + 1
                q.append(v)
    return dist


@pytest.mark.parametrize("path", ["smem", "cluster", "gang", "stream_gen1", "variant"])
def test_node_philox_init_is_the_host_restatement(path):
    """GX_INIT_PHILOX at num_epochs = 1 returns (sigmoid(M0_ij) + sigmoid(M0_ji)) / 2 with M0 from gnnx_oracle.philox_m0 (key = the
    explained node, slot = canonical edge slot, std sqrt(2/n)) in every node-mode kernel; "smem" includes the outer pairs kernel."""
    fx = util.load_fixture("syn1")
    eng = util.make_engine(fx)
    nodes = fx.nodes[:12]
    if path == "variant":
        eng.set_model(fx.weights, bn=True)
    elif path == "cluster":
        eng.debug_cluster(4, 1)
    elif path in ("gang", "stream_gen1"):
        eng.debug_force_stream(True)
        eng.debug_gang(0 if path == "gang" else -1)
    plan = eng.plan_nodes(nodes, 3)
    counts, _ = eng.plan_class_counts()
    if path == "smem":
        assert counts[:5].sum() == len(nodes)
    elif path == "cluster":
        assert counts[6] == len(nodes)
    else:
        assert counts[5] == len(nodes)
    seed = 99 + (5 << 32)
    out = np.zeros(plan.total_edges, np.float32)
    eng.explain_nodes_host(eng.make_hparams(num_epochs=1, init=_abi.GX_INIT_PHILOX, seed=seed), None, out)
    eng.close()
    m0 = np.concatenate([O.philox_m0(seed, node, int(plan.edge_off[t + 1] - plan.edge_off[t]), plan.n(t)) for t, node in enumerate(nodes)])
    n_outer = 0
    for t in range(plan.count):
        S = _sig(plan.dense_of(t, m0))
        r, c = plan.rows_cols_of(t)
        got, want = out[plan.edge_off[t]:plan.edge_off[t + 1]], ((S + S.T) / 2)[r, c]
        assert np.abs(got - want).max() <= 1e-6, (path, nodes[t])
        rp, col = plan.csr_of(t)
        dist = _dist_from(rp, col, int(plan.node_idx_new[t]))
        outer = (dist[r] == 3) & (dist[c] == 3)               # pairs between two outermost nodes
        n_outer += int(outer.sum())
        assert np.abs(got[outer] - want[outer]).max(initial=0) <= 1e-6
    assert n_outer > 0
