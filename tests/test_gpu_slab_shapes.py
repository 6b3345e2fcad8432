"""GPU (-m gpu): the slab-class kernels (explain_gang.cu, the first-generation explain_stream.cu, explain_var.cu) at the shapes where
they take code paths of their own, against fp64 / line-by-line CPU references:

  * width 32 (hid, emb <= 32 other than 20/20, zero-padded): the 4-slot edge layout (H4 == 8), the NTL = 4 tensor-core tiles, the
    trace instantiations, pred_model in shared memory up to C = 21 and read from global memory from C = 22, and the cluster class;
  * rows with more than kLongEdges = 512 induced edges, sliced over all warps of a CTA, at hop distance 0..3 from the explained node;
  * a config-5 sized subgraph (n >= 65 535) that lands in the slab class without any debug knob;
  * feature masks of subgraphs spanning many 128-node blocks of the dL/dsF reduction;
  * node-mode model variants whose conv weights (over kVarWeightWords floats) are read through L2 instead of shared memory.

Every run checks what it claims about its regime (launch class, n, induced degree per hop distance) so that a change to a builder cannot
silently move a case off the path it exists for."""
import types

import networkx as nx
import numpy as np
import pytest
import torch

import gnnx
import gnnx_oracle as O
import kernel_spec as KS
import util
from gnnx import _abi

pytestmark = pytest.mark.gpu

SLAB = 5                                     # launch class of the slab kernels (gx_plan_class_counts)
CLUSTER = 6                                  # launch class of the thread-block-cluster kernel
GANGS = (0, 1, 3, 16)                        # CTAs per task of explain_gang.cu (0 = automatic); -1 = explain_stream.cu
LONG = 512                                   # kLongEdges of explain_gang.cu: rows with more induced edges are sliced over a CTA


def _assert_kernel(gang_res, stream1_res, gang_runs):
    """Which slab kernel ran.  explain_gang.cu needs its whole working set in shared memory: at padded width 32 that is 230 KB at d = 112
    and 247 KB at d = 128, over the 227 KB limit, so there the slab class runs the first-generation explain_stream.cu whatever the
    gang setting.  The two kernels sum in different orders, so their bits differ exactly when both really ran."""
    same = all(np.array_equal(a, b) for a, b in zip(gang_res, stream1_res))
    assert same != gang_runs, "expected %s" % ("explain_gang.cu" if gang_runs else "explain_stream.cu for every gang setting")


def _weights(rng, d, C, hid, emb, L=3, scale=0.5):
    dims = [d] + [hid] * (L - 1) + [emb]
    sc = lambda *s: (rng.normal(size=s) * scale).astype(np.float32)
    w = {}
    for l in range(1, L + 1):
        w["W%d" % l] = sc(dims[l - 1], dims[l]); w["b%d" % l] = sc(dims[l])
    w["Wp"] = sc(C, hid * (L - 1) + emb); w["bp"] = sc(C)
    return w


def _ba_case(seed, N, m, d, C, hid, emb, L=3, bn=False):
    """BA graph, random features / labels / model; pred_label from the model's own forward pass (torch, dense)."""
    rng = np.random.default_rng(seed)
    G = nx.barabasi_albert_graph(N, m, seed=seed)
    rowptr, col = O.csr_from_edges(N, np.array(G.edges(), dtype=np.int64))
    feat = rng.normal(size=(N, d)).astype(np.float32)
    label = rng.integers(0, C, N).astype(np.int32)
    w = _weights(rng, d, C, hid, emb, L)
    A = O.dense_from_csr(rowptr, col)
    with torch.no_grad():
        pred = O._gcn_forward_torch(torch.tensor(feat[None]), torch.tensor(A[None], dtype=torch.float), O.weights_to_torch(w, False), False, bn=bn)[0].numpy()
    return types.SimpleNamespace(N=N, rowptr=rowptr, col=col, feat=feat, label=label, weights=w, L=L, bn=bn,
                                 pred_label=np.argmax(pred, 1).astype(np.int32))


def _engine(cs, force_stream=False, gang=0):
    eng = gnnx.Engine(0)
    eng.set_model(cs.weights, num_layers=cs.L, bn=cs.bn)
    eng.set_graph_csr(cs.rowptr, cs.col, cs.feat, cs.label, cs.pred_label)
    eng.debug_force_stream(force_stream)
    eng.debug_gang(gang)
    return eng


def _dense_m0(plan, seed):
    """Reference-style M0 (ExplainModule.construct_edge_mask) per task: packed edge values and the dense (n, n) arrays."""
    m0 = np.empty(plan.total_edges, np.float32)
    dense = []
    for t in range(plan.count):
        M0 = O.draw_m0(plan.n(t), seed=seed + t)
        r, c = plan.rows_cols_of(t)
        m0[plan.edge_off[t]:plan.edge_off[t + 1]] = M0[r, c]
        dense.append(M0)
    return m0, dense


def _edge_m0(plan, seed):
    """M0 drawn per edge slot (same distribution as the reference's), for subgraphs too large for a dense (n, n) draw."""
    rng = np.random.default_rng(seed)
    m0 = np.empty(plan.total_edges, np.float32)
    for t in range(plan.count):
        n = plan.n(t)
        std = np.sqrt(2.0) * np.sqrt(2.0 / (n + n))        # calculate_gain("relu") * sqrt(2 / (n + n))
        m0[plan.edge_off[t]:plan.edge_off[t + 1]] = rng.normal(1.0, std, plan.edge_off[t + 1] - plan.edge_off[t])
    return m0


def _explain(eng, plan, m0, epochs, d):
    out = np.zeros(plan.total_edges, np.float32)
    fm = np.zeros((plan.count, d), np.float32)
    eng.explain_nodes_host(eng.make_hparams(num_epochs=epochs), m0, out, fm)
    return out, fm


def _sig(x):
    return 1 / (1 + np.exp(-x))


# ------------------------------------------------------------------------------------------------ B. width 32 through the slab kernels
W32_CASES = [   # (seed, N, hid, emb, d, C): every width with d in {1, 5, 33, 112, 128} and C in {2, 21, 22, 40}; C = 21 is the last class
    # count whose pred_model (C x (96 + 1) floats at padded width 32) is staged in shared memory, C = 22 the first read from global
    # memory.  d = 112 is the widest input the gang kernel takes at width 32; at d = 128 the slab class runs explain_stream.cu.
    (21, 48, 32, 32, 128, 21), (22, 36, 32, 32, 1, 22), (23, 60, 32, 32, 33, 40), (24, 30, 32, 32, 5, 2),
    (25, 44, 24, 17, 5, 2), (26, 52, 24, 17, 128, 22), (27, 40, 20, 32, 33, 21), (28, 34, 20, 32, 5, 40),
    (29, 56, 8, 28, 128, 40), (30, 38, 8, 28, 33, 2), (31, 46, 24, 17, 1, 21), (32, 50, 32, 32, 112, 22), (33, 42, 8, 28, 112, 21),
]


@pytest.mark.parametrize("seed,N,hid,emb,d,C", W32_CASES, ids=["h%de%d_d%d_C%d" % c[2:] for c in W32_CASES])
def test_width32_slab_kernels_match_oracle(seed, N, hid, emb, d, C):
    """Both slab kernels at padded width 32, forced into the slab class: edge masks against the line-by-line torch port at 30 epochs,
    feature masks against the closed form's state, and gang sizes 1 / 3 / 16 / automatic bit-identical."""
    cs = _ba_case(seed, N, 2, d, C, hid, emb)
    nodes = list(range(0, N, N // 5))[:5]
    E = 30
    refs = []
    for node in nodes:
        idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(cs.rowptr, cs.col, cs.feat, cs.label, node, 3)
        refs.append((idx, O.dense_from_csr(srp, scol), sfeat, slabel[idx], cs.pred_label[nbrs]))
    res = {}
    for gang in GANGS + (-1,):
        eng = _engine(cs, force_stream=True, gang=gang)
        plan = eng.plan_nodes(nodes, 3)
        assert eng.plan_class_counts()[0][SLAB] == len(nodes)
        if gang == GANGS[0]:
            m0, dense = _dense_m0(plan, 1000 * seed)
        res[gang] = _explain(eng, plan, m0, E, d)
        eng.close()
    for t, node in enumerate(nodes):
        idx, A, sfeat, gt, pl = refs[t]
        hp = O.default_hparams(num_epochs=E)
        port = O.explain_dense_torch(A, sfeat, gt, pl, idx, cs.weights, dense[t], hp=hp)
        c64 = O.explain_closed_form(A, sfeat, gt, pl, idx, cs.weights, dense[t], hp=hp)
        _, st = O.explain_closed_form(A, sfeat, gt, pl, idx, cs.weights, dense[t], hp=O.default_hparams(num_epochs=E - 1), return_state=True)
        tol = max(1e-4, 3 * O.rel_l2(c64, port))
        for gang, (out, fm) in res.items():
            err = O.rel_l2(plan.dense_of(t, out), port)
            assert err <= tol, (gang, node, err, tol)
            assert np.abs(fm[t] - _sig(st["F"])).max() < max(2e-4, 30 * O.rel_l2(c64, port)), (gang, node)
    for gang in GANGS[1:]:
        assert np.array_equal(res[gang][0], res[0][0]) and np.array_equal(res[gang][1], res[0][1]), gang
    _assert_kernel(res[0], res[-1], d < 128)


@pytest.mark.parametrize("gang", [0, -1], ids=["gang", "stream1"])
def test_width32_trace_matches_port(gang):
    """The kTrace instantiations at width 32 (gx_explain_nodes_ex with a trace): per-epoch loss, density and prediction against the
    torch port's, and requesting a trace does not change the masks."""
    seed, N, hid, emb, d, C = 40, 44, 32, 32, 33, 22
    cs = _ba_case(seed, N, 2, d, C, hid, emb)
    nodes = [0, 11, 30]
    E = 12
    eng = _engine(cs, force_stream=True, gang=gang)
    plan = eng.plan_nodes(nodes, 3)
    assert eng.plan_class_counts()[0][SLAB] == len(nodes)
    m0, dense = _dense_m0(plan, 4000)
    hp = eng.make_hparams(num_epochs=E)
    out = np.zeros(plan.total_edges, np.float32); fm = np.zeros((plan.count, d), np.float32)
    trace = np.zeros((plan.count, E, _abi.GX_TRACE_COLS), np.float32)
    pred = np.zeros((plan.count, E, C), np.float32)
    eng.explain_nodes_ex(hp, m0, out, feat_mask_out=fm, trace=trace, trace_pred=pred)
    plain, fm_plain = _explain(eng, plan, m0, E, d)
    eng.close()
    assert np.array_equal(plain, out) and np.array_equal(fm_plain, fm), "requesting a trace changed the masks"
    for t, node in enumerate(nodes):
        idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(cs.rowptr, cs.col, cs.feat, cs.label, node, 3)
        tr = []
        port = O.explain_dense_torch(O.dense_from_csr(srp, scol), sfeat, slabel[idx], cs.pred_label[nbrs], idx, cs.weights, dense[t],
                                     hp=O.default_hparams(num_epochs=E), trace=tr)
        assert O.rel_l2(plan.dense_of(t, out), port) <= 1e-4, node
        for e in range(E):
            edges = tr[e]["pred_loss"] + tr[e]["size_edges"] + tr[e]["ent_edges"] + tr[e]["lap"] + tr[e]["feat_size"]
            assert abs(trace[t, e, _abi.TR_LOSS_EDGES] - edges) <= 1e-5 * abs(edges), (node, e)
            assert abs(trace[t, e, _abi.TR_DENSITY] - tr[e]["density"]) <= 1e-5, (node, e)
            assert np.abs(pred[t, e] - tr[e]["pred"]).max() <= 1e-5, (node, e)
            assert abs(trace[t, e, _abi.TR_PGT] - pred[t, e, int(slabel[idx])]) <= 1e-6, (node, e)


@pytest.mark.parametrize("d", [96, 128])
def test_width32_natural_slab_class(d):
    """A 32/32 model on BA(1500, 6): the tasks exceed shared memory by themselves and land in the slab class without any debug knob
    (the gang kernel at d = 96, explain_stream.cu at d = 128).  Edge masks against the torch port, feature masks (about ten 128-node
    blocks) against the fp64 edge-list spec, for the automatic choice and for the first-generation kernel."""
    cs = _ba_case(11, 1500, 6, d, 4, 32, 32)
    nodes = [0, 700]
    E = 10
    res = {}
    for gang in (0, -1):
        eng = _engine(cs, gang=gang)
        plan = eng.plan_nodes(nodes, 3)
        assert eng.plan_class_counts()[0][SLAB] == len(nodes)
        assert min(plan.n(t) for t in range(plan.count)) >= 400
        if not res:
            m0, dense = _dense_m0(plan, 900)
        res[gang] = _explain(eng, plan, m0, E, d)
        eng.close()
    _assert_kernel(res[0], res[-1], d < 128)
    for (out, fm), t, node in [(res[g], t, node) for g in res for t, node in enumerate(nodes)]:
        idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(cs.rowptr, cs.col, cs.feat, cs.label, node, 3)
        assert np.array_equal(nbrs, plan.neighbors_of(t))
        port = O.explain_dense_torch(O.dense_from_csr(srp, scol), sfeat, slabel[idx], cs.pred_label[nbrs], idx, cs.weights, dense[t],
                                     hp=O.default_hparams(num_epochs=E))
        r, c = plan.rows_cols_of(t)
        assert util.rel_l2(out[plan.edge_off[t]:plan.edge_off[t + 1]], port[r, c]) <= 1e-4, node
        _, F = KS.explain_pruned_edges_sparse(srp, scol, sfeat, slabel[idx], cs.pred_label[nbrs], idx, cs.weights, dense[t][r, c],
                                              num_epochs=E, return_F=True)
        assert np.abs(fm[t] - _sig(F)).max() <= 2e-5, (node, np.abs(fm[t] - _sig(F)).max())


@pytest.mark.parametrize("cs_size", [2, 4])
def test_width32_cluster_class_matches_single_cta(cs_size):
    """The cluster class of explain_node.cu at padded width 32 agrees with the single-CTA kernel to round-off."""
    cs = _ba_case(50, 60, 3, 33, 22, 24, 17)
    nodes = [0, 5, 12, 31, 59]
    eng = _engine(cs)
    res = {}
    for size in (1, cs_size):
        eng.debug_cluster(size, 1)
        plan = eng.plan_nodes(nodes, 3)
        counts, csz = eng.plan_class_counts()
        assert counts[CLUSTER] == (len(nodes) if size > 1 else 0) and csz == size, (counts, csz)
        if size == 1:
            m0, _ = _dense_m0(plan, 5000)
        res[size] = _explain(eng, plan, m0, 10, 33)
    eng.close()
    assert util.rel_l2(res[cs_size][0], res[1][0]) < 2e-6
    assert np.allclose(res[cs_size][1], res[1][1], rtol=1e-5, atol=1e-7)


# ------------------------------------------------------------------------------------------------ C. hub rows around kLongEdges
HUB_DEGREES = (511, 512, 513)
BIG = 2048


def _hub_graph(pool=2100, seed=4):
    """BA(pool, 2) plus planted rows: a connector c adjacent to every pool node, hubs of degree 511 / 512 / 513 / 2048 adjacent to c and
    to pool nodes, r2 - c and r3 - p3 - c, and a separate 40-node BA component.  Every hub neighbour is at most one hop from c, so:
    explaining a hub puts it at distance 0, explaining c puts the hubs at distance 1, r2 at distance 2 and r3 at distance 3 -- with
    every neighbour of a distance-3 hub (c at 2, pool nodes at 3) inside the 3-hop ball, so its induced degree is its full degree.
    c itself (degree > 2000) sits at distance 0, 1 and 2 of those tasks."""
    rng = np.random.default_rng(seed)
    edges = [tuple(e) for e in nx.barabasi_albert_graph(pool, 2, seed=seed).edges()]
    c = pool
    edges += [(c, p) for p in range(pool)]
    hubs = {}
    nxt = pool + 1
    for D in HUB_DEGREES + (BIG,):
        h = nxt; nxt += 1
        hubs[D] = h
        edges.append((c, h))
        edges += [(h, int(p)) for p in rng.choice(pool, D - 1, replace=False)]
    r2, r3, p3 = nxt, nxt + 1, nxt + 2
    nxt += 3
    edges += [(r2, c), (r3, p3), (p3, c)]
    small0 = nxt
    edges += [(small0 + a, small0 + b) for a, b in nx.barabasi_albert_graph(40, 2, seed=seed).edges()]
    N = small0 + 40
    rowptr, col = O.csr_from_edges(N, np.array(edges, np.int64))
    return types.SimpleNamespace(N=N, rowptr=rowptr, col=col, c=c, hubs=hubs, r2=r2, r3=r3, small=[small0, small0 + 17, small0 + 33],
                                 hub_nodes=[c, hubs[511], hubs[512], hubs[513], r2, r3])


def _hub_case(hid=20, emb=20, L=3, bn=False, seed=7, d=128):
    g = _hub_graph()
    rng = np.random.default_rng(seed)
    C = 4
    feat = rng.normal(size=(g.N, d)).astype(np.float32)
    label = rng.integers(0, C, g.N).astype(np.int32)
    pred_label = rng.integers(0, C, g.N).astype(np.int32)       # an input of the Laplacian term; any labelling exercises it
    return types.SimpleNamespace(N=g.N, rowptr=g.rowptr, col=g.col, feat=feat, label=label, pred_label=pred_label,
                                 weights=_weights(rng, d, C, hid, emb, L), L=L, bn=bn, g=g)


@pytest.fixture(scope="module")
def hub20():
    return _hub_case()


def _assert_long_rows_regime(plan, L=3):
    """Every (hop distance, induced degree) combination of interest is present in the batch: 511 / 512 / 513 and >= 2000 at distance
    0, 1, 2 and 3 from the explained node."""
    seen = set()
    for t in range(plan.count):
        rp, col = plan.csr_of(t)
        dist = KS.hop_distances(rp, col, int(plan.node_idx_new[t]), L)
        assert (dist >= 0).all()
        deg = np.diff(rp)
        for k in range(4):
            for D in HUB_DEGREES:
                if ((dist == k) & (deg == D)).any():
                    seen.add((k, D))
            if ((dist == k) & (deg >= 2000)).any():
                seen.add((k, "big"))
    want = {(k, D) for k in range(4) for D in HUB_DEGREES + ("big",)}
    assert seen >= want, sorted(want - seen, key=str)


def _spec(cs, plan, m0, epochs):
    """fp64 edge-list specification of every task: (edge mask, F).  The sparse form for the default model, the np.add.at form for variants."""
    res = []
    for t in range(plan.count):
        rp, col = plan.csr_of(t)
        nbrs = plan.neighbors_of(t)
        idx = int(plan.node_idx_new[t])
        args = (rp, col, cs.feat[nbrs], cs.label[nbrs][idx], cs.pred_label[nbrs], idx, cs.weights, m0[plan.edge_off[t]:plan.edge_off[t + 1]])
        if cs.L == 3 and not cs.bn:
            res.append(KS.explain_pruned_edges_sparse(*args, num_epochs=epochs, return_F=True))
        else:
            a, _, F = KS.explain_pruned_edges(*args, num_epochs=epochs, bn=cs.bn, return_F=True)
            res.append((a, F))
    return res


def _assert_vs_spec(plan, out, fm, spec, label):
    errs = []
    for t in range(plan.count):
        a, F = spec[t]
        err = util.rel_l2(out[plan.edge_off[t]:plan.edge_off[t + 1]], a)
        ferr = np.abs(fm[t] - _sig(F)).max()
        assert err <= 1e-4 and ferr <= 2e-5, (label, int(plan.nodes[t]), err, ferr)
        errs.append(err)
    assert np.median(errs) <= 2e-6, (label, errs)


@pytest.mark.parametrize("width", [20, 32])
def test_hub_rows_match_spec(hub20, width):
    """Rows with 511 / 512 / 513 and >= 2000 induced edges at hop distance 0..3: both slab kernels against the fp64 spec at 10 epochs,
    gang sizes 1 / 5 / 16 / automatic bit-identical, the first-generation kernel bit-identical to itself across runs.  The 32/32 model
    takes d = 96, the gang kernel's limit at that width being below 128."""
    cs = hub20 if width == 20 else _hub_case(32, 32, d=96)
    nodes = cs.g.hub_nodes
    d = cs.feat.shape[1]
    E = 10
    res = {}
    for gang in (0, 1, 5, 16, -1, -1):
        eng = _engine(cs, gang=gang)
        plan = eng.plan_nodes(nodes, 3)
        assert eng.plan_class_counts()[0][SLAB] == len(nodes)
        if not res:
            _assert_long_rows_regime(plan)
            m0 = _edge_m0(plan, 11)
            spec = _spec(cs, plan, m0, E)
        out, fm = _explain(eng, plan, m0, E, d)
        eng.close()
        if gang in res:
            assert np.array_equal(out, res[gang][0]) and np.array_equal(fm, res[gang][1]), "first-generation kernel is not deterministic"
        res[gang] = (out, fm)
    for gang in (0, -1):
        _assert_vs_spec(plan, *res[gang], spec, (width, gang))
    for gang in (1, 5, 16):
        assert np.array_equal(res[gang][0], res[0][0]) and np.array_equal(res[gang][1], res[0][1]), gang
    _assert_kernel(res[0], res[-1], True)


def test_hub_slab_reuse_is_bit_identical(hub20):
    """[hub, small, hub, small, hub] with 64-CTA gangs (two gangs for five tasks): a gang runs several tasks one after the other in
    the same slab, and every task gets the bits it gets when it is explained alone."""
    cs = hub20
    g = cs.g
    nodes = [g.c, g.small[0], g.hubs[513], g.small[1], g.r3]
    d = cs.feat.shape[1]
    eng = _engine(cs, force_stream=True, gang=64)
    plan = eng.plan_nodes(nodes, 3)
    assert eng.plan_class_counts()[0][SLAB] == len(nodes)
    assert [plan.n(t) < 100 for t in range(plan.count)] == [False, True, False, True, False]
    m0 = _edge_m0(plan, 12)
    out, fm = _explain(eng, plan, m0, 10, d)
    for t, node in enumerate(nodes):
        p1 = eng.plan_nodes([node], 3)
        o1, f1 = _explain(eng, p1, m0[plan.edge_off[t]:plan.edge_off[t + 1]], 10, d)
        assert np.array_equal(o1, out[plan.edge_off[t]:plan.edge_off[t + 1]]) and np.array_equal(f1[0], fm[t]), node
    eng.close()


# ------------------------------------------------------------------------------------------------ D. the config-5 regime
def test_config5_sized_subgraph_matches_sparse_spec():
    """BA(90 000, 4, seed 0), d = 128: the 3-hop neighbourhood of the highest-degree node has n >= 65 535 (the 16-bit index limit of the
    shared-memory classes), so the plan puts it in the slab class without any knob and the automatic gang spans the device.  4 epochs
    with host M0 against the fp64 sparse spec; a second, much smaller task in the same batch gets the bits it gets alone."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import dijkstra
    N, d, C = 90000, 128, 4
    rowptr, col = O.csr_from_edges(N, np.array(nx.barabasi_albert_graph(N, 4, seed=0).edges(), dtype=np.int64))
    rng = np.random.default_rng(5)
    feat = rng.normal(size=(N, d)).astype(np.float32)
    label = rng.integers(0, C, N).astype(np.int32)
    cs = types.SimpleNamespace(rowptr=rowptr, col=col, feat=feat, label=label, pred_label=rng.integers(0, C, N).astype(np.int32),
                               weights=_weights(rng, d, C, 20, 20), L=3, bn=False)
    hub = int(np.argmax(np.diff(rowptr)))
    eng = _engine(cs)
    cand = np.arange(N - 400, N, dtype=np.int32)
    n_c, _ = eng.count_nodes(cand, 3)
    ok = n_c >= 2000                                   # far beyond shared memory at d = 128, far below the hub's ball
    small = int(cand[ok][np.argmin(n_c[ok])])
    nodes = [hub, small]
    plan = eng.plan_nodes(nodes, 3)
    counts = eng.plan_class_counts()[0]
    assert counts[SLAB] == 2 and counts.sum() == 2, counts
    n = plan.n(0)
    assert n >= 65535 and plan.n(1) * 10 < n, (n, plan.n(1))
    # the plan's subgraph is the induced 3-hop ball (checked independently of gx_plan_nodes)
    A = sp.csr_matrix((np.ones(len(col), np.float32), col, rowptr), shape=(N, N))
    ball = np.nonzero(np.isfinite(dijkstra(A, indices=hub, unweighted=True, limit=3.5)))[0]
    assert np.array_equal(plan.neighbors_of(0), ball)
    sub = A[ball][:, ball].tocsr(); sub.sort_indices()
    rp, scol = plan.csr_of(0)
    assert np.array_equal(rp, sub.indptr) and np.array_equal(scol, sub.indices)
    assert (np.diff(rp) > LONG).sum() >= 5
    m0 = _edge_m0(plan, 13)
    E = 4
    out, fm = _explain(eng, plan, m0, E, d)
    p1 = eng.plan_nodes([small], 3)
    assert eng.plan_class_counts()[0][SLAB] == 1
    o1, f1 = _explain(eng, p1, m0[plan.edge_off[1]:], E, d)
    eng.close()
    assert np.array_equal(o1, out[plan.edge_off[1]:]) and np.array_equal(f1[0], fm[1])
    idx = int(plan.node_idx_new[0])
    a, F = KS.explain_pruned_edges_sparse(rp, scol, feat[ball], label[hub], cs.pred_label[ball], idx, cs.weights,
                                          m0[:plan.edge_off[1]], num_epochs=E, return_F=True)
    err = util.rel_l2(out[:plan.edge_off[1]], a)
    ferr = float(np.abs(fm[0] - _sig(F)).max())
    print("config-5 subgraph: n %d, E_d %d, rows over %d edges %d; edge mask rel-L2 %.2e, feature mask max-abs %.2e vs fp64 spec"
          % (n, len(scol), LONG, (np.diff(rp) > LONG).sum(), err, ferr))
    assert err <= 1e-5 and ferr <= 2e-5, (err, ferr)


# ------------------------------------------------------------------------------------------------ E. variant kernel, weights through L2
VAR_CASES = [(61, 4, False, 128, 128), (62, 4, True, 128, 128), (63, 3, True, 128, 96), (64, 2, False, 128, 128)]


@pytest.mark.parametrize("seed,L,bn,hid,emb", VAR_CASES, ids=["L4", "L4bn", "L3bn_h128e96", "L2_smem"])
def test_variant_weights_through_l2_match_oracle(seed, L, bn, hid, emb):
    """Node-mode explain_var.cu with d = 128: conv weights of 65 536 / 45 056 floats exceed kVarWeightWords (36 864) and are read
    through L2; the 2-layer 128-wide model (32 768) is the shared-memory control.  Torch port at 20 epochs, feature masks against the
    closed form's state."""
    d, C = 128, 5
    cs = _ba_case(seed, 48, 2, d, C, hid, emb, L=L, bn=bn)
    wwords = sum(cs.weights["W%d" % l].size for l in range(1, L + 1))
    assert (wwords > 36 * 1024) == (L > 2), wwords
    nodes = [0, 7, 23, 47]
    E = 20
    eng = _engine(cs)
    plan = eng.plan_nodes(nodes, L)
    assert eng.plan_class_counts()[0][SLAB] == len(nodes)
    m0, dense = _dense_m0(plan, 500 * seed)
    out, fm = _explain(eng, plan, m0, E, d)
    eng.close()
    for t, node in enumerate(nodes):
        idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(cs.rowptr, cs.col, cs.feat, cs.label, node, L)
        A = O.dense_from_csr(srp, scol)
        hp = O.default_hparams(num_epochs=E)
        port = O.explain_dense_torch(A, sfeat, slabel[idx], cs.pred_label[nbrs], idx, cs.weights, dense[t], hp=hp, bn=bn)
        c64 = O.explain_closed_form(A, sfeat, slabel[idx], cs.pred_label[nbrs], idx, cs.weights, dense[t], hp=hp, bn=bn)
        tol = max(1e-4, 3 * O.rel_l2(c64, port))
        assert O.rel_l2(plan.dense_of(t, out), port) <= tol, (node, O.rel_l2(plan.dense_of(t, out), port), tol)
        _, st = O.explain_closed_form(A, sfeat, slabel[idx], cs.pred_label[nbrs], idx, cs.weights, dense[t],
                                      hp=O.default_hparams(num_epochs=E - 1), bn=bn, return_state=True)
        assert np.abs(fm[t] - _sig(st["F"])).max() < max(2e-4, 30 * O.rel_l2(c64, port)), node


def test_variant_weights_through_l2_on_hub_rows():
    """The 4-layer 128-wide --bn model (weights through L2) on the hub graph's 4-hop neighbourhoods, against the fp64 edge-list spec."""
    cs = _hub_case(128, 128, L=4, bn=True, seed=8)
    g = cs.g
    nodes = [g.r3, g.hubs[513]]
    eng = _engine(cs)
    plan = eng.plan_nodes(nodes, 4)
    assert eng.plan_class_counts()[0][SLAB] == len(nodes)
    assert max(np.diff(plan.csr_of(t)[0]).max() for t in range(plan.count)) > 2000
    m0 = _edge_m0(plan, 14)
    out, fm = _explain(eng, plan, m0, 10, cs.feat.shape[1])
    eng.close()
    spec = _spec(cs, plan, m0, 10)
    for t in range(plan.count):
        a, F = spec[t]
        err = util.rel_l2(out[plan.edge_off[t]:plan.edge_off[t + 1]], a)
        ferr = np.abs(fm[t] - _sig(F)).max()
        assert err <= 1e-4 and ferr <= 2e-5, (nodes[t], err, ferr)
