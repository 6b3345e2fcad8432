"""GPU (-m gpu): parity of the CUDA path, called through the C ABI, against
  (1) the golden vectors produced by the unmodified reference (tests/golden, oracle/gen_golden.py),
  (2) the CPU oracle on seeded random inputs (sizes the oracle finishes in seconds),
  (3) size-independent properties at BASELINE.json's full size (all 700 syn1 nodes).
Tolerances: k-hop extraction bit-exact; masks 1e-4 relative L2 per node (north_star) wherever the
reference's own result is reproducible to 1e-4 under fp reordering, else 3x the spread of the two
independent CPU restatements (tests/golden/*_cond.npz, oracle/gen_conditioning.py)."""
import math
import os
import types

import numpy as np
import pytest
import torch

import gnnx
from gnnx import _abi
import gnnx_oracle as O
import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=["rand", "syn4", "syn1"])
def fx(request):
    return util.load_fixture(request.param)


@pytest.fixture(scope="module")
def syn1():
    return util.load_fixture("syn1")




# ------------------------------------------------------------------------------------ k-hop (integer, bit-exact)
def test_khop_matches_reference_bit_exact(fx):
    eng = util.make_engine(fx)
    plan = eng.plan_nodes(fx.nodes, 3)
    for t, node in enumerate(fx.nodes):
        assert np.array_equal(plan.neighbors_of(t), fx.gold["n%d_nbrs" % node]), node
        assert int(plan.node_idx_new[t]) == int(fx.gold["n%d_idx_new" % node]), node
        # induced sub-adjacency == reference's adj[nbrs][:, nbrs] in row-major nonzero order
        idx, srp, scol, _, _, _ = O.extract_neighborhood(fx.rowptr, fx.col, fx.feat, fx.label, node, 3)
        rp, col = plan.csr_of(t)
        assert np.array_equal(rp, srp) and np.array_equal(col, scol), node
    eng.close()


@pytest.mark.parametrize("name", ["syn1", "syn4"])
def test_neighborhoods_full_matrix_bit_exact(name):
    fx = util.load_fixture(name)
    hops = np.load(util.GOLDEN + "/%s_hops.npz" % name)
    ref = np.unpackbits(hops["hop_bits"], axis=1)[:, : fx.N]
    A = O.dense_from_csr(fx.rowptr, fx.col)
    got = gnnx.graph_utils.neighborhoods(A[None], 3, True)
    assert got.dtype == int and got.shape == (1, fx.N, fx.N)
    assert np.array_equal(got[0].astype(np.uint8), ref)
    for k in (1, 2, 4):
        assert np.array_equal(gnnx.graph_utils.neighborhoods(A[None], k, True), O.neighborhoods_dense(A[None], k))


def test_khop_edge_cases():
    # path 0-1-2-3-4, an isolated node 5, a self loop on 4
    rowptr = np.array([0, 1, 3, 5, 7, 9, 9], np.int32)
    col = np.array([1, 0, 2, 1, 3, 2, 4, 3, 4], np.int32)
    N = 6
    A = O.dense_from_csr(rowptr, col, N)
    eng = gnnx.Engine(0)
    eng.set_graph_csr_structure(rowptr, col)
    for k in (1, 2, 3, 5):
        rows = eng.neighborhood_rows(np.arange(N), k)
        assert np.array_equal(rows.astype(int), O.neighborhoods_dense(A[None], k)[0]), k
    eng.close()


# ------------------------------------------------------------------------------------ masks vs the reference
def _run_golden(fx, num_epochs):
    eng = util.make_engine(fx)
    plan = eng.plan_nodes(fx.nodes, 3)
    out = np.zeros(plan.total_edges, np.float32)
    eng.explain_nodes_host(eng.make_hparams(num_epochs=num_epochs), util.golden_m0(fx, plan), out)
    eng.close()
    return plan, out


def _errs_vs(fx, golden_file, epochs):
    g = np.load(util.GOLDEN + "/" + golden_file)
    assert int(g["num_epochs"]) == epochs
    plan, out = _run_golden(fx, epochs)
    return {node: util.rel_l2(out[plan.edge_off[t]:plan.edge_off[t + 1]], g["n%d_mask" % node])
            for t, node in enumerate(fx.nodes)}


def test_masks_match_reference_golden_10_epochs(fx):
    """Short horizon (10 epochs, golden from the unmodified reference): EVERY node within 1e-4 --
    nine Adam steps leave no room for a trajectory to amplify rounding differences (DESIGN.md 'Parity')."""
    errs = _errs_vs(fx, "%s_golden_e10.npz" % fx.name, 10)
    bad = {n: e for n, e in errs.items() if not e <= 1e-4}
    assert not bad, bad
    assert np.median(list(errs.values())) < 2e-6


def test_masks_match_reference_golden_30_epochs(fx):
    """30 epochs, PER NODE: within 1e-4 of the reference wherever the reference itself is reproducible under +-1 ulp input
    noise (79 of the 81 syn1 nodes, every syn4 / rand node), within 3x the reference's own spread on the two syn1 nodes whose
    trajectories have started to separate (293, 533: tests/golden/syn1_sens.npz)."""
    errs = _errs_vs(fx, "%s_golden_e30.npz" % fx.name, 30)
    tol = util.assert_per_node(errs, fx.name, 30)
    assert sum(t > 1e-4 for t in tol.values()) <= (2 if fx.name == "syn1" else 0)
    assert np.median(list(errs.values())) < 2e-6


def test_masks_match_reference_golden_100_epochs(fx):
    """Full horizon (the reference default, 100 epochs), PER NODE.  Six syn1 trajectories are chaotic (0, 3, 23, 33, 163, 293: a relu
    kink crossed one epoch earlier or later moves the final mask by 1e-4..7e-2; the bit-exact port of the reference does that to
    ITSELF when M0 is nudged by one ulp, tests/golden/syn1_sens.npz): there the bar is 3x the reference's own spread.  Every other
    node -- 73 of 81 on syn1 (two more sit at 3.6e-5 / 5.2e-5 spread), all of syn4 and rand -- must be within the north-star 1e-4."""
    plan, out = _run_golden(fx, 100)
    errs = {node: util.rel_l2(out[plan.edge_off[t]:plan.edge_off[t + 1]], fx.gold["n%d_mask" % node])
            for t, node in enumerate(fx.nodes)}
    tol = util.assert_per_node(errs, fx.name, 100)
    assert sum(t > 1e-4 for t in tol.values()) <= (8 if fx.name == "syn1" else 0)
    assert np.median(list(errs.values())) < 1e-5


def _random_case(seed, n_nodes, m, d, C, graph="ba"):
    import networkx as nx
    rng = np.random.default_rng(seed)
    if graph == "ba":
        G = nx.barabasi_albert_graph(n_nodes, m, seed=seed)
    elif graph == "path":
        G = nx.path_graph(n_nodes)
    elif graph == "star":
        G = nx.star_graph(n_nodes - 1)
    elif graph == "complete":
        G = nx.complete_graph(n_nodes)
    else:
        G = nx.gnp_random_graph(n_nodes, 0.15, seed=seed)
        G.add_edges_from((i, (i + 1) % n_nodes) for i in range(n_nodes))
    A = nx.to_numpy_array(G)
    N = A.shape[0]
    rowptr, col = O.csr_from_dense(A)
    feat = rng.normal(size=(N, d)).astype(np.float32)
    label = rng.integers(0, C, N)
    sc = lambda *s: (rng.normal(size=s) * 0.5).astype(np.float32)
    w = dict(W1=sc(d, 20), b1=sc(20), W2=sc(20, 20), b2=sc(20), W3=sc(20, 20), b3=sc(20), Wp=sc(C, 60), bp=sc(C))
    Wt = O.weights_to_torch(w, False)
    with torch.no_grad():
        pred = O._gcn_forward_torch(torch.tensor(feat[None]), torch.tensor(A[None], dtype=torch.float), Wt, False)[0].numpy()
    return types.SimpleNamespace(N=N, rowptr=rowptr, col=col, feat=feat, label=label, weights=w,
                                 pred_label=np.argmax(pred, 1).astype(np.int32))


@pytest.mark.parametrize("seed,n_nodes,m,d,C,graph", [
    (1, 40, 2, 10, 4, "ba"), (2, 30, 1, 1, 2, "ba"), (3, 25, 3, 3, 7, "ba"), (4, 12, 0, 16, 3, "path"),
    (5, 9, 0, 5, 2, "star"), (6, 6, 0, 10, 4, "complete"), (7, 45, 0, 33, 5, "gnp"), (8, 35, 2, 64, 3, "ba"),
    (9, 30, 2, 128, 2, "ba"), (10, 50, 4, 32, 40, "ba"),
])
def test_masks_match_oracle_random(seed, n_nodes, m, d, C, graph):
    """Line-by-line torch port (bit-exact to the reference on the golden set) vs the kernel."""
    cs = _random_case(seed, n_nodes, m, d, C, graph)
    eng = util.make_engine(cs)
    nodes = list(range(0, cs.N, max(1, cs.N // 5)))[:5]
    plan = eng.plan_nodes(nodes, 3)
    m0 = np.empty(plan.total_edges, np.float32)
    dense_m0 = []
    for t in range(plan.count):
        M0 = O.draw_m0(plan.n(t), seed=100 * seed + t)
        r, c = plan.rows_cols_of(t)
        m0[plan.edge_off[t]:plan.edge_off[t + 1]] = M0[r, c]
        dense_m0.append(M0)
    out = np.zeros(plan.total_edges, np.float32)
    fm = np.zeros((plan.count, d), np.float32)
    hp = eng.make_hparams(num_epochs=30)
    eng.explain_nodes_host(hp, m0, out, fm)
    for t, node in enumerate(nodes):
        idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(cs.rowptr, cs.col, cs.feat, cs.label, node, 3)
        assert np.array_equal(nbrs, plan.neighbors_of(t))
        A = O.dense_from_csr(srp, scol)
        ref = O.explain_dense_torch(A, sfeat, slabel[idx], cs.pred_label[nbrs], idx, cs.weights, dense_m0[t],
                                    hp=O.default_hparams(num_epochs=30))
        got = plan.dense_of(t, out)
        # the two independent CPU restatements bound what fp reordering does to this trajectory
        c64 = O.explain_closed_form(A, sfeat, slabel[idx], cs.pred_label[nbrs], idx, cs.weights, dense_m0[t],
                                    hp=O.default_hparams(num_epochs=30))
        tol = max(1e-4, 3 * O.rel_l2(c64, ref))
        assert O.rel_l2(got, ref) <= tol, (node, O.rel_l2(got, ref), tol)
        # feature mask after the last observed update (29 updates) against the closed form's state
        _, st = O.explain_closed_form(A, sfeat, slabel[idx], cs.pred_label[nbrs], idx, cs.weights, dense_m0[t],
                                      hp=O.default_hparams(num_epochs=29), return_state=True)
        assert np.abs(fm[t] - 1 / (1 + np.exp(-st["F"]))).max() < max(2e-4, 30 * O.rel_l2(c64, ref)), node
    eng.close()


def test_one_epoch_returns_initial_mask(syn1):
    eng = util.make_engine(syn1)
    nodes = syn1.nodes[:10]
    plan = eng.plan_nodes(nodes, 3)
    m0 = util.golden_m0(syn1, plan)
    out = np.zeros(plan.total_edges, np.float32)
    eng.explain_nodes_host(eng.make_hparams(num_epochs=1), m0, out)
    for t in range(plan.count):
        M = plan.dense_of(t, m0)
        S = 1 / (1 + np.exp(-M))
        r, c = plan.rows_cols_of(t)
        exp = ((S + S.T) / 2)[r, c]
        assert np.abs(out[plan.edge_off[t]:plan.edge_off[t + 1]] - exp).max() < 1e-6
    eng.close()


# ------------------------------------------------------------------------------------ full size: properties
def test_full_syn1_properties(syn1):
    """All 700 nodes (BASELINE.json config 2), device-side init: symmetry, range, determinism,
    independence of batching/order (what makes N-GPU sharding bit-identical), golden subset."""
    eng = util.make_engine(syn1)
    nodes = np.arange(syn1.N)
    plan = eng.plan_nodes(nodes, 3)
    hp = eng.make_hparams(init=_abi.GX_INIT_PHILOX, seed=1234)
    out = np.zeros(plan.total_edges, np.float32)
    eng.explain_nodes_host(hp, None, out)
    assert np.isfinite(out).all() and out.min() > 0 and out.max() < 1
    for t in range(0, syn1.N, 9):
        D = plan.dense_of(t, out)
        assert np.array_equal(D, D.T) and np.all(np.diag(D) == 0)
    out2 = np.zeros_like(out)
    eng.explain_nodes_host(hp, None, out2)
    assert np.array_equal(out, out2), "not deterministic"
    # a different order / a sub-batch must give the same bits per node
    perm = np.random.default_rng(0).permutation(syn1.N)[:200]
    plan_p = eng.plan_nodes(perm, 3)
    out_p = np.zeros(plan_p.total_edges, np.float32)
    eng.explain_nodes_host(hp, None, out_p)
    for t, node in enumerate(perm):
        a = out_p[plan_p.edge_off[t]:plan_p.edge_off[t + 1]]
        b = out[plan.edge_off[node]:plan.edge_off[node + 1]]
        assert np.array_equal(a, b), node
    # different seed => different masks (the init really is random)
    out3 = np.zeros_like(out)
    eng.plan_nodes(nodes, 3)
    eng.explain_nodes_host(eng.make_hparams(init=_abi.GX_INIT_PHILOX, seed=99), None, out3)
    assert not np.array_equal(out, out3)
    eng.close()


def test_sharding_is_bit_identical(syn1):
    """Emulates ranks 0/1 of a 2-GPU run on one device: per-node arithmetic never depends on which
    other nodes share the launch."""
    from gnnx.dist import shard_indices
    eng = util.make_engine(syn1)
    nodes = np.array(syn1.nodes)
    plan = eng.plan_nodes(nodes, 3)
    m0 = util.golden_m0(syn1, plan)
    full = np.zeros(plan.total_edges, np.float32)
    eng.explain_nodes_host(eng.make_hparams(), m0, full)
    costs = np.diff(plan.edge_off)
    for rank in range(2):
        pos = shard_indices(len(nodes), 2, rank, costs)
        p = eng.plan_nodes(nodes[pos], 3)
        o = np.zeros(p.total_edges, np.float32)
        eng.explain_nodes_host(eng.make_hparams(), util.golden_m0(syn1, p), o)
        for t, gpos in enumerate(pos):
            assert np.array_equal(o[p.edge_off[t]:p.edge_off[t + 1]], full[plan.edge_off[gpos]:plan.edge_off[gpos + 1]])
    eng.close()


# ------------------------------------------------------------------------------------ drop-in Python surface
def _explainer(fx, tmp_path, **over):
    args = types.SimpleNamespace(num_gc_layers=3, num_epochs=100, lr=0.1, opt="adam", opt_scheduler="none",
                                 mask_act="sigmoid", mask_bias=False, gpu=False, bias=True, method="base",
                                 dataset=fx.name, bmname=None, hidden_dim=20, output_dim=20, name_suffix="",
                                 explainer_suffix="", logdir=str(tmp_path))
    for k, v in over.items():
        setattr(args, k, v)
    model = gnnx.models.GcnEncoderNode(fx.feat.shape[1], 20, 20, fx.weights["Wp"].shape[0], 3, bn=False, args=args)
    sd = {"conv_first.weight": fx.weights["W1"], "conv_first.bias": fx.weights["b1"],
          "conv_block.0.weight": fx.weights["W2"], "conv_block.0.bias": fx.weights["b2"],
          "conv_last.weight": fx.weights["W3"], "conv_last.bias": fx.weights["b3"],
          "pred_model.weight": fx.weights["Wp"], "pred_model.bias": fx.weights["bp"]}
    model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    A = O.dense_from_csr(fx.rowptr, fx.col)
    ex = gnnx.Explainer(model=model, adj=A[None], feat=fx.feat[None].astype(np.float64), label=fx.label[None],
                        pred=fx.pred[None], train_idx=list(range(fx.N)), args=args, writer=None,
                        print_training=False, graph_idx=-1)
    return ex, args


def test_explainer_dropin_reproduces_reference_under_torch_seed(syn1, tmp_path):
    """Explainer.explain with the reference's call sequence: torch.manual_seed(s) then explain(node).
    The M0 draw consumes torch's CPU RNG exactly like ExplainModule.construct_edge_mask, so the
    same seed reproduces the reference's mask."""
    g30 = np.load(util.GOLDEN + "/syn1_golden_e10.npz")
    ex, args = _explainer(syn1, tmp_path, num_epochs=10)
    for node in [300, 450, 683, 13]:
        torch.manual_seed(int(syn1.gold["n%d_seed" % node]))
        masked = ex.explain(node, graph_idx=0)
        n = len(syn1.gold["n%d_nbrs" % node])
        assert isinstance(masked, np.ndarray) and masked.dtype == np.float64 and masked.shape == (n, n)
        idx_new, sub_adj, sub_feat, sub_label, nbrs = ex.extract_neighborhood(node)
        assert np.array_equal(nbrs, syn1.gold["n%d_nbrs" % node]) and idx_new == int(syn1.gold["n%d_idx_new" % node])
        ei, ej = np.nonzero(sub_adj)
        assert util.rel_l2(masked[ei, ej], g30["n%d_mask" % node]) <= 1e-4
        off = masked.copy(); off[ei, ej] = 0
        assert np.all(off == 0)
        f = os.path.join(str(tmp_path), "masked_adj_syn1_base_h20_o20_explainnode_idx_%dgraph_idx_-1.npy" % node)
        assert np.array_equal(np.load(f), masked)                      # explain.py:216-220 side effect
    # batched explain_nodes == the same calls one by one (RNG consumed in node order)
    nodes = [450, 683, 620]
    torch.manual_seed(7)
    one_by_one = [ex.explain(n) for n in nodes]
    torch.manual_seed(7)
    batched = ex.explain_nodes(nodes, args)
    for a, b in zip(one_by_one, batched):
        assert np.array_equal(a, b)
    hop = ex.neighborhoods
    assert hop.shape == (1, syn1.N, syn1.N) and hop[0, 300].sum() == len(syn1.gold["n300_nbrs"])


def test_node_tasks_on_a_batch_of_graphs(syn1, tmp_path):
    """explain.py:80-95 index adj / feat / label / pred with graph_idx: an Explainer built on a batch (B, N, N) of graphs must
    explain node i of graph g exactly like an Explainer built on graph g alone (here: graph 1 = syn1 relabelled by a permutation,
    so graph 0 and graph 1 give different sub-graph orderings for the same node id)."""
    fx = syn1
    rng = np.random.default_rng(3)
    perm = rng.permutation(fx.N)
    A0 = O.dense_from_csr(fx.rowptr, fx.col)
    A1 = A0[perm][:, perm]
    adj = np.stack([A0, A1]); feat = np.stack([fx.feat, fx.feat[perm]]).astype(np.float64)
    label = np.stack([fx.label, fx.label[perm]]); pred = np.stack([fx.pred, fx.pred[perm]])
    ex, args = _explainer(fx, tmp_path, num_epochs=10)
    both = gnnx.Explainer(model=ex.model, adj=adj, feat=feat, label=label, pred=pred, train_idx=list(range(fx.N)), args=args, writer=None,
                          print_training=False, graph_idx=-1)
    only1 = gnnx.Explainer(model=ex.model, adj=adj[1:], feat=feat[1:], label=label[1:], pred=pred[1:], train_idx=list(range(fx.N)), args=args,
                           writer=None, print_training=False, graph_idx=-1)
    for node in (5, 300, 620):
        torch.manual_seed(11 + node); a = both.explain(node, graph_idx=1)
        torch.manual_seed(11 + node); b = only1.explain(node, graph_idx=0)
        assert np.array_equal(a, b)
        torch.manual_seed(11 + node); c = both.explain(node, graph_idx=0)
        torch.manual_seed(11 + node); d = ex.explain(node, graph_idx=0)
        assert np.array_equal(c, d)
        _, sa, sf, sl, nb = both.extract_neighborhood(node, graph_idx=1)
        assert np.array_equal(sa, A1[nb][:, nb]) and np.array_equal(sl, label[1][nb])
    torch.manual_seed(5); batch1 = both.explain_nodes([5, 300], args, graph_idx=1, save=False)
    torch.manual_seed(5); solo1 = only1.explain_nodes([5, 300], args, graph_idx=0, save=False)
    assert all(np.array_equal(x, y) for x, y in zip(batch1, solo1))
    assert both.neighborhoods.shape == (2, fx.N, fx.N)


def test_error_behaviour(tmp_path):
    fx = util.load_fixture("rand")
    eng = util.make_engine(fx)
    with pytest.raises(_abi.GnnxError):
        eng.plan_nodes([fx.N + 5], 3)                                   # out of range
    with pytest.raises(_abi.GnnxError):
        eng.explain_nodes_host(eng.make_hparams(), None, np.zeros(4, np.float32))   # no plan after failure
    # isolated node: the reference's row is empty (it then crashes, explain.py:496-501); we raise
    rowptr = np.concatenate([fx.rowptr, [fx.rowptr[-1]]]).astype(np.int32)
    eng.set_graph_csr(rowptr, fx.col, np.vstack([fx.feat, fx.feat[:1]]), np.append(fx.label, 0), np.append(fx.pred_label, 0))
    with pytest.raises(_abi.GnnxError) as ei:
        eng.plan_nodes([fx.N], 3)
    assert ei.value.status == -4
    # asymmetric adjacency is rejected, not silently symmetrised
    with pytest.raises(_abi.GnnxError):
        eng.set_graph_csr(np.array([0, 1, 1], np.int32), np.array([1], np.int32), np.zeros((2, 16), np.float32), None, np.zeros(2, np.int32))
    # unsupported hyper-parameters fail loudly
    eng2 = util.make_engine(fx)
    eng2.plan_nodes([0], 3)
    with pytest.raises(_abi.GnnxError):
        eng2.explain_nodes_host(eng2.make_hparams(mask_act=1), np.zeros(10000, np.float32), np.zeros(10000, np.float32))
    # --mask-bias is accepted and, as in the reference (tests/test_oracle.py), changes nothing
    pl = eng2.plan_nodes([0, 7], 3)
    m0 = np.random.default_rng(0).normal(1, 0.3, pl.total_edges).astype(np.float32)
    o1 = np.zeros(pl.total_edges, np.float32); o2 = np.zeros(pl.total_edges, np.float32)
    eng2.explain_nodes_host(eng2.make_hparams(num_epochs=10), m0, o1)
    eng2.explain_nodes_host(eng2.make_hparams(num_epochs=10, mask_bias=1), m0, o2)
    assert np.array_equal(o1, o2) and o1.max() > 0
    eng.close(); eng2.close()


# ------------------------------------------------------------------------------------ other layer widths (--hidden-dim / --output-dim)
@pytest.mark.parametrize("hid,emb,d,C", [(16, 12, 10, 3), (32, 32, 7, 2), (8, 28, 5, 4)])
def test_other_widths_match_oracle(hid, emb, d, C):
    """Widths <= 32 run on the 32/32 instantiation with exactly-zero padding (api.cu gx_set_model)."""
    import networkx as nx
    rng = np.random.default_rng(hid * 100 + emb)
    Gx = nx.barabasi_albert_graph(45, 2, seed=hid)
    A = nx.to_numpy_array(Gx)
    N = A.shape[0]
    rowptr, col = O.csr_from_dense(A)
    feat = rng.normal(size=(N, d)).astype(np.float32)
    label = rng.integers(0, C, N)
    sc = lambda *s: (rng.normal(size=s) * 0.5).astype(np.float32)
    w = dict(W1=sc(d, hid), b1=sc(hid), W2=sc(hid, hid), b2=sc(hid), W3=sc(hid, emb), b3=sc(emb), Wp=sc(C, 2 * hid + emb), bp=sc(C))
    Wt = O.weights_to_torch(w, False)
    with torch.no_grad():
        pred = O._gcn_forward_torch(torch.tensor(feat[None]), torch.tensor(A[None], dtype=torch.float), Wt, False)[0].numpy()
    cs = types.SimpleNamespace(N=N, rowptr=rowptr, col=col, feat=feat, label=label, weights=w,
                               pred_label=np.argmax(pred, 1).astype(np.int32))
    eng = util.make_engine(cs)
    nodes = [0, 9, 30, 44]
    plan = eng.plan_nodes(nodes, 3)
    m0 = np.empty(plan.total_edges, np.float32); dense = []
    for t in range(plan.count):
        M0 = O.draw_m0(plan.n(t), seed=hid + t)
        r, c = plan.rows_cols_of(t)
        m0[plan.edge_off[t]:plan.edge_off[t + 1]] = M0[r, c]; dense.append(M0)
    out = np.zeros(plan.total_edges, np.float32)
    eng.explain_nodes_host(eng.make_hparams(num_epochs=20), m0, out)
    for t, node in enumerate(nodes):
        idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(rowptr, col, feat, label, node, 3)
        ref = O.explain_dense_torch(O.dense_from_csr(srp, scol), sfeat, slabel[idx], cs.pred_label[nbrs], idx, w, dense[t],
                                    hp=O.default_hparams(num_epochs=20))
        assert O.rel_l2(plan.dense_of(t, out), ref) <= 1e-4, (node, O.rel_l2(plan.dense_of(t, out), ref))
    eng.close()


def test_gnn_stats_auc_matches_reference(syn1, tmp_path, monkeypatch):
    """Known-answer check downstream of the masks (SURVEY 4 item 3): ROC-AUC of the edge masks against the planted
    house motifs, same nodes and seeds as the reference golden run, within 0.01 of the reference's AUC."""
    import os
    au = np.load(os.path.join(util.GOLDEN, "auc_golden.npz"))
    monkeypatch.chdir(tmp_path)
    ex, args = _explainer(syn1, tmp_path)
    nodes = [int(n) for n in au["syn1_nodes"]]
    # per-node seeds of the golden run: draw M0 node by node exactly as the reference did
    masks = []
    for node in nodes:
        torch.manual_seed(int(syn1.gold["n%d_seed" % node]))
        masks.append(ex.explain_nodes_gnn_stats([node], args)[0])
    torch.manual_seed(0)
    ex.explain_nodes_gnn_stats(nodes, args)
    assert os.path.exists(os.path.join("log", "pr", "auc_syn1_exp.txt"))
    from sklearn.metrics import roc_auc_score
    pr = [ex.make_pred_real(m, int(syn1.gold["n%d_idx_new" % n])) for m, n in zip(masks, nodes)]
    auc = roc_auc_score(np.concatenate([r for _, r in pr]), np.concatenate([p for p, _ in pr]))
    assert abs(auc - float(au["syn1_auc"])) < 0.01, (auc, float(au["syn1_auc"]))


@pytest.mark.parametrize("which", ["syn1", "rand"])
def test_grad_baseline_matches_reference(which, tmp_path):
    """Explainer.explain(model="grad") (explain.py:125-133,717-738): gx_grad_nodes against masks produced by the unmodified
    reference (tests/golden/grad_golden.npz, oracle/gen_golden.py --only grad), shared-memory and streaming kernels."""
    fx = util.load_fixture(which)
    g = np.load(util.GOLDEN + "/grad_golden.npz")
    nodes = [int(x) for x in g[which + "_nodes"]]
    for stream in (False, True):
        eng = util.make_engine(fx)
        if stream:
            eng.debug_force_stream(True)
        plan = eng.plan_nodes(nodes, 3)
        out = np.zeros(plan.total_edges, np.float32)
        eng.grad_nodes_host(out)
        eng.close()
        for t, node in enumerate(nodes):
            ref = g["%s_n%d_mask" % (which, node)]
            got = out[plan.edge_off[t]:plan.edge_off[t + 1]]
            assert len(ref) == len(got)
            assert util.rel_l2(got, ref) <= 1e-5, (which, node, stream, util.rel_l2(got, ref))
            assert np.abs(got - ref).max() <= 1e-5
    if which == "syn1":
        ex, args = _explainer(fx, tmp_path, num_epochs=10)
        masked = ex.explain(300, graph_idx=0, model="grad")
        idx_new, sub_adj, _, _, _ = ex.extract_neighborhood(300)
        ei, ej = np.nonzero(sub_adj)
        assert util.rel_l2(masked[ei, ej], g["syn1_n300_mask"]) <= 1e-5


# ------------------------------------------------------------------------------------ denoise_graph thresholding on device
@pytest.mark.parametrize("which", ["syn1", "syn4"])
def test_denoise_topk_matches_reference(which, tmp_path):
    """gx_denoise_topk + Explainer.denoise_nodes on the reference's own golden masks (so the values are identical) against the
    UNMODIFIED reference's denoise_graph(threshold_num=20) output: thresholded edge set, weights, largest component (bit-exact)."""
    fx = util.load_fixture(which)
    dg = np.load(util.GOLDEN + "/denoise_golden.npz")
    nodes = [int(x) for x in dg[which + "_nodes"]]
    ex, args = _explainer(fx, tmp_path)
    plan = ex.engine.plan_nodes(nodes, 3)
    mask = np.concatenate([fx.gold["n%d_mask" % n] for n in nodes]).astype(np.float32)
    G0s, thr = ex.denoise_nodes(plan, mask, threshold_num=int(dg["threshold_num"]), max_component=False)
    G1s, _ = ex.denoise_nodes(plan, mask, threshold_num=int(dg["threshold_num"]), max_component=True)
    for t, node in enumerate(nodes):
        e = np.array(sorted((min(u, v), max(u, v)) for u, v in G0s[t].edges()), np.int32).reshape(-1, 2)
        assert np.array_equal(e, dg["%s_n%d_edges" % (which, node)]), (which, node)
        assert np.array_equal(np.array([G0s[t][u][v]["weight"] for u, v in e], np.float32), dg["%s_n%d_weights" % (which, node)])
        assert sorted(G1s[t].nodes()) == list(dg["%s_n%d_cc" % (which, node)])
        assert thr[t] == dg["%s_n%d_weights" % (which, node)].min()


def test_denoise_topk_properties_random():
    """Random packed values incl. ties, zeros and a capacity smaller than the number of survivors, against numpy."""
    fx = util.load_fixture("syn1")
    eng = util.make_engine(fx)
    nodes = [0, 3, 300, 683, 13, 699]
    plan = eng.plan_nodes(nodes, 3)
    rng = np.random.default_rng(5)
    vals = rng.random(plan.total_edges).astype(np.float32)
    vals[rng.random(plan.total_edges) < 0.1] = 0.0
    sl = slice(plan.edge_off[2], plan.edge_off[3])
    vals[sl] = np.round(vals[sl] * 8) / 8                      # heavy ties
    vals[plan.edge_off[4]:plan.edge_off[5]] = 0.0              # a task without positive entries
    for k, cap in ((20, 64), (5, 8), (3, 4096)):
        thr, cnt, slots, out_vals = eng.denoise_topk(vals, k, cap=cap)
        for t in range(plan.count):
            v = vals[plan.edge_off[t]:plan.edge_off[t + 1]]
            pos = v[v > 0]
            if len(pos) == 0:
                assert cnt[t] == 0 and np.isinf(thr[t])
                continue
            kk = min(len(pos), 2 * k)
            want_thr = np.sort(pos)[-kk]
            assert thr[t] == want_thr
            keep = np.nonzero(v >= want_thr)[0]
            assert cnt[t] == len(keep)
            m = min(len(keep), cap)
            assert np.array_equal(slots[t, :m], keep[:m]) and np.array_equal(out_vals[t, :m], v[keep[:m]])
            assert np.all(slots[t, m:] == -1)
    eng.close()


def test_destroy_releases_device_memory():
    """gx_destroy frees every device buffer the handle allocated: 20 create / plan / explain / destroy cycles, through the
    shared-memory and the slab kernels, leave the free device memory where it was."""
    fx = util.load_fixture("rand")
    nodes = fx.nodes[:4]

    def cycle():
        for stream in (False, True):
            eng = util.make_engine(fx)
            eng.debug_force_stream(stream)
            plan = eng.plan_nodes(nodes, 3)
            out = np.zeros(plan.total_edges, np.float32)
            eng.explain_nodes_host(eng.make_hparams(num_epochs=10), util.golden_m0(fx, plan), out)
            eng.close()

    cycle()   # loads the kernels the cycle uses: their code stays with the context
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(20):
        cycle()
    free1 = torch.cuda.mem_get_info()[0]
    assert abs(free1 - free0) <= 2 << 20, (free0, free1)
