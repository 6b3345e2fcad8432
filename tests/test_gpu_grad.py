"""GPU (-m gpu): the gradient baseline (Explainer.explain(model="grad"), explain.py:125-133,717-738; gx_grad_nodes) on every kernel that
runs it -- the shared-memory classes and the cluster class of explain_node.cu, explain_gang.cu, explain_stream.cu and the outer-pair
kernel -- against the fp64 closed form (oracle.grad_closed_form; kernel_spec.grad_edges_sparse for large subgraphs), and node mode on
graphs with self loops: the plan, the optimisation masks, the traced mask density and the refused gradient baseline.

Every case checks that it reached the path it exists for (launch class counts, subgraph size, induced degree per hop distance)."""
import types

import networkx as nx
import numpy as np
import pytest
import torch

import dense_oracle as DO
import gnnx
import gnnx_oracle as O
import kernel_spec as KS
import util
from gnnx import _abi
from test_gpu_slab_shapes import _assert_long_rows_regime, _ba_case, _hub_case, _weights
from test_oracle_att import random_att_model

pytestmark = pytest.mark.gpu

SLAB, CLUSTER = 5, 6                         # launch classes of gx_plan_class_counts (0..4: the shared-memory classes)
GANGS = (0, 1, 3, 16)                        # CTAs per task of explain_gang.cu (0 = automatic); -1 = explain_stream.cu
TOL = 1e-5                                   # rel-L2 and max abs per node, as tests/test_gpu_parity.py's grad test


def _engine(cs, force_stream=False, gang=0, cluster=1):
    eng = gnnx.Engine(0)
    eng.set_model(cs.weights, num_layers=cs.L, bn=cs.bn)
    eng.set_graph_csr(cs.rowptr, cs.col, cs.feat, cs.label, cs.pred_label)
    eng.debug_force_stream(force_stream)
    eng.debug_gang(gang)
    eng.debug_cluster(cluster, 1)
    return eng


def _grad(eng, nodes, L=3):
    plan = eng.plan_nodes(nodes, L)
    out = np.zeros(plan.total_edges, np.float32)
    eng.grad_nodes_host(out)
    return plan, out


def _random_labels(cs, seed):
    """Labels and predicted labels drawn independently: most nodes have pred_label != label."""
    rng = np.random.default_rng(seed)
    C = cs.weights["Wp"].shape[0]
    cs.label = rng.integers(0, C, cs.N).astype(np.int32)
    cs.pred_label = rng.integers(0, C, cs.N).astype(np.int32)
    return cs


def _spec(cs, plan, sparse=False):
    """fp64 gradient baseline of every task at its CSR slots."""
    res = []
    for t in range(plan.count):
        rp, col = plan.csr_of(t)
        nbrs = plan.neighbors_of(t)
        idx = int(plan.node_idx_new[t])
        pl = int(cs.pred_label[int(plan.nodes[t])])
        if sparse:
            res.append(KS.grad_edges_sparse(rp, col, cs.feat[nbrs], pl, idx, cs.weights)[0])
        else:
            r, c = plan.rows_cols_of(t)
            res.append(O.grad_closed_form(O.dense_from_csr(rp, col), cs.feat[nbrs], pl, idx, cs.weights)[r, c])
    return res


def _check(plan, out, spec, what, L=3):
    """Every task within TOL of the spec; every slot of an edge between two distance-L nodes exactly 0.5f.  -> number of such slots."""
    outer_slots = 0
    for t in range(plan.count):
        got = out[plan.edge_off[t]:plan.edge_off[t + 1]]
        err, mx = util.rel_l2(got, spec[t]), float(np.abs(got - spec[t]).max()) if len(got) else 0.0
        assert err <= TOL and mx <= TOL, (what, int(plan.nodes[t]), err, mx)
        rp, col = plan.csr_of(t)
        dist = KS.hop_distances(rp, col, int(plan.node_idx_new[t]), L)
        ei = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
        outer = (dist[ei] == L) & (dist[col] == L)
        assert (got[outer] == np.float32(0.5)).all(), (what, int(plan.nodes[t]))
        outer_slots += int(outer.sum())
    return outer_slots


# ------------------------------------------------------------------------------------------------ shared-memory classes 0..4
COMPONENTS = (2, 3, 4, 6, 9, 14, 20, 30, 45, 70, 100, 150, 220, 330, 500, 900, 1400, 2200)
STAR = 40                                    # leaves of the star component: its centre's row has more than kLongRow = 32 edges


def _components_case(seed, d, C, hid, emb):
    """Disjoint components of growing size (one edge, a 3-node path, then BA graphs): the k-hop sets range from 2 nodes to a few
    thousand, so one batch spans the shared-memory classes; the larger components have hubs with far more than kLongRow = 32 induced
    edges.  A star of STAR leaves (centre cs.star) is small enough for the shared-memory classes at every d."""
    rng = np.random.default_rng(seed)
    edges, starts, base = [], [], 0
    for s in COMPONENTS:
        G = nx.path_graph(s) if s < 4 else nx.barabasi_albert_graph(s, 2, seed=seed + s)
        edges += [(base + a, base + b) for a, b in G.edges()]
        starts.append(base)
        base += s
    edges += [(base, base + k) for k in range(1, STAR + 1)]
    N = base + STAR + 1
    rowptr, col = O.csr_from_edges(N, np.array(edges, np.int64))
    cs = types.SimpleNamespace(N=N, rowptr=rowptr, col=col, feat=rng.normal(size=(N, d)).astype(np.float32),
                               weights=_weights(rng, d, C, hid, emb), L=3, bn=False, starts=starts, star=base)
    return _random_labels(cs, seed + 1)


def _one_per_class(eng, cs, lowest=None):
    """One node of every shared-memory class the model reaches, found by planning candidates one at a time.  The model's fixed share
    of shared memory (weights, pred_model up to C = 21) grows with d, widths and C, so the smallest classes only hold small models: the
    classes found must run from the class of the 2-node task (the smallest task there is) up to class 4 without a gap.  lowest: the
    class the 2-node task must land in."""
    found = {}
    for b, s in zip(cs.starts, COMPONENTS):
        for node in sorted({b, b + 1, b + s // 3, b + s // 2, b + s - 1}):
            eng.plan_nodes([node], 3)
            c = int(np.argmax(eng.plan_class_counts()[0]))
            if c < SLAB:
                found.setdefault(c, node)
    lo = min(found)
    assert found[lo] == cs.starts[0] and sorted(found) == list(range(lo, 5)), sorted(found)
    assert lowest is None or lo == lowest, sorted(found)
    return [found[c] for c in range(lo, 5)]


SMEM_CASES = [   # (hid, emb, d, C, the lowest class reachable: 0 wherever the model is small enough for every class)
    (20, 20, 10, 2, 0), (20, 20, 1, 40, 0), (16, 12, 1, 21, None), (32, 32, 33, 40, None), (20, 20, 64, 40, None), (16, 12, 128, 2, None),
    (32, 32, 128, 21, None)]


@pytest.mark.parametrize("hid,emb,d,C,lowest", SMEM_CASES, ids=["h%de%d_d%d_C%d" % c[:4] for c in SMEM_CASES])
def test_grad_shared_memory_classes_match_closed_form(hid, emb, d, C, lowest):
    """One batch with a task in each shared-memory class the model reaches (all of 0..4 for the small models) and the star's centre
    (a row of more than 32 induced edges), against the fp64 closed form; outer edges exactly 0.5."""
    cs = _components_case(100 + d + C, d, C, hid, emb)
    eng = _engine(cs)
    nodes = _one_per_class(eng, cs, lowest)
    lo = 5 - len(nodes)
    nodes.append(cs.star)
    plan, out = _grad(eng, nodes)
    counts = eng.plan_class_counts()[0]
    eng.close()
    assert counts[:lo].sum() == 0 and (counts[lo:5] >= 1).all() and counts[:5].sum() == len(nodes), counts
    assert max(np.diff(plan.csr_of(t)[0]).max() for t in range(plan.count)) > 32
    assert any(cs.pred_label[n] != cs.label[n] for n in nodes)
    assert _check(plan, out, _spec(cs, plan), (hid, emb, d, C)) > 0


# ------------------------------------------------------------------------------------------------ cluster class
@pytest.mark.parametrize("cs_size", [2, 4])
def test_grad_cluster_class_matches_closed_form(cs_size):
    """explain_node.cu on thread-block clusters of 2 / 4 CTAs: against the closed form and the single-CTA run."""
    cs = _random_labels(_ba_case(50, 60, 3, 33, 22, 24, 17), 51)
    nodes = [0, 5, 12, 31, 59]
    res = {}
    for size in (1, cs_size):
        eng = _engine(cs, cluster=size)
        plan, out = _grad(eng, nodes)
        counts, csz = eng.plan_class_counts()
        eng.close()
        assert counts[CLUSTER] == (len(nodes) if size > 1 else 0) and csz == size, (counts, csz)
        res[size] = out
    assert _check(plan, res[cs_size], _spec(cs, plan), ("cluster", cs_size)) > 0
    assert np.abs(res[cs_size] - res[1]).max() <= 1e-6


# ------------------------------------------------------------------------------------------------ slab kernels
@pytest.mark.parametrize("seed,N,d,C,hid,emb", [(21, 48, 33, 21, 32, 32), (22, 60, 10, 4, 20, 20), (23, 40, 128, 40, 16, 12)],
                         ids=["h32_d33", "h20_d10", "h16e12_d128"])
def test_grad_slab_kernels_match_closed_form(seed, N, d, C, hid, emb):
    """Forced into the slab class: explain_gang.cu with 1 / 3 / 16 CTAs per task and automatic bit-identical, explain_stream.cu
    (gang -1) and the gang kernel against the closed form."""
    cs = _random_labels(_ba_case(seed, N, 2, d, C, hid, emb), seed)
    nodes = list(range(0, N, N // 5))[:5]
    res = {}
    for gang in GANGS + (-1,):
        eng = _engine(cs, force_stream=True, gang=gang)
        plan, res[gang] = _grad(eng, nodes)
        assert eng.plan_class_counts()[0][SLAB] == len(nodes)
        eng.close()
    spec = _spec(cs, plan)
    for gang in (0, -1):
        assert _check(plan, res[gang], spec, gang) > 0
    for gang in GANGS[1:]:
        assert np.array_equal(res[gang], res[0]), gang


def test_grad_hub_rows_match_sparse_spec():
    """Rows of 511 / 512 / 513 and >= 2000 induced edges at hop distance 0..3 (explain_gang.cu slices rows over 512 edges across a
    CTA): both slab kernels against the sparse fp64 spec, gang sizes bit-identical."""
    cs = _hub_case()
    nodes = cs.g.hub_nodes
    res = {}
    for gang in (0, 1, 16, -1):
        eng = _engine(cs, gang=gang)
        plan, res[gang] = _grad(eng, nodes)
        assert eng.plan_class_counts()[0][SLAB] == len(nodes)
        eng.close()
    _assert_long_rows_regime(plan)
    spec = _spec(cs, plan, sparse=True)
    for gang in (0, -1):
        assert _check(plan, res[gang], spec, ("hub", gang)) > 0
    for gang in (1, 16):
        assert np.array_equal(res[gang], res[0]), gang


def test_grad_config5_sized_subgraph_matches_sparse_spec():
    """BA(90 000, 4), d = 128: the highest-degree node's 3-hop set (n >= 65 535) reaches the slab class without any knob."""
    N, d, C = 90000, 128, 4
    rowptr, col = O.csr_from_edges(N, np.array(nx.barabasi_albert_graph(N, 4, seed=0).edges(), dtype=np.int64))
    rng = np.random.default_rng(5)
    cs = types.SimpleNamespace(N=N, rowptr=rowptr, col=col, feat=rng.normal(size=(N, d)).astype(np.float32),
                               weights=_weights(rng, d, C, 20, 20), L=3, bn=False)
    _random_labels(cs, 6)
    hub = int(np.argmax(np.diff(rowptr)))
    eng = _engine(cs)
    plan, out = _grad(eng, [hub])
    counts = eng.plan_class_counts()[0]
    eng.close()
    assert counts[SLAB] == 1 and counts.sum() == 1, counts
    assert plan.n(0) >= 65535
    spec = _spec(cs, plan, sparse=True)
    print("config-5 subgraph: n %d, E_d %d; rel-L2 %.2e, max abs %.2e vs the fp64 spec"
          % (plan.n(0), plan.total_edges, util.rel_l2(out, spec[0]), np.abs(out - spec[0]).max()))
    assert _check(plan, out, spec, "config5") > 0


# ------------------------------------------------------------------------------------------------ labels, batch independence
PATHS = {"smem": dict(), "cluster": dict(cluster=2), "gang": dict(force_stream=True), "stream1": dict(force_stream=True, gang=-1)}


@pytest.mark.parametrize("path", list(PATHS))
def test_grad_follows_predicted_label(path):
    """The loss is taken at pred_label: changing label leaves the output bit-identical, changing pred_label changes every task."""
    cs = _random_labels(_ba_case(31, 50, 2, 10, 5, 20, 20), 32)
    nodes = [0, 9, 17, 33, 49]
    assert sum(cs.pred_label[n] != cs.label[n] for n in nodes) >= 2
    outs = []
    for label, pred_label in ((cs.label, cs.pred_label), ((cs.label + 1) % 5, cs.pred_label), (cs.label, (cs.pred_label + 1) % 5)):
        eng = _engine(types.SimpleNamespace(**{**vars(cs), "label": label.astype(np.int32), "pred_label": pred_label.astype(np.int32)}),
                      **PATHS[path])
        plan, out = _grad(eng, nodes)
        counts = eng.plan_class_counts()[0]
        eng.close()
        assert counts[{"smem": slice(0, 5), "cluster": CLUSTER}.get(path, SLAB)].sum() == len(nodes), counts
        outs.append(out)
    assert _check(plan, outs[0], _spec(cs, plan), path) > 0
    assert np.array_equal(outs[0], outs[1])
    for t in range(plan.count):
        s = slice(plan.edge_off[t], plan.edge_off[t + 1])
        assert not np.array_equal(outs[0][s], outs[2][s]), (path, nodes[t])


def test_grad_batch_independent():
    """A node's output is bit-identical alone, inside the mixed-class batch and in shuffled order."""
    cs = _components_case(7, 10, 4, 20, 20)
    eng = _engine(cs)
    nodes = _one_per_class(eng, cs)
    plan, out = _grad(eng, nodes)
    got = {n: out[plan.edge_off[t]:plan.edge_off[t + 1]] for t, n in enumerate(nodes)}
    shuffled = [nodes[i] for i in (3, 0, 4, 2, 1)]
    p2, o2 = _grad(eng, shuffled)
    for t, n in enumerate(shuffled):
        assert np.array_equal(o2[p2.edge_off[t]:p2.edge_off[t + 1]], got[n]), n
        _, o1 = _grad(eng, [n])
        assert np.array_equal(o1, got[n]), n
    eng.close()


# ------------------------------------------------------------------------------------------------ the drop-in
def _dropin(rowptr, col, A, feat, label, pred_label, w, hid, emb, tmp_path, L=3):
    args = types.SimpleNamespace(num_gc_layers=L, num_epochs=10, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                 mask_bias=False, gpu=False, bias=True, method="base", dataset="grad", bmname=None, hidden_dim=hid,
                                 output_dim=emb, name_suffix="", explainer_suffix="", logdir=str(tmp_path))
    C = w["Wp"].shape[0]
    model = gnnx.models.GcnEncoderNode(feat.shape[1], hid, emb, C, L, bn=False, args=args)
    sd = {"conv_first.weight": w["W1"], "conv_first.bias": w["b1"], "conv_block.0.weight": w["W2"], "conv_block.0.bias": w["b2"],
          "conv_last.weight": w["W3"], "conv_last.bias": w["b3"], "pred_model.weight": w["Wp"], "pred_model.bias": w["bp"]}
    model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    pred = np.eye(C, dtype=np.float32)[pred_label][None]
    return gnnx.Explainer(model=model, adj=A[None], feat=feat[None].astype(np.float64), label=label[None], pred=pred,
                          train_idx=list(range(len(feat))), args=args, writer=None, print_training=False, graph_idx=-1)


def test_grad_dropin_on_gang_class_node(tmp_path):
    """Explainer.explain(node, model="grad") on a node whose subgraph exceeds shared memory (explain_gang.cu): the dense array
    against the closed form."""
    cs = _hub_case()
    node = cs.g.hubs[513]
    A = O.dense_from_csr(cs.rowptr, cs.col)
    ex = _dropin(cs.rowptr, cs.col, A, cs.feat, cs.label, cs.pred_label, cs.weights, 20, 20, tmp_path)
    masked = ex.explain(node, model="grad")
    assert ex.engine.plan_class_counts()[0][SLAB] == 1
    idx, sub_adj, sub_feat, _, nbrs = ex.extract_neighborhood(node)
    ref = O.grad_closed_form(sub_adj, cs.feat[nbrs], cs.pred_label[node], idx, cs.weights)
    r, c = np.nonzero(sub_adj)
    assert (masked[sub_adj == 0] == 0).all()
    assert util.rel_l2(masked[r, c], ref[r, c]) <= TOL and np.abs(masked - ref).max() <= TOL


# ------------------------------------------------------------------------------------------------ node mode with self loops
def _loop_case(seed=3, N=60, d=10, C=4, hid=20, emb=20, L=3, bn=False, att=False):
    """BA(N, 2) with a self loop on about a third of its nodes, a separate loop-free BA(20, 2) component, and one isolated node
    whose only edge is its self loop."""
    rng = np.random.default_rng(seed)
    M = N + 20 + 1
    A = np.zeros((M, M))
    for a, b in nx.barabasi_albert_graph(N, 2, seed=seed).edges():
        A[a, b] = A[b, a] = 1
    for a, b in nx.barabasi_albert_graph(20, 2, seed=seed + 1).edges():
        A[N + a, N + b] = A[N + b, N + a] = 1
    loops = np.zeros(M, bool)
    loops[:N] = rng.random(N) < 0.35
    loops[M - 1] = True
    A[np.arange(M), np.arange(M)] = loops
    rowptr, col = O.csr_from_dense(A)
    feat = rng.normal(size=(M, d)).astype(np.float32)
    w = random_att_model(rng, d, hid, emb, C, L) if att else _weights(rng, d, C, hid, emb, L)
    hop = O.neighborhoods_dense(A[None], L)[0]
    looped = [n for n in range(0, N, 3) if loops[hop[n] > 0].any()][:10]     # nodes with a self loop in their neighbourhood
    assert len(looped) == 10 and not any(loops[hop[n] > 0].any() for n in range(N, N + 20))
    cs = types.SimpleNamespace(N=M, A=A, rowptr=rowptr, col=col, feat=feat, weights=w, L=L, bn=bn, att=att, loops=loops,
                               looped=looped, clean=[N, N + 7, N + 19], iso=M - 1)
    return _random_labels(cs, seed + 2)


def _loop_engine(cs, **knobs):
    eng = gnnx.Engine(0)
    eng.set_model(cs.weights, num_layers=cs.L, bn=cs.bn, att=[cs.weights["Wa%d" % l] for l in range(1, cs.L + 1)] if cs.att else None)
    eng.set_graph_csr(cs.rowptr, cs.col, cs.feat, cs.label, cs.pred_label)
    eng.debug_force_stream(knobs.get("force_stream", False))
    eng.debug_gang(knobs.get("gang", 0))
    return eng


def _reference_subgraph(cs, node):
    """The reference's extract_neighborhood (explain.py:492-501) on the dense adjacency, self loops included."""
    hop = O.neighborhoods_dense(cs.A[None], cs.L)[0]
    nbrs = np.nonzero(hop[node])[0]
    return int(hop[node][:node].sum()), cs.A[nbrs][:, nbrs], nbrs


def test_self_loop_plan_matches_reference(tmp_path):
    """neighbors, node_idx_new and the sub-adjacency of the plan bit for bit against the reference's extraction with the diagonal
    removed (the CSR oracle agrees); the drop-in's extract_neighborhood keeps the diagonal, as adj[nbrs][:, nbrs] does.  The isolated
    self-loop node is a task of n = 1 and no edge."""
    cs = _loop_case()
    eng = _loop_engine(cs)
    nodes = cs.looped + cs.clean + [cs.iso]
    plan = eng.plan_nodes(nodes, 3)
    eng.close()
    for t, node in enumerate(nodes):
        idx, sub, nbrs = _reference_subgraph(cs, node)
        assert np.array_equal(plan.neighbors_of(t), nbrs) and int(plan.node_idx_new[t]) == idx, node
        rp, col = plan.csr_of(t)
        ref_rp, ref_col = O.csr_from_dense(sub * (1 - np.eye(len(nbrs))))
        assert np.array_equal(rp, ref_rp) and np.array_equal(col, ref_col), node
        oidx, orp, ocol, _, _, onbrs = O.extract_neighborhood(cs.rowptr, cs.col, cs.feat, cs.label, node, 3)
        keep = np.repeat(np.arange(len(onbrs)), np.diff(orp)) != ocol
        assert np.array_equal(onbrs, nbrs) and oidx == idx and np.array_equal(ocol[keep], col), node
    t_iso = nodes.index(cs.iso)
    assert plan.n(t_iso) == 1 and plan.edge_off[t_iso + 1] == plan.edge_off[t_iso]
    assert sum(np.diag(_reference_subgraph(cs, n)[1]).sum() for n in cs.looped) > 0
    ex = _dropin(cs.rowptr, cs.col, cs.A, cs.feat, cs.label, cs.pred_label, cs.weights, 20, 20, tmp_path)
    for node in cs.looped[:4] + [cs.iso]:
        idx, sub, nbrs = _reference_subgraph(cs, node)
        got = ex.extract_neighborhood(node)
        assert got[0] == idx and np.array_equal(got[1], sub) and np.array_equal(got[4], nbrs), node


def _port(cs, sub, X, gt, pl, idx, M0, E, path):
    """(fp32 port, its fp64 restatement) of the optimisation on the reference's sub_adj, diagonal included."""
    hp = O.default_hparams(num_epochs=E)
    if path == "att":
        return (O.explain_dense_torch(sub, X, gt, pl, idx, cs.weights, M0, hp, bn=cs.bn),
                O.explain_dense_torch(sub, X, gt, pl, idx, cs.weights, M0, hp, bn=cs.bn, dtype=torch.float64))
    if path == "unconstrained":
        return (O.explain_dense_torch(sub, X, gt, pl, idx, cs.weights, M0, hp, bn=cs.bn, unconstrained=True),
                DO.explain_closed_form(sub, X, gt, pl, idx, cs.weights, M0, hp, bn=cs.bn))
    return (O.explain_dense_torch(sub, X, gt, pl, idx, cs.weights, M0, hp=hp, bn=cs.bn),
            O.explain_closed_form(sub, X, gt, pl, idx, cs.weights, M0, hp=hp, bn=cs.bn))


LOOP_PATHS = {"smem": dict(), "gang": dict(force_stream=True), "stream1": dict(force_stream=True, gang=-1),
              "var_L2_bn": dict(L=2, bn=True), "att": dict(att=True), "unconstrained": dict()}


@pytest.mark.parametrize("path", list(LOOP_PATHS))
def test_self_loop_masks_match_port(path):
    """The optimisation on graphs with self loops (diag_mask removes them) against the port on the reference's sub_adj with its
    diagonal, 20 epochs; the n = 1 task returns [[0.]]."""
    kn = LOOP_PATHS[path]
    cs = _loop_case(L=kn.get("L", 3), bn=kn.get("bn", False), att=kn.get("att", False))
    eng = _loop_engine(cs, **kn)
    nodes = cs.looped[:5] + cs.clean[:1] + [cs.iso]
    plan = eng.plan_nodes(nodes, cs.L)
    counts = eng.plan_class_counts()[0]
    E = 20
    dense = [O.draw_m0(plan.n(t), seed=70 + t) for t in range(plan.count)]
    out = np.zeros(plan.total_edges, np.float32)
    if path == "unconstrained":
        eng.explain_nodes_unconstrained(eng.make_hparams(num_epochs=E), np.concatenate([D.reshape(-1) for D in dense]), out)
    else:
        m0 = np.concatenate([D[plan.rows_cols_of(t)] for t, D in enumerate(dense)]).astype(np.float32)
        eng.explain_nodes_host(eng.make_hparams(num_epochs=E), m0, out)
    eng.close()
    if path in ("gang", "stream1", "var_L2_bn", "att"):
        assert counts[SLAB] == len(nodes), counts
    elif path == "smem":
        assert counts[:5].sum() == len(nodes), counts
    for t, node in enumerate(nodes):
        idx, sub, nbrs = _reference_subgraph(cs, node)
        port, p64 = _port(cs, sub, cs.feat[nbrs], cs.label[node], cs.pred_label[nbrs], idx, dense[t], E, path)
        got = plan.dense_of(t, out)
        if node == cs.iso:
            assert got.shape == (1, 1) and got[0, 0] == 0.0 and port[0, 0] == 0.0
            continue
        tol = max(1e-4, 3 * O.rel_l2(p64, port))
        assert O.rel_l2(got, port) <= tol, (path, node, O.rel_l2(got, port), tol)


@pytest.mark.parametrize("unconstrained", [False, True], ids=["tuned", "unconstrained"])
def test_self_loop_trace_density_matches_port(unconstrained):
    """print_training's mask density divides by sum(adj), self loops included (explain.py:680-683): the trace's density column
    against the port's at every epoch, to 1e-6."""
    cs = _loop_case()
    eng = _loop_engine(cs)
    nodes = cs.looped[:4] + cs.clean[:1] + [cs.iso]
    plan = eng.plan_nodes(nodes, 3)
    E = 12
    C = cs.weights["Wp"].shape[0]
    dense = [O.draw_m0(plan.n(t), seed=90 + t) for t in range(plan.count)]
    hp = eng.make_hparams(num_epochs=E)
    out = np.zeros(plan.total_edges, np.float32)
    trace = np.zeros((plan.count, E, _abi.GX_TRACE_COLS), np.float32)
    pred = np.zeros((plan.count, E, C), np.float32)
    if unconstrained:
        eng.explain_nodes_unconstrained(hp, np.concatenate([D.reshape(-1) for D in dense]), out, trace=trace, trace_pred=pred)
    else:
        m0 = np.concatenate([D[plan.rows_cols_of(t)] for t, D in enumerate(dense)]).astype(np.float32)
        eng.explain_nodes_ex(hp, m0, out, trace=trace, trace_pred=pred)
    eng.close()
    for t, node in enumerate(nodes):
        idx, sub, nbrs = _reference_subgraph(cs, node)
        tr = []
        args = (sub, cs.feat[nbrs], cs.label[node], cs.pred_label[nbrs], idx, cs.weights, dense[t])
        if unconstrained:
            O.explain_dense_torch(*args, hp=O.default_hparams(num_epochs=E), trace=tr, unconstrained=True)
        else:
            O.explain_dense_torch(*args, hp=O.default_hparams(num_epochs=E), trace=tr)
        want = np.array([e["density"] for e in tr])
        assert np.abs(trace[t, :, _abi.TR_DENSITY] - want).max() <= 1e-6, (node, trace[t, :, _abi.TR_DENSITY], want)


def test_grad_refuses_self_loops(tmp_path):
    """gx_grad_nodes refuses a plan with a self loop in some neighbourhood (GX_ERR_UNSUPPORTED naming the node) -- the reference's
    result would differ off the diagonal and have a diagonal entry >= 0.5; the drop-in raises NotImplementedError without consuming
    torch's RNG.  Loop-free neighbourhoods of the same graph still run, against the closed form."""
    cs = _loop_case()
    eng = _loop_engine(cs)
    for nodes in ([cs.looped[1]], cs.clean + [cs.looped[2]], [cs.iso]):
        plan = eng.plan_nodes(nodes, 3)
        with pytest.raises(_abi.GnnxError) as e:
            eng.grad_nodes_host(np.zeros(max(plan.total_edges, 1), np.float32))
        assert e.value.status == -3 and "node %d" % nodes[-1] in str(e.value), str(e.value)
    plan, out = _grad(eng, cs.clean)
    eng.close()
    assert _check(plan, out, _spec(cs, plan), "loop-free") >= 0
    ex = _dropin(cs.rowptr, cs.col, cs.A, cs.feat, cs.label, cs.pred_label, cs.weights, 20, 20, tmp_path)
    state = torch.get_rng_state()
    with pytest.raises(NotImplementedError, match="self loop"):
        ex.explain(cs.looped[1], model="grad")
    assert torch.equal(torch.get_rng_state(), state)
    masked = ex.explain(cs.clean[0], model="grad")
    assert not torch.equal(torch.get_rng_state(), state)          # the loop-free call draws its n^2 normals like the reference
    idx, sub, nbrs = _reference_subgraph(cs, cs.clean[0])
    assert np.abs(masked - O.grad_closed_form(sub, cs.feat[nbrs], cs.pred_label[cs.clean[0]], idx, cs.weights)).max() <= TOL
