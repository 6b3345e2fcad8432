"""GPU (-m gpu): exact ties in graph mode's max-pool readout, on every graph kernel.  The readout's backward sends each pooled column's
gradient to one row, the first maximal one (torch.max); these batches make ties on purpose, which random inputs never do:

  * twin leaves: two leaves with identical features on the same hub, whose four edge entries of M0 are equal, so their rows are equal
    in every layer at epoch 0 -- at low and high indices, separated by an isolated node, after an isolated node at index 0;
  * ties with the edge-less constant: a component whose features are all zero (its layer-1 rows are the constant), after an isolated
    atom (torch and the kernels both take a row without gradient) and at index 0 (torch takes row 0, a row with edges; the kernels take
    the constant -- both send nothing to M or F, so the masks must agree);
  * a ReLU column that is 0 in every row and in the constant (W1 column 0 is zero, b1[0] negative).

Each kernel is checked against the fp64 torch port (tests/pool_oracle.py): one update within 1e-5 with the twins' edge-mask
difference within 1e-6 of the port's (so a kernel that routed a twin tie to the other twin fails), and ten Adam epochs within 1e-4 on
the graph whose ties are with the constant."""
import numpy as np
import pytest
import torch

import gnnx
import gnnx_oracle as O
import pool_oracle as PO
from test_gpu_deep import _hp, random_model
from test_gpu_head import head_model

pytestmark = pytest.mark.gpu

N = 12
# (edges, twin pairs (t1, t2, hub), zero-feature nodes)
GRAPHS = [
    ([(0, 2), (1, 2), (2, 3), (3, 4), (4, 5), (5, 6), (3, 6)], [(0, 1, 2)], []),            # twins at the lowest indices
    ([(0, 1), (1, 2), (2, 3), (3, 4), (4, 10), (4, 11)], [(10, 11, 4)], []),                 # twins at the highest, isolated rows before
    ([(1, 2), (2, 3), (2, 5), (2, 6), (6, 7), (1, 7)], [(3, 5, 2)], []),                     # isolated 0; twins 3, 5 around isolated 4
    ([(1, 2), (2, 3), (1, 3), (5, 6), (6, 7), (7, 8), (5, 8), (8, 9)], [], [1, 2, 3]),       # isolated 0; a zero-feature triangle
    ([(0, 1), (1, 2), (0, 2), (3, 4), (4, 5), (5, 6), (3, 6), (6, 7)], [], [0, 1, 2]),       # a zero-feature triangle at 0
]
CONSTANT_TIES = [3, 4]   # the graphs whose ties are with the edge-less constant


def _batch(d, seed):
    rng = np.random.default_rng(seed)
    G = len(GRAPHS)
    adj = np.zeros((G, N, N), np.float32)
    feat = np.zeros((G, N, d), np.float32)
    m0 = []
    for g, (edges, twins, zero) in enumerate(GRAPHS):
        for i, j in edges:
            adj[g, i, j] = adj[g, j, i] = 1
        deg = adj[g].sum(1) > 0
        feat[g] = rng.normal(size=(N, d)) * deg[:, None]
        feat[g, zero] = 0
        M0 = O.draw_m0(N, seed=100 * seed + g)
        for t1, t2, hub in twins:
            feat[g, t2] = feat[g, t1]
            M0[t2, hub] = M0[hub, t1] = M0[hub, t2] = M0[t1, hub]
        m0.append(M0)
    return adj, feat, np.arange(G, dtype=np.int32) % 3, m0


def _model(kind, d):
    """(weights, L, bn, att list, head) of a graph path; W1's column 0 is zero and b1[0] negative: an all-zero ReLU column."""
    rng = np.random.default_rng(7)
    L, bn, att, hid, emb, widths = dict(tuned20=(3, False, False, 20, 20, None), tuned32=(3, False, False, 32, 32, None),
                                        kw1=(3, True, False, 20, 20, None), kw2=(2, True, False, 64, 48, None),
                                        kw4=(4, True, False, 128, 100, None), kblk=(3, True, False, 160, 136, None),
                                        att=(3, False, True, 24, 24, None), head=(3, True, False, 32, 32, [40]),
                                        wide=(3, False, False, 32, 32, None), dense=(3, False, False, 20, 20, None))[kind]
    w = head_model(rng, d, hid, emb, 3, L, widths) if widths else random_model(rng, d, hid, emb, 3, L, att)
    w["W1"][:, 0] = 0
    w["b1"][0] = -0.5
    return w, L, bn


def _nobias(w, L):
    return dict(w, **{"b%d" % l: None for l in range(1, L + 1)})


PATHS = [("tuned20", 8, True), ("tuned20", 8, False), ("tuned32", 8, True), ("kw1", 8, True), ("kw2", 8, True), ("kw4", 8, True),
         ("kblk", 8, True), ("att", 8, True), ("head", 8, True), ("wide", 300, True), ("dense", 8, True)]


def _run(kind, d, bias, E, gids=None, **over):
    w, L, bn = _model(kind, d)
    if not bias:
        w = _nobias(w, L)
    adj, feat, label, m0 = _batch(d, 3)
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bn, att=[w["Wa%d" % l] for l in range(1, L + 1)] if "Wa1" in w else None, head=w.get("head"))
    eng.set_graph_batch(adj, feat, label)
    gids = gids or list(range(len(GRAPHS)))
    edge_off = eng.plan_graphs(gids)
    rc = [eng.graph_rows_cols(g) for g in gids]
    out = np.zeros(int(edge_off[-1]), np.float32)
    fm = np.zeros((len(gids), d), np.float32)
    hp = _hp(eng, E, **over)
    if kind == "dense":
        eng.explain_graphs_unconstrained(hp, np.concatenate([m0[g].reshape(-1) for g in gids]).astype(np.float32), out)
        fm = None
    else:
        eng.explain_graphs_host(hp, np.concatenate([m0[g][rc[t]] for t, g in enumerate(gids)]).astype(np.float32), out, fm)
    eng.close()
    res = []
    for t, g in enumerate(gids):
        Dm = np.zeros((N, N))
        Dm[rc[t]] = out[edge_off[t]:edge_off[t + 1]]
        ref, f64 = PO.explain_torch_pool(adj[g].astype(np.float64), feat[g], int(label[g]), w, m0[g], O.default_hparams(num_epochs=E, **over),
                                         bn=bn,
                                         dtype=torch.float64, unconstrained=kind == "dense")
        res.append((g, adj[g].astype(np.float64), Dm, None if fm is None else fm[t], ref, f64))
    return res


@pytest.mark.parametrize("kind,d,bias", PATHS, ids=lambda v: str(v))
def test_exact_ties_one_update_match_fp64_port(kind, d, bias):
    """One update of Adam with eps = 1 (the step grows with the gradient instead of being +-lr, so the routed pooled gradient shows
    in the twins' edge masks)."""
    routed = 0.0
    for g, A, Dm, fm, ref, f64 in _run(kind, d, bias, 2, eps=1.0):
        ei, ej = np.nonzero(A)
        assert O.rel_l2(Dm[ei, ej], ref[ei, ej]) <= 1e-5, (kind, g, O.rel_l2(Dm[ei, ej], ref[ei, ej]))
        if fm is not None:
            assert np.abs(fm - f64).max() <= 1e-5, (kind, g)
        if kind == "dense":
            continue   # the dense mask's other entries of the twins' rows differ: no tie there, only the mask comparison above
        for t1, t2, hub in GRAPHS[g][1]:
            dk, dp = Dm[t1, hub] - Dm[t2, hub], ref[t1, hub] - ref[t2, hub]
            assert abs(dk - dp) <= 1e-6, (kind, g, dk, dp)
            routed = max(routed, abs(dp))
    if kind != "dense" and bias:
        assert routed > 1e-4   # the tie routes a real gradient: a kernel sending it to the other twin fails above


@pytest.mark.parametrize("kind,d,bias", PATHS, ids=lambda v: str(v))
def test_constant_ties_ten_epochs_match_fp64_port(kind, d, bias):
    """Ten epochs on the batch whose ties are with the edge-less constant and in the all-zero ReLU column (they carry no gradient).
    Twins are not checked past one update: once they part, their rows are near ties in every later epoch."""
    w, L, bn = _model(kind, d)
    adj, feat, label, m0 = _batch(d, 3)
    for g, A, Dm, fm, ref, f64 in _run(kind, d, bias, 10, gids=CONSTANT_TIES):
        ei, ej = np.nonzero(A)
        # the nearest admissible trajectory: the fp64 port's, or an fp32 one with a near tie of a later epoch taken the other way (the
        # KW = 2 model has one, at epoch 1, and the kernel lands 1.80e-4 from the fp64 port, where the flipped fp32 port lands)
        cands = [(ref, f64)] + [(m, f) for flip, m, f in PO.admissible(A, feat[g], int(label[g]), w if bias else _nobias(w, L),
                                                                        m0[g], O.default_hparams(num_epochs=10), bn,
                                                                        unconstrained=kind == "dense") if flip is not None]
        errs = [(O.rel_l2(Dm[ei, ej], m[ei, ej]), 0.0 if fm is None else float(np.abs(fm - f).max())) for m, f in cands]
        assert min(max(e) for e in errs) <= 1e-4, (kind, g, errs)
