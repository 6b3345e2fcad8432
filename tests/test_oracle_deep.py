"""CPU: GCNs with five to seven graph-convolution layers.  The torch port (gnnx_oracle.explain_dense_torch) reproduces bit for bit every
mask the unmodified reference returned (tests/golden/deep_golden.npz, tools/gen_deep_golden.py), and the fp64 closed form
(oracle/gnnx_oracle.explain_closed_form, the specification of explain_var.cu) matches torch autograd's dL/dM and dL/dF
(tests/mask_grad_oracle.py) at 5 and 7 layers, node and graph mode, with and without --bn."""
import os

import numpy as np
import pytest

import gnnx_oracle as O
import mask_grad_oracle as MG

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "deep_golden.npz")


def golden_cases():
    """(name, mode) of every case of tests/golden/deep_golden.npz."""
    g = np.load(GOLDEN)
    return [(str(c), int(g["%s_mode" % c])) for c in g["cases"]]


def case_weights(g, case):
    p = case + "_w_"
    return {k[len(p):]: g[k] for k in g.files if k.startswith(p)}


def golden_items(g, case):
    """(key, A, X, gt, pred_label, idx, M0 seed) of every node / graph of a case."""
    k = lambda s_: g["%s_%s" % (case, s_)]
    if int(k("mode")) == 0:
        rg = np.load(os.path.join(os.path.dirname(GOLDEN), "rand_graph.npz"))
        N = int(rg["N"])
        rowptr, col = O.csr_from_edges(N, rg["edges"])
        pred_label = np.argmax(k("pred"), 1)
        for node in k("nodes"):
            idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(rowptr, col, rg["feat"], rg["label"], int(node), int(k("L")))
            assert np.array_equal(nbrs, g["%s_n%d_nbrs" % (case, node)])
            yield ("%s_n%d" % (case, node), O.dense_from_csr(srp, scol), sfeat.astype(np.float32), int(slabel[idx]), pred_label[nbrs], idx,
                   int(g["%s_n%d_seed" % (case, node)]))
    else:
        gg = np.load(os.path.join(os.path.dirname(GOLDEN), "graphs_golden.npz"))
        for gi in range(int(gg["num_graphs"])):
            yield ("%s_g%d" % (case, gi), np.asarray(gg["adj"][gi], np.float64), gg["feat"][gi].astype(np.float32), int(gg["label"][gi]),
                   None, 0, int(gg["g%d_seed" % gi]))


def test_golden_covers_the_issue_cases():
    g = np.load(GOLDEN)
    L = {str(c): int(g["%s_L" % c]) for c in g["cases"]}
    assert sorted(set(L.values())) == [5, 6, 7]
    assert os.path.getsize(GOLDEN) <= 2 * 1024 * 1024


@pytest.mark.parametrize("case,mode", golden_cases(), ids=lambda c: str(c))
def test_port_matches_reference_golden(case, mode):
    """The torch port reproduces every mask the unmodified reference returned bit for bit (graph 8 of graphs_bn_L7 included, whose
    trajectory amplifies rounding), and the model's preds to 1e-5."""
    g = np.load(GOLDEN)
    w = case_weights(g, case)
    hp = O.default_hparams(num_epochs=int(g[case + "_epochs"]), opt=str(g[case + "_opt"]))
    bn, att = bool(g[case + "_bn"]), bool(g[case + "_att"])
    for key, A, X, gt, pl, idx, seed in golden_items(g, case):
        got = O.explain_dense_torch(A, X, gt, pl, idx, w, O.draw_m0(A.shape[0], seed=seed), hp, graph_mode=mode == 1, bn=bn)
        ei, ej = np.nonzero(A)
        assert O.rel_l2(got[ei, ej], g[key + "_mask"]) == 0.0, key
    if mode == 0 and not att:
        rg = np.load(os.path.join(os.path.dirname(GOLDEN), "rand_graph.npz"))
        Af = O.dense_from_csr(*O.csr_from_edges(int(rg["N"]), rg["edges"]))
        pred = O.model_pred(Af, rg["feat"], w, bn=bn)
        assert np.abs(pred - g[case + "_pred"]).max() <= 1e-5 * max(1.0, np.abs(pred).max())


@pytest.mark.parametrize("L,bn,graph_mode", [(5, False, False), (5, True, False), (7, False, False), (7, True, False),
                                             (5, False, True), (5, True, True), (7, False, True), (7, True, True)])
def test_closed_form_matches_autograd(L, bn, graph_mode):
    rng = np.random.default_rng(100 * L + 10 * bn + graph_mode)
    n, d, hid, emb, C = 14, 6, 12, 10, 3
    A = np.triu((rng.random((n, n)) < 0.25).astype(np.float64), 1)
    for i in range(n - 1):   # connected: a path through every node
        A[i, i + 1] = 1
    A = A + A.T
    dims = [d] + [hid] * (L - 1) + [emb]
    w = {}
    for l in range(1, L + 1):
        w["W%d" % l] = rng.normal(size=(dims[l - 1], dims[l])) * 1.5 / np.sqrt(dims[l - 1])
        w["b%d" % l] = rng.normal(size=dims[l]) * 0.3
    w["Wp"] = rng.normal(size=(C, hid * (L - 1) + emb)) * 0.5
    w["bp"] = rng.normal(size=C) * 0.3
    X = rng.normal(size=(n, d))
    M = 1 + 0.4 * rng.normal(size=(n, n))
    F = 0.3 * rng.normal(size=d)
    pl = rng.integers(0, C, n)
    hp = O.default_hparams(num_epochs=1)
    state = dict(m=np.zeros((n, n)), v=np.zeros((n, n)), feat=(F, np.zeros(d), np.zeros(d)), step=0)
    _, st = O.explain_closed_form(A, X, 1, pl, 2, w, M, hp=hp, graph_mode=graph_mode, bn=bn, return_state=True, init_state=state)
    g = MG.mask_grads(A, X, 1, pl, 2, w, M, F, hp, graph_mode=graph_mode, bn=bn)
    assert np.abs(st["gM"] - g.gM).max() <= 1e-9 * max(1.0, np.abs(g.gM).max())
    assert np.abs(st["gF"] - g.gF).max() <= 1e-9 * max(1.0, np.abs(g.gF).max())
