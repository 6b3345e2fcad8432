"""CPU: attention models.  The closed-form backward of tests/att_oracle.py (the kernel's specification) matches torch autograd
(tests/mask_grad_oracle.py) on random attention models, node and graph mode, --bn, 2 / 3 / 4 layers, widths up to 128; the port
(gnnx_oracle.explain_dense_torch) reproduces the unmodified reference's masks and preds (tests/golden/att_golden.npz)."""
import os
import types

import numpy as np
import pytest

import att_oracle as AO
import gnnx_oracle as O
import mask_grad_oracle as MG

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "att_golden.npz")


def random_att_model(rng, d, hid, emb, C, L, scale=0.3):
    """Weights in the shapes of an attention GcnEncoderNode (xavier-like scale), biases N(0, scale)."""
    w = {}
    for l in range(L):
        win, wout = (d if l == 0 else hid), (emb if l == L - 1 else hid)
        w["W%d" % (l + 1)] = (rng.standard_normal((win, wout)) * np.sqrt(2.0 / (win + wout))).astype(np.float32)
        w["b%d" % (l + 1)] = (rng.standard_normal(wout) * scale).astype(np.float32)
        w["Wa%d" % (l + 1)] = (rng.standard_normal((win, win)) * np.sqrt(1.0 / win)).astype(np.float32)
    w["Wp"] = (rng.standard_normal((C, hid * (L - 1) + emb)) * 0.3).astype(np.float32)
    w["bp"] = (rng.standard_normal(C) * scale).astype(np.float32)
    return w


def random_graph(rng, n, p=0.25):
    A = (rng.random((n, n)) < p).astype(np.float32)
    A = np.triu(A, 1)
    A = A + A.T
    for i in range(n - 1):   # connected: a path through all nodes
        A[i, i + 1] = A[i + 1, i] = 1
    return A


CASES = [  # (d, hid, emb, C, L, bn, graph_mode)
    (7, 20, 20, 4, 3, False, False),
    (7, 20, 20, 4, 2, True, False),
    (10, 16, 12, 3, 4, False, False),
    (33, 128, 128, 4, 3, True, False),
    (7, 20, 20, 2, 3, False, True),
    (12, 24, 20, 3, 4, True, True),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "d%d_h%d_e%d_L%d%s%s" % (c[0], c[1], c[2], c[4], "_bn" if c[5] else "",
                                                                             "_graph" if c[6] else ""))
def test_closed_form_matches_autograd(case):
    d, hid, emb, C, L, bn, graph_mode = case
    rng = np.random.default_rng(hash(case) % 2**32)
    n = 11
    w = random_att_model(rng, d, hid, emb, C, L)
    A = random_graph(rng, n)
    X = rng.standard_normal((n, d)).astype(np.float32)
    M = (1 + 0.4 * rng.standard_normal((n, n))).astype(np.float32)
    F = (0.3 * rng.standard_normal(d)).astype(np.float32)
    pl = rng.integers(0, C, n)
    args = (A, X, 1, pl, 2, w, M, F)
    g = MG.mask_grads(*args, O.default_hparams(), graph_mode=graph_mode, bn=bn)
    cM, cF = AO.mask_grads_closed_form(*args, graph_mode=graph_mode, bn=bn)
    assert np.abs(g.gM - cM).max() <= 1e-9 * max(1.0, np.abs(g.gM).max())
    assert np.abs(g.gF - cF).max() <= 1e-9 * max(1.0, np.abs(g.gF).max())


def test_port_fp32_tracks_fp64():
    """The fp32 port and its fp64 twin agree on a short run (the fp64 port is what the kernel's single update is checked against)."""
    import torch
    rng = np.random.default_rng(5)
    w = random_att_model(rng, 7, 20, 20, 4, 3)
    A = random_graph(rng, 9)
    X = rng.standard_normal((9, 7)).astype(np.float32)
    M0 = (1 + 0.4 * rng.standard_normal((9, 9))).astype(np.float32)
    pl = rng.integers(0, 4, 9)
    hp = O.default_hparams(num_epochs=5)
    a32 = O.explain_dense_torch(A, X, 1, pl, 0, w, M0, hp)
    a64 = O.explain_dense_torch(A, X, 1, pl, 0, w, M0, hp, dtype=torch.float64)
    assert O.rel_l2(a32, a64) < 1e-4


def golden_cases():
    """(name, mode) of every case of tests/golden/att_golden.npz (tools/gen_att_golden.py)."""
    g = np.load(GOLDEN)
    return [(str(c), int(g[str(c) + "_mode"])) for c in g["cases"]]


def case_weights(g, case):
    return {k[len(case) + 3:]: g[k] for k in g.files if k.startswith(case + "_w_")}


def fixture_graph(name):
    """rowptr, col, dense adjacency and labels of a committed node fixture graph"""
    fg = np.load(os.path.join(os.path.dirname(GOLDEN), name + "_graph.npz"))
    N = int(fg["N"])
    rowptr, col = O.csr_from_edges(N, fg["edges"])
    return rowptr, col, O.dense_from_csr(rowptr, col, N), fg["label"].astype(np.int32)


@pytest.mark.parametrize("case,mode", golden_cases(), ids=lambda c: str(c))
def test_port_reproduces_reference_golden(case, mode):
    """The port reproduces every node mask the unmodified reference returned bit for bit, and lands within max(1e-6, 3 x the
    reference's own spread) of every graph mask (1e-6 on every trajectory that is not chaotic); the port's model forward reproduces the
    reference model's predictions (node mode: also with a self loop on every node, where s_ii enters)."""
    g = np.load(GOLDEN)
    k = lambda s_: g["%s_%s" % (case, s_)]
    w = case_weights(g, case)
    L, bn = int(k("L")), bool(k("bn"))
    hp = O.default_hparams(num_epochs=int(k("epochs")), opt=str(k("opt")))
    if mode == 0:
        rowptr, col, A_full, label = fixture_graph(str(k("graph")))
        feat = k("feat")
        pred = O.model_pred(A_full, feat, w, bn=bn)
        assert np.abs(pred - k("pred")).max() <= 1e-5 * max(1.0, np.abs(k("pred")).max())
        pred_loop = O.model_pred(A_full + np.eye(len(A_full), dtype=A_full.dtype), feat, w, bn=bn)
        assert np.abs(pred_loop - k("pred_loop")).max() <= 1e-5 * max(1.0, np.abs(k("pred_loop")).max())
        pred_label = np.argmax(k("pred"), 1)
        for node in [int(v) for v in k("nodes")]:
            idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(rowptr, col, feat, label, node, L)
            assert np.array_equal(nbrs, g["%s_n%d_nbrs" % (case, node)])
            A = O.dense_from_csr(srp, scol)
            M0 = O.draw_m0(len(nbrs), seed=int(g["%s_n%d_seed" % (case, node)]))
            got = O.explain_dense_torch(A, sfeat, slabel[idx], pred_label[nbrs], idx, w, M0, hp, bn=bn)
            ei, ej = np.nonzero(A)
            assert O.rel_l2(got[ei, ej], g["%s_n%d_mask" % (case, node)]) == 0.0, (case, node)
    else:
        gg = np.load(os.path.join(os.path.dirname(GOLDEN), "graphs_golden.npz"))
        n = int(gg["max_nodes"])
        for gi in range(int(gg["num_graphs"])):
            A = gg["adj"][gi].astype(np.float64)
            pred = O.model_pred(A, gg["feat"][gi], w, bn=bn, graph_mode=True)
            assert np.abs(pred - k("pred")[gi]).max() <= 1e-5 * max(1.0, np.abs(k("pred")[gi]).max())
            got = O.explain_dense_torch(A, gg["feat"][gi], int(gg["label"][gi]), None, 0, w, O.draw_m0(n, seed=int(gg["g%d_seed" % gi])),
                                        hp, graph_mode=True, bn=bn)
            ei, ej = np.nonzero(A)
            tol = max(1e-6, 3 * float(g["%s_g%d_spread" % (case, gi)]))
            assert O.rel_l2(got[ei, ej], g["%s_g%d_mask" % (case, gi)]) <= tol, (case, gi)
