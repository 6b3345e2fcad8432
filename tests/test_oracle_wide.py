"""CPU: the layer-1 contraction order of explain_var.cu's wide path (tests/wide_oracle.py, numpy fp64) against torch autograd on the
reference's order, (A_m (X (.) sigmoid(F))) W1, in node and graph mode, with and without --bn, 2 and 4 layers, d = 300; and the torch
port (gnnx_oracle.explain_dense_torch) against the masks the unmodified reference returned (tests/golden/wide_golden.npz,
tools/gen_wide_golden.py)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import gnnx_oracle as O
import wide_oracle as WO


def _setup(seed, L, d=300, n=24, hid=40, C=3):
    rng = np.random.default_rng(seed)
    A = np.triu((rng.random((n, n)) < 0.2).astype(np.float64), 1)
    A = A + A.T
    S = 1 / (1 + np.exp(-rng.normal(1.0, 0.3, size=(n, n))))
    a = A * (S + S.T) / 2
    X = rng.normal(size=(n, d))
    F = rng.normal(size=d) * 0.5
    dims = [d] + [hid] * L
    w = {"W%d" % l: rng.normal(size=(dims[l - 1], dims[l])) / np.sqrt(dims[l - 1]) for l in range(1, L + 1)}
    w.update({"b%d" % l: rng.normal(size=hid) * 0.3 for l in range(1, L + 1)})
    w["Wp"] = rng.normal(size=(C, hid * L)) * 0.5
    w["bp"] = rng.normal(size=C) * 0.5
    return a, X, F, w


@pytest.mark.parametrize("graph_mode,bn,L", [(False, True, 2), (False, False, 4), (True, True, 4), (True, False, 2)])
def test_wide_contraction_order_matches_autograd(graph_mode, bn, L):
    a, X, F, w = _setup(10 * L + bn + 2 * graph_mode, L)
    t = lambda v, g=False: torch.tensor(v, dtype=torch.float64, requires_grad=g)
    a1, a_rest, sF = t(a, True), t(a), t(1 / (1 + np.exp(-F)), True)
    y = a1 @ (t(X) * sF) @ t(w["W1"]) + t(w["b1"])          # the reference's order (explain.py:707, models.py:70-76)
    y.retain_grad()
    outs, h = [], None
    for l in range(1, L + 1):
        if l > 1:
            y = a_rest @ h @ t(w["W%d" % l]) + t(w["b%d" % l])
        z = Fn.normalize(y, p=2, dim=1)
        if l < L:
            z = torch.relu(z)
            if bn:
                z = Fn.batch_norm(z[None], None, None, None, None, True, 0.1, 1e-5)[0]
        outs.append(z)
        h = z
        if l == 1:
            y1 = y
    emb = torch.cat([o.max(0)[0] for o in outs]) if graph_mode else torch.cat(outs, 1)[0]
    loss = -torch.log_softmax(emb @ t(w["Wp"]).T + t(w["bp"]), 0)[1]
    loss.backward()
    assert np.abs(WO.layer1_wide_forward(a, X, F, w["W1"], w["b1"]) - y1.detach().numpy()).max() <= 1e-9
    dsF, da = WO.layer1_wide_grads(a, X, F, w["W1"], y1.grad.numpy(), c_feat=0.0)
    assert np.abs(dsF - sF.grad.numpy()).max() <= 1e-9 * max(1.0, np.abs(sF.grad.numpy()).max())
    assert np.abs(da - a1.grad.numpy()).max() <= 1e-9 * max(1.0, np.abs(a1.grad.numpy()).max())


# ------------------------------------------------------------------------------------------------------------- the unmodified reference
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wide_golden.npz")


def golden_cases():
    g = np.load(GOLDEN)
    return [(str(c), int(g["%s_mode" % c])) for c in g["cases"]]


def case_weights(g, case):
    p = case + "_w_"
    return {k[len(p):]: g[k] for k in g.files if k.startswith(p)}


def golden_items(g, case):
    """(key, A, X, gt, pred_label, idx, M0 seed) of every node / graph of a case of tests/golden/wide_golden.npz."""
    k = lambda s_: g["%s_%s" % (case, s_)]
    if int(k("mode")) == 0:
        rg = np.load(os.path.join(os.path.dirname(GOLDEN), "rand_graph.npz"))
        N = int(rg["N"])
        rowptr, col = O.csr_from_edges(N, rg["edges"])
        pred_label = np.argmax(k("pred"), 1)
        for node in k("nodes"):
            idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(rowptr, col, k("feat"), rg["label"], int(node), int(k("L")))
            assert np.array_equal(nbrs, g["%s_n%d_nbrs" % (case, node)])
            yield ("%s_n%d" % (case, node), O.dense_from_csr(srp, scol), sfeat, int(slabel[idx]), pred_label[nbrs], idx,
                   int(g["%s_n%d_seed" % (case, node)]))
    else:
        gg = np.load(os.path.join(os.path.dirname(GOLDEN), "graphs_golden.npz"))
        for gi in range(int(gg["num_graphs"])):
            yield ("%s_g%d" % (case, gi), np.asarray(gg["adj"][gi], np.float64), k("feat")[gi], int(gg["label"][gi]), None, 0,
                   int(gg["g%d_seed" % gi]))


@pytest.mark.parametrize("case,mode", golden_cases(), ids=lambda c: str(c))
def test_port_matches_reference_golden(case, mode):
    """The torch port reproduces every mask the unmodified reference returned on d = 300 (node mode) and d = 190 (graph mode) bit for
    bit."""
    g = np.load(GOLDEN)
    w = case_weights(g, case)
    hp = O.default_hparams(num_epochs=int(g[case + "_epochs"]), opt=str(g[case + "_opt"]))
    bn = bool(g[case + "_bn"])
    for key, A, X, gt, pl, idx, seed in golden_items(g, case):
        port = O.explain_dense_torch(A, X, gt, pl, idx, w, O.draw_m0(A.shape[0], seed=seed), hp, graph_mode=mode == 1, bn=bn)
        ei, ej = np.nonzero(A)
        assert O.rel_l2(port[ei, ej], g[key + "_mask"]) == 0.0, key
