"""CPU: GCNs with hidden / output widths of 129 .. 256.  The torch port (gnnx_oracle.explain_dense_torch) reproduces bit for bit every
mask the unmodified reference returned (tests/golden/wide_layers_golden.npz, tools/gen_wide_layers_golden.py), and the fp64 closed form
(gnnx_oracle.explain_closed_form, the specification of explain_var.cu) matches torch autograd's dL/dM and dL/dF
(tests/mask_grad_oracle.py) at width 256, 2 and 5 layers, node and graph mode, with and without --bn."""
import os

import numpy as np
import pytest

import gnnx_oracle as O
import mask_grad_oracle as MG
from test_oracle_deep import golden_items

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wide_layers_golden.npz")


def golden_cases():
    """(name, mode) of every case of tests/golden/wide_layers_golden.npz."""
    g = np.load(GOLDEN)
    return [(str(c), int(g["%s_mode" % c])) for c in g["cases"]]


def case_weights(g, case):
    """The case's model as float32 (the fixture stores each model once, as float16: its parameters are float16 values)."""
    p = str(g[case + "_wfrom"]) + "_w_"
    return {k[len(p):]: g[k].astype(np.float32) for k in g.files if k.startswith(p)}


def test_golden_covers_the_issue_cases():
    g = np.load(GOLDEN)
    widths = {str(c): (int(g["%s_hid" % c]), int(g["%s_emb" % c])) for c in g["cases"]}
    assert max(max(w) for w in widths.values()) == 256 and all(max(w) > 128 for w in widths.values())
    assert {int(g["%s_L" % c]) for c in g["cases"]} == {2, 3, 4, 5}
    assert os.path.getsize(GOLDEN) <= 1200 * 1024


@pytest.mark.parametrize("case,mode", golden_cases(), ids=lambda c: str(c))
def test_port_matches_reference_golden(case, mode):
    """The torch port reproduces every mask the unmodified reference returned bit for bit, and the model's preds to 1e-5."""
    g = np.load(GOLDEN)
    w = case_weights(g, case)
    hp = O.default_hparams(num_epochs=int(g[case + "_epochs"]), opt=str(g[case + "_opt"]))
    bn = bool(g[case + "_bn"])
    for key, A, X, gt, pl, idx, seed in golden_items(g, case):
        got = O.explain_dense_torch(A, X, gt, pl, idx, w, O.draw_m0(A.shape[0], seed=seed), hp, graph_mode=mode == 1, bn=bn)
        ei, ej = np.nonzero(A)
        assert O.rel_l2(got[ei, ej], g[key + "_mask"]) == 0.0, key
    if mode == 0:
        rg = np.load(os.path.join(os.path.dirname(GOLDEN), "rand_graph.npz"))
        Af = O.dense_from_csr(*O.csr_from_edges(int(rg["N"]), rg["edges"]))
        pred = O.model_pred(Af, rg["feat"], w, bn=bn)
        assert np.abs(pred - g[case + "_pred"]).max() <= 1e-5 * max(1.0, np.abs(pred).max())


@pytest.mark.parametrize("L,bn,graph_mode", [(2, False, False), (2, True, False), (5, False, False), (5, True, False),
                                             (2, False, True), (2, True, True), (5, False, True), (5, True, True)])
def test_closed_form_matches_autograd_at_width_256(L, bn, graph_mode):
    rng = np.random.default_rng(300 + 100 * L + 10 * bn + graph_mode)
    n, d, hid, emb, C = 14, 6, 256, 200, 3
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
