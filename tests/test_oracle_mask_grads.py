"""CPU: tests/mask_grad_oracle.mask_grads against what the suite already pins, at spread-out points (M, F ~ N(0, 1.5^2)), so that
tests/test_gpu_mask_grads.py can compare the kernels' gradients with it:

  * the default model and its depth / --bn variants, node and graph mode: the gM / gF gnnx_oracle.explain_closed_form reports after one
    update from that state (init_state), to 1e-9; inputs wider than 128 (the wide path's d) the same way;
  * attention models: att_oracle.mask_grads_closed_form;
  * every other model (5 / 7 layers, widths to 256, MLP heads, unconstrained=True): one fp64 SGD step of the torch port
    (gnnx_oracle.explain_dense_torch) from a symmetric M0 lands on M0 - lr g, and dense_oracle.explain_closed_form's gradient for
    unconstrained=True."""
import numpy as np
import pytest
import torch

import att_oracle as AO
import dense_oracle as D
import gnnx_oracle as O
import mask_grad_oracle as MG
from test_oracle_att import random_att_model, random_graph
from test_oracle_hparams import PROBLEMS, _args

HP = O.default_hparams()


def _point(rng, n, d, sym=False):
    M = rng.normal(0, 1.5, (n, n))
    if sym:
        M = np.triu(M) + np.triu(M, 1).T
    return M, rng.normal(0, 1.5, d)


def _close(a, b, tol=1e-9):
    return np.abs(a - b).max() <= tol * np.abs(b).max()


@pytest.mark.parametrize("prob", list(PROBLEMS))
def test_default_models_equal_the_closed_form(prob):
    p = PROBLEMS[prob]()
    n, d = p["A"].shape[0], p["X"].shape[1]
    M, F = _point(np.random.default_rng(len(prob)), n, d)
    z = np.zeros((n, n))
    _, st = O.explain_closed_form(*_args(p), M, hp=O.default_hparams(num_epochs=1), graph_mode=p["graph_mode"], bn=p["bn"],
                                  return_state=True, init_state=dict(m=z, v=z, feat=np.stack([F, np.zeros(d), np.zeros(d)]), step=0))
    g = MG.mask_grads(*_args(p), M, F, HP, graph_mode=p["graph_mode"], bn=p["bn"])
    assert _close(g.gM, st["gM"]) and _close(g.gF, st["gF"]), prob
    assert g.kink > 0


def _random_problem(seed, n, d, hid, emb, C, L, head=None, bn=False):
    rng = np.random.default_rng(seed)
    dims = [d] + [hid] * (L - 1) + [emb]
    w = {}
    for l in range(1, L + 1):
        w["W%d" % l] = (rng.normal(size=(dims[l - 1], dims[l])) * np.sqrt(2.0 / (dims[l - 1] + dims[l]))).astype(np.float32)
        w["b%d" % l] = (rng.normal(size=dims[l]) * 0.3).astype(np.float32)
    width = hid * (L - 1) + emb
    if head:
        w["head"] = []
        for h in head:
            w["head"].append(((rng.normal(size=(h, width)) * np.sqrt(2.0 / width)).astype(np.float32), (rng.normal(size=h) * 0.3).astype(np.float32)))
            width = h
    w["Wp"] = (rng.normal(size=(C, width)) * 0.5).astype(np.float32)
    w["bp"] = (rng.normal(size=C) * 0.3).astype(np.float32)
    A = random_graph(rng, n, 0.2)
    X = rng.normal(size=(n, d)).astype(np.float32)
    return rng, w, A, X, rng.integers(0, C, n)


@pytest.mark.parametrize("graph_mode", [False, True], ids=["node", "graph"])
@pytest.mark.parametrize("d", [129, 200])
def test_wide_inputs_equal_the_closed_form(d, graph_mode):
    rng, w, A, X, pl = _random_problem(d, 13, d, 20, 20, 3, 3)
    M, F = _point(rng, 13, d)
    z = np.zeros((13, 13))
    _, st = O.explain_closed_form(A, X, 1, pl, 2, w, M, hp=O.default_hparams(num_epochs=1), graph_mode=graph_mode, return_state=True,
                                  init_state=dict(m=z, v=z, feat=np.stack([F, np.zeros(d), np.zeros(d)]), step=0))
    g = MG.mask_grads(A, X, 1, pl, 2, w, M, F, HP, graph_mode=graph_mode)
    assert _close(g.gM, st["gM"]) and _close(g.gF, st["gF"])


@pytest.mark.parametrize("graph_mode", [False, True], ids=["node", "graph"])
@pytest.mark.parametrize("L,bn", [(3, True), (2, False), (4, False)])
def test_attention_equals_its_closed_form(L, bn, graph_mode):
    rng = np.random.default_rng(10 * L + bn)
    w = random_att_model(rng, 7, 20, 20, 4, L)
    A = random_graph(rng, 12)
    X = rng.standard_normal((12, 7)).astype(np.float32)
    M, F = _point(rng, 12, 7)
    pl = rng.integers(0, 4, 12)
    gM, gF = AO.mask_grads_closed_form(A, X, 1, pl, 2, w, M, F, graph_mode=graph_mode, bn=bn)
    g = MG.mask_grads(A, X, 1, pl, 2, w, M, F, HP, graph_mode=graph_mode, bn=bn)
    assert _close(g.gM, gM) and _close(g.gF, gF)


def _sgd_step_grads(port, A, M0, lr, **kw):
    """g on the edges and gF from one fp64 SGD step of a port (two epochs: the returned mask is sigmoid(M0 - lr g) on the edges, the
    feature mask sigmoid(-lr gF))."""
    out, fm = port(**kw, M0=M0, hp=O.default_hparams(num_epochs=2, opt="sgd", lr=lr), dtype=torch.float64, return_feat=True)
    ei, ej = np.nonzero(A)
    logit = lambda p: np.log(p) - np.log1p(-p)
    return (M0[ei, ej] - logit(out[ei, ej])) / lr, -logit(fm) / lr


OTHER = {  # (n, d, hid, emb, C, L, head, bn)
    "L5": (14, 6, 20, 20, 3, 5, None, False), "L7_bn": (14, 6, 20, 20, 3, 7, None, True), "w200_256": (12, 9, 200, 256, 4, 3, None, False),
    "w128_bn": (12, 9, 128, 128, 4, 3, None, True), "head50": (12, 9, 20, 20, 4, 3, [50], False),
    "head256_7_bn": (12, 9, 20, 20, 4, 3, [256, 7], True),
}


@pytest.mark.parametrize("graph_mode", [False, True], ids=["node", "graph"])
@pytest.mark.parametrize("case", list(OTHER))
def test_other_models_take_the_ports_sgd_step(case, graph_mode):
    n, d, hid, emb, C, L, head, bn = OTHER[case]
    rng, w, A, X, pl = _random_problem(100 + list(OTHER).index(case), n, d, hid, emb, C, L, head, bn)
    M0, _ = _point(rng, n, d, sym=True)
    g = MG.mask_grads(A, X, 1, None if graph_mode else pl, 2, w, M0, np.zeros(d), HP, graph_mode=graph_mode, bn=bn)
    ei, ej = np.nonzero(A)
    lr = 1e-3 / np.abs(g.gM).max()
    gM, gF = _sgd_step_grads(O.explain_dense_torch, A, M0, lr, sub_adj=A, sub_feat=X, gt_label=1, pred_label=None if graph_mode else pl,
                             node_idx_new=2, weights=w, graph_mode=graph_mode, bn=bn)
    assert np.abs(gM - g.gM[ei, ej]).max() <= 1e-7 * np.abs(g.gM).max(), case
    assert np.abs(gF - g.gF).max() <= 1e-7 * np.abs(g.gF).max(), case


@pytest.mark.parametrize("graph_mode", [False, True], ids=["node", "graph"])
@pytest.mark.parametrize("model", ["default", "bn", "head"])
def test_unconstrained_mask(model, graph_mode):
    """unconstrained=True: every entry of the dense mask against dense_oracle's closed form (plain models) or, with a head, the edges of
    the unconstrained port after one SGD step."""
    rng, w, A, X, pl = _random_problem(7 + len(model), 15, 8, 20, 20, 3, 3, [50] if model == "head" else None)
    bn = model == "bn"
    M0, _ = _point(rng, 15, 8, sym=True)
    kw = dict(graph_mode=graph_mode, bn=bn, unconstrained=True)
    g = MG.mask_grads(A, X, 1, None if graph_mode else pl, 2, w, M0, np.zeros(8), HP, **kw)
    assert np.abs(g.gF - 0.25 * HP.feat_size / 8).max() <= 1e-15          # the forward never sees F
    if model == "head":
        lr = 1e-3 / np.abs(g.gM).max()
        ei, ej = np.nonzero(A)
        gM, _ = _sgd_step_grads(O.explain_dense_torch, A, M0, lr, sub_adj=A, sub_feat=X, gt_label=1,
                                pred_label=None if graph_mode else pl, node_idx_new=2, weights=w, graph_mode=graph_mode, bn=bn,
                                unconstrained=True)
        assert np.abs(gM - g.gM[ei, ej]).max() <= 1e-7 * np.abs(g.gM).max()
    else:
        _, st = D.explain_closed_form(A, X, 1, pl, 2, w, M0, hp=O.default_hparams(num_epochs=1), graph_mode=graph_mode, bn=bn,
                                      return_state=True)
        assert _close(g.gM, st["gM"])


def test_float32_is_close_and_margins_are_reported():
    """The float32 evaluation (the kernels' rounding yardstick) is a few 1e-7 off the fp64 one; the ReLU margin is reported."""
    p = PROBLEMS["graph_L3"]()
    n, d = p["A"].shape[0], p["X"].shape[1]
    M, F = _point(np.random.default_rng(3), n, d)
    g64 = MG.mask_grads(*_args(p), M, F, HP, graph_mode=True)
    g32 = MG.mask_grads(*_args(p), M, F, HP, graph_mode=True, dtype=torch.float32)
    assert 0 < np.abs(g32.gM - g64.gM).max() <= 1e-5 * np.abs(g64.gM).max()
    assert 0 < g64.kink < 1 and isinstance(g64.ties, list)
