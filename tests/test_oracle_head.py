"""CPU: the MLP prediction head (pred_hidden_dims, models.py:193-207) -- the torch port (gnnx_oracle.explain_dense_torch) against
autograd and the reference, and gnnx.models' GcnEncoderNode / GcnEncoderGraph(pred_hidden_dims=[..]) against the reference's layout and
the port."""
import os
import types

import numpy as np
import pytest
import torch

import gnnx_oracle as O
import util


def _args(bn):
    return types.SimpleNamespace(num_gc_layers=3, bias=True, gpu=False, method="base", bn=bn)


def _weights(model):
    from gnnx.explain import model_weights
    return model_weights(model)


@pytest.mark.parametrize("cls,graph", [("GcnEncoderNode", False), ("GcnEncoderGraph", True)])
def test_models_head_layout_and_forward(cls, graph):
    """state_dict keys pred_model.0 / .2 / .. (ReLUs at the odd indices), every Linear with a bias, torch's default init drawn in
    construction order; the forward equals the port's; model_weights returns the hidden Linears as "head" and the last as Wp / bp."""
    import gnnx.models as M
    torch.manual_seed(7)
    model = getattr(M, cls)(10, 20, 16, 3, 4, pred_hidden_dims=[50, 7], bn=True, args=_args(True))
    keys = [k for k in model.state_dict() if k.startswith("pred_model")]
    assert keys == ["pred_model.0.weight", "pred_model.0.bias", "pred_model.2.weight", "pred_model.2.bias", "pred_model.4.weight",
                    "pred_model.4.bias"]
    assert isinstance(model.pred_model[1], torch.nn.ReLU) and isinstance(model.pred_model[3], torch.nn.ReLU)
    assert tuple(model.pred_model[0].weight.shape) == (50, 20 * 3 + 16) and tuple(model.pred_model[4].weight.shape) == (3, 7)
    ref = getattr(M, cls)(10, 20, 16, 3, 4, bn=True, args=_args(True))
    w, L = _weights(model)
    assert L == 4 and [h[0].shape for h in w["head"]] == [(50, 76), (7, 50)] and w["Wp"].shape == (3, 7)
    assert np.array_equal(w["head"][0][0], model.pred_model[0].weight.detach().numpy())
    assert ref.pred_model.weight.shape == (3, 76)
    rng = np.random.default_rng(1)
    n = 12
    A = (rng.random((n, n)) < 0.3).astype(np.float32)
    A = np.maximum(A, A.T)
    X = rng.normal(size=(n, 10)).astype(np.float32)
    with torch.no_grad():
        got = model(torch.tensor(X[None]), torch.tensor(A[None]))[0][0].numpy()
    want = O.model_pred(A, X, w, bn=True, graph_mode=graph)
    assert np.abs(got - want).max() <= 1e-6


def test_port_matches_autograd_of_the_head():
    """One epoch of the port in fp64: its mask gradient equals autograd through an independently written head (nn.Sequential)."""
    rng = np.random.default_rng(2)
    n, d = 9, 6
    A = (rng.random((n, n)) < 0.4).astype(np.float64)
    A = np.triu(A, 1); A = A + A.T
    X = rng.normal(size=(n, d))
    w = {"W1": rng.normal(size=(d, 8)), "b1": rng.normal(size=8) * 0.3, "W2": rng.normal(size=(8, 5)) * 0.5, "b2": rng.normal(size=5) * 0.3,
         "head": [(rng.normal(size=(11, 13)), rng.normal(size=11) * 0.3)], "Wp": rng.normal(size=(3, 11)), "bp": rng.normal(size=3)}
    M0 = rng.normal(1.0, 0.3, size=(n, n))
    hp = O.default_hparams(num_epochs=2, opt="sgd")
    out = O.explain_dense_torch(A, X, 1, np.zeros(n), 2, w, M0, hp, dtype=torch.float64)
    seq = torch.nn.Sequential(torch.nn.Linear(13, 11), torch.nn.ReLU(), torch.nn.Linear(11, 3)).double()
    with torch.no_grad():
        seq[0].weight.copy_(torch.tensor(w["head"][0][0])); seq[0].bias.copy_(torch.tensor(w["head"][0][1]))
        seq[2].weight.copy_(torch.tensor(w["Wp"])); seq[2].bias.copy_(torch.tensor(w["bp"]))
    W = O.weights_to_torch(w, dtype=torch.float64)
    M = torch.tensor(M0, requires_grad=True)
    S = torch.sigmoid(M); S = (S + S.t()) / 2
    At = torch.tensor(A)[None]
    masked = At * S * (1 - torch.eye(n, dtype=torch.float64))
    Wn = dict(W, head=[], pred_w=torch.eye(13, dtype=torch.float64), pred_b=torch.zeros(13, dtype=torch.float64))
    e = O._gcn_forward_torch(torch.tensor(X)[None] * 0.5, masked, Wn, False)[0, 2]
    res = torch.softmax(seq(e), 0)
    m = torch.sigmoid(M)
    ent = -m * torch.log(m) - (1 - m) * torch.log(1 - m)
    pl = torch.zeros(n, dtype=torch.float64)
    Dg = torch.diag(torch.sum(masked[0], 0))
    loss = -torch.log(res[1]) + hp.size * m.sum() + hp.ent * ent.mean() + hp.feat_size * 0.5 + hp.lap * (pl @ (Dg - masked[-1]) @ pl) / At.numel()
    loss.backward()
    M1 = M0 - hp.lr * M.grad.numpy()   # SGD's first step (momentum buffer = the gradient)
    S1 = 1 / (1 + np.exp(-M1)); S1 = (S1 + S1.T) / 2
    assert np.abs(out - A * S1 * (1 - np.eye(n))).max() <= 1e-12


# ---------------------------------------------------------------------------------------------- against the reference (head_golden.npz)
GOLDEN = np.load(os.path.join(util.GOLDEN, "head_golden.npz"))


def golden_cases(mode):
    return [str(c) for c in GOLDEN["cases"] if int(GOLDEN[c + "_mode"]) == mode]


def case_weights(c):
    """The case's weights as float32, the head as "head" = [(W, b), ..] (Engine.set_model's form)."""
    p = c + "_w_"
    w = {k[len(p):]: GOLDEN[k].astype(np.float32) for k in GOLDEN.files if k.startswith(p)}
    w["head"] = O.head_layers(w)
    for k in [k for k in w if k.startswith(("Wh", "bh"))]:
        del w[k]
    return w


def case_feat(c):
    """(adj (1, N, N), feat (N, d), label) of a node-mode case: the rand graph, with the case's own features where it has them."""
    fx = util.load_fixture("rand")
    feat = GOLDEN[c + "_feat"].astype(np.float32) if (c + "_feat") in GOLDEN.files else fx.feat
    return fx, feat


def _hp(c):
    return O.default_hparams(num_epochs=int(GOLDEN[c + "_epochs"]), opt=str(GOLDEN[c + "_opt"]))


@pytest.mark.parametrize("case", golden_cases(0))
def test_port_matches_reference_nodes(case):
    fx, feat = case_feat(case)
    w, L, bn, unc = case_weights(case), int(GOLDEN[case + "_L"]), bool(GOLDEN[case + "_bn"]), bool(GOLDEN[case + "_unc"])
    pred_label = np.argmax(GOLDEN[case + "_pred"], axis=1)
    for node in GOLDEN[case + "_nodes"]:
        key = "%s_n%d" % (case, node)
        idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(fx.rowptr, fx.col, feat, fx.label, int(node), L)
        assert np.array_equal(nbrs, GOLDEN[key + "_nbrs"])
        A = O.dense_from_csr(srp, scol)
        ei, ej = np.nonzero(A)
        M0 = O.draw_m0(len(nbrs), seed=int(GOLDEN[key + "_seed"]))
        got = O.explain_dense_torch(A, X, int(lab[idx]), pred_label[nbrs], idx, w, M0, _hp(case), bn=bn, unconstrained=unc)[ei, ej]
        assert O.rel_l2(got, GOLDEN[key + "_mask"]) == 0.0, key


@pytest.mark.parametrize("case", golden_cases(1))
def test_port_matches_reference_graphs(case):
    gg = np.load(os.path.join(util.GOLDEN, "graphs_golden.npz"))
    w, bn, unc = case_weights(case), bool(GOLDEN[case + "_bn"]), bool(GOLDEN[case + "_unc"])
    n = int(gg["max_nodes"])
    for g in range(int(gg["num_graphs"])):
        key = "%s_g%d" % (case, g)
        A = gg["adj"][g].astype(np.float64)
        ei, ej = np.nonzero(A)
        M0 = O.draw_m0(n, seed=int(gg["g%d_seed" % g]))
        got = O.explain_dense_torch(A, gg["feat"][g].astype(np.float32), int(gg["label"][g]), None, 0, w, M0, _hp(case), graph_mode=True,
                                    bn=bn, unconstrained=unc)[ei, ej]
        assert O.rel_l2(got, GOLDEN[key + "_mask"]) == 0.0, key


def test_models_init_matches_reference():
    """gnnx.models.GcnEncoderNode(pred_hidden_dims=[50, 7]) under the reference's seed: the reference's keys and parameters, bit for bit."""
    import gnnx.models as M
    torch.manual_seed(int(GOLDEN["init_seed"]))
    model = M.GcnEncoderNode(10, 20, 20, 3, 3, pred_hidden_dims=[50, 7], bn=True, args=_args(True))
    sd = model.state_dict()
    want = {k[len("init_"):] for k in GOLDEN.files if k.startswith("init_") and k != "init_seed"}
    assert set(sd) == want
    for k in want:
        assert np.array_equal(sd[k].numpy(), GOLDEN["init_" + k]), k


@pytest.mark.parametrize("case", golden_cases(0) + golden_cases(1))
def test_models_load_reference_weights_and_forward(case):
    """The case's reference weights load into gnnx.models under the reference's state_dict keys; model_weights reads them back and the
    forward reproduces the reference's pred."""
    import gnnx.models as M
    w, L, bn, att = case_weights(case), int(GOLDEN[case + "_L"]), bool(GOLDEN[case + "_bn"]), bool(GOLDEN[case + "_att"])
    graph = int(GOLDEN[case + "_mode"]) == 1
    widths = [int(x) for x in GOLDEN[case + "_head"]]
    d = w["W1"].shape[0]
    args = types.SimpleNamespace(num_gc_layers=L, bias=True, gpu=False, method="att" if att else "base", bn=bn)
    model = (M.GcnEncoderGraph if graph else M.GcnEncoderNode)(d, int(GOLDEN[case + "_hid"]), int(GOLDEN[case + "_emb"]), w["Wp"].shape[0], L,
                                                              pred_hidden_dims=widths, bn=bn, args=args)
    keys = ["conv_first"] + ["conv_block.%d" % i for i in range(L - 2)] + ["conv_last"]
    sd = {}
    for l, k in enumerate(keys, 1):
        sd[k + ".weight"], sd[k + ".bias"] = w["W%d" % l], w["b%d" % l]
        if att:
            sd[k + ".att_weight"] = w["Wa%d" % l]
    for j, (W, b) in enumerate(w["head"] + [(w["Wp"], w["bp"])]):
        sd["pred_model.%d.weight" % (2 * j)], sd["pred_model.%d.bias" % (2 * j)] = W, b
    model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    got_w, got_L = _weights(model)
    assert got_L == L and len(got_w["head"]) == len(widths)
    for (a, b), (c, e) in zip(got_w["head"] + [(got_w["Wp"], got_w["bp"])], w["head"] + [(w["Wp"], w["bp"])]):
        assert np.array_equal(a, c) and np.array_equal(b, e)
    with torch.no_grad():
        if graph:
            gg = np.load(os.path.join(util.GOLDEN, "graphs_golden.npz"))
            got = np.stack([model(torch.tensor(gg["feat"][g:g + 1].astype(np.float32)), torch.tensor(gg["adj"][g:g + 1], dtype=torch.float))[0][0]
                            .numpy() for g in range(int(gg["num_graphs"]))])
        else:
            fx, feat = case_feat(case)
            A = O.dense_from_csr(fx.rowptr, fx.col).astype(np.float32)
            got = model(torch.tensor(feat[None]), torch.tensor(A[None]))[0][0].numpy()
    assert np.abs(got - GOLDEN[case + "_pred"]).max() <= 1e-6
