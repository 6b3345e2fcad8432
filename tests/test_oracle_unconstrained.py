"""explain(..., unconstrained=True) on the CPU: the line-by-line port against the UNMODIFIED reference's own results
(tests/golden/unconstrained_golden.npz, tools/gen_unconstrained_golden.py), and the fp64 closed form -- the dense kernel's
specification -- against torch autograd and the port."""
import os

import numpy as np
import pytest
import torch

import dense_oracle as D
import gnnx_oracle as O
import mask_grad_oracle as MG
import util

U = np.load(os.path.join(util.GOLDEN, "unconstrained_golden.npz"))
GG = np.load(os.path.join(util.GOLDEN, "graphs_golden.npz"))


def node_case(fx, node, n_hops=3):
    """(A, X, gt, y, idx, M0, (ei, ej)) of a node of a fixture, M0 = the reference's full (n, n) draw from the node's seed."""
    idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(fx.rowptr, fx.col, fx.feat, fx.label, node, n_hops)
    A = O.dense_from_csr(srp, scol)
    return A, sfeat, int(slabel[idx]), fx.pred_label[nbrs], idx, O.draw_m0(len(nbrs), seed=int(fx.gold["n%d_seed" % node])), np.nonzero(A)


def graph_case(g):
    A = GG["adj"][g].astype(np.float64)
    return A, GG["feat"][g], int(GG["label"][g]), None, 0, O.draw_m0(int(GG["max_nodes"]), seed=int(GG["g%d_seed" % g])), np.nonzero(A)


def graph_weights():
    return {k: GG[k] for k in util.WKEYS}


def var_weights(tag, where):
    pre = "var_%s_%s_" % (tag, where)
    return {k[len(pre):]: U[k] for k in U.files if k.startswith(pre) and k[len(pre):][0] in "Wb"}


@pytest.mark.parametrize("which,nodes,epochs", [("rand", None, (10, 30, 100)), ("syn4", None, (10, 30, 100)),
                                                ("syn1", [300, 313, 343, 33], (10,))])
def test_port_reproduces_reference_nodes(which, nodes, epochs):
    fx = util.load_fixture(which)
    for node in nodes or [int(v) for v in U[which + "_nodes"]]:
        A, X, gt, y, idx, M0, (ei, ej) = node_case(fx, node)
        for E in epochs:
            out = O.explain_dense_torch(A, X, gt, y, idx, fx.weights, M0, hp=O.default_hparams(num_epochs=E), unconstrained=True)
            assert O.rel_l2(out[ei, ej], U["%s_n%d_e%d_mask" % (which, node, E)]) == 0.0, (which, node, E)


@pytest.mark.parametrize("epochs", [10, 30])
def test_port_reproduces_reference_graphs(epochs):
    W = graph_weights()
    for g in range(int(GG["num_graphs"])):
        A, X, gt, _, _, M0, (ei, ej) = graph_case(g)
        out = O.explain_dense_torch(A, X, gt, None, 0, W, M0, hp=O.default_hparams(num_epochs=epochs), graph_mode=True, unconstrained=True)
        assert O.rel_l2(out[ei, ej], U["graphs_g%d_e%d_mask" % (g, epochs)]) == 0.0, (g, epochs)


@pytest.mark.parametrize("tag", ["bn", "L4", "sgd"])
def test_port_reproduces_reference_variants(tag):
    L, bn, E = int(U["var_%s_L" % tag]), bool(U["var_%s_bn" % tag]), int(U["var_epochs"])
    over = dict(opt="sgd") if tag == "sgd" else {}
    fx = util.load_fixture("rand")
    Wn = fx.weights if tag == "sgd" else var_weights(tag, "rand")
    for node in [0, 33, 149]:
        idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(fx.rowptr, fx.col, fx.feat, fx.label, node, L)
        assert np.array_equal(nbrs, U["var_%s_rand_n%d_nbrs" % (tag, node)])
        A = O.dense_from_csr(srp, scol); ei, ej = np.nonzero(A)
        pred_label = fx.pred_label if tag == "sgd" else variant_pred_label(fx, Wn, L, bn)
        M0 = O.draw_m0(len(nbrs), seed=int(fx.gold["n%d_seed" % node]))
        out = O.explain_dense_torch(A, X, int(lab[idx]), pred_label[nbrs], idx, Wn, M0, hp=O.default_hparams(num_epochs=E, **over), bn=bn,
                                    unconstrained=True)
        assert O.rel_l2(out[ei, ej], U["var_%s_rand_n%d_mask" % (tag, node)]) == 0.0, (tag, node)
    Wg = graph_weights() if tag == "sgd" else var_weights(tag, "graphs")
    for g in (0, 5, 11):
        A, X, gt, _, _, M0, (ei, ej) = graph_case(g)
        out = O.explain_dense_torch(A, X, gt, None, 0, Wg, M0, hp=O.default_hparams(num_epochs=E, **over), graph_mode=True, bn=bn,
                                    unconstrained=True)
        assert O.rel_l2(out[ei, ej], U["var_%s_graphs_g%d_mask" % (tag, g)]) == 0.0, (tag, g)


def variant_pred_label(fx, W, L, bn):
    """argmax of the random variant model's logits on the whole rand graph (what the fixture's Explainer was given as pred)."""
    A = O.dense_from_csr(fx.rowptr, fx.col)
    with torch.no_grad():
        logits = O._gcn_forward_torch(torch.tensor(fx.feat[None], dtype=torch.float), torch.tensor(A[None], dtype=torch.float),
                                      O.weights_to_torch(W, requires_grad=False), False, bn)
    return np.argmax(logits[0].numpy(), axis=1)


@pytest.mark.parametrize("which", ["syn1", "rand"])
def test_port_prints_reference_rows(which):
    """print_training=True: loss, mask density and softmax row of every epoch (what the reference printed, parsed)."""
    fx = util.load_fixture(which)
    E = int(U["trace_epochs"])
    for node in [int(v) for v in U["trace_%s_nodes" % which]]:
        A, X, gt, y, idx, M0, _ = node_case(fx, node)
        tr = []
        O.explain_dense_torch(A, X, gt, y, idx, fx.weights, M0, hp=O.default_hparams(num_epochs=E), trace=tr, unconstrained=True)
        ref = U["trace_%s_n%d" % (which, node)]
        got = np.array([[t["loss"], t["density"]] + list(t["pred"]) for t in tr])
        # the reference prints 8 decimals of every value: the port must agree to that print precision
        assert np.abs(got - ref).max() <= 5e-8 + 1e-7 * np.abs(ref).max(), (which, node, np.abs(got - ref).max())


@pytest.mark.parametrize("case", ["node", "node_bn", "node_L4", "graph", "graph_bn", "graph_L4"])
def test_closed_form_gradient_matches_autograd(case):
    """One step of the fp64 closed form: its dL/dM (all n^2 entries) and dL/dF equal torch autograd's to 1e-9."""
    graph_mode = case.startswith("graph")
    tag = case.split("_")[1] if "_" in case else None
    bn = tag == "bn"
    if graph_mode:
        A, X, gt, y, idx, M0, _ = graph_case(4)
        W = graph_weights() if tag is None else var_weights(tag, "graphs")
    else:
        fx = util.load_fixture("rand")
        W = fx.weights if tag is None else var_weights(tag, "rand")
        A, X, gt, y, idx, M0, _ = node_case(fx, 33, n_hops=4 if tag == "L4" else 3)
    _, st = D.explain_closed_form(A, X, gt, y, idx, W, M0, hp=O.default_hparams(num_epochs=1), graph_mode=graph_mode, bn=bn,
                                  return_state=True)
    g = MG.mask_grads(A, X, gt, y, idx, W, M0, np.zeros(X.shape[1]), O.default_hparams(), graph_mode=graph_mode, bn=bn, unconstrained=True)
    gM, gF = g.gM, g.gF
    assert np.abs(gM).max() > 0 and np.abs(gF).max() > 0
    assert np.abs(st["gM"] - gM).max() <= 1e-9 * max(1.0, np.abs(gM).max()), case
    assert np.abs(st["gF"] - gF).max() <= 1e-9, case
    off = ~np.asarray(A, bool) & ~np.eye(len(A), dtype=bool)
    assert np.abs(gM[off]).max() > 1e-6   # non-edges carry more than the regularisers: the dense path is exercised


@pytest.mark.parametrize("opt", ["adam", "sgd", "rmsprop", "adagrad", "adamstep"])
def test_closed_form_follows_port(opt):
    """fp64 closed form vs the port at 10 epochs, every optimiser (and a scheduler), node and graph mode: within 1e-6."""
    over = dict(opt="adam", opt_scheduler="step", opt_decay_step=3, opt_decay_rate=0.5) if opt == "adamstep" else dict(opt=opt)
    hp = O.default_hparams(num_epochs=10, **over)
    fx = util.load_fixture("rand")
    for node in (33, 149):
        A, X, gt, y, idx, M0, (ei, ej) = node_case(fx, node)
        port = O.explain_dense_torch(A, X, gt, y, idx, fx.weights, M0, hp=hp, unconstrained=True)
        cf = D.explain_closed_form(A, X, gt, y, idx, fx.weights, M0, hp=hp)
        assert O.rel_l2(cf[ei, ej], port[ei, ej]) <= 1e-6, (opt, node, O.rel_l2(cf[ei, ej], port[ei, ej]))
    W = graph_weights()
    for g in (2, 9):
        A, X, gt, _, _, M0, (ei, ej) = graph_case(g)
        port = O.explain_dense_torch(A, X, gt, None, 0, W, M0, hp=hp, graph_mode=True, unconstrained=True)
        cf = D.explain_closed_form(A, X, gt, None, 0, W, M0, hp=hp, graph_mode=True)
        assert O.rel_l2(cf[ei, ej], port[ei, ej]) <= 1e-6, (opt, g, O.rel_l2(cf[ei, ej], port[ei, ej]))
