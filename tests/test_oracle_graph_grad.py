"""CPU: the specifications of the gradient baseline in graph-classification mode (tests/graph_grad_oracle.py) against the unmodified
reference's ExplainModule.adj_feat_grad (tests/golden/graph_grad_golden.npz, tools/gen_graph_grad_golden.py), on the 12 padded graphs of
graphs_golden.npz with two models."""
import numpy as np
import pytest

import gnnx_oracle as O
import graph_grad_oracle as GO
import util

WKEYS = ("W1", "b1", "W2", "b2", "W3", "b3", "Wp", "bp")


@pytest.fixture(scope="module")
def golden():
    gold = np.load(util.GOLDEN + "/graph_grad_golden.npz")
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    return gold, gg


def weights(gold, m):
    return {k: gold["%s_w_%s" % (m, k)].astype(np.float32) for k in WKEYS}


def _cases(gold, gg):
    for m in gold["models"]:
        m = str(m)
        w = weights(gold, m)
        for g in range(int(gg["num_graphs"])):
            yield m, w, g, gg["adj"][g].astype(np.float64), gg["feat"][g], np.nonzero(gg["adj"][g])


def test_golden_labels_are_the_model_predictions(golden):
    """explain.py:102: the label is argmax(pred[0][g]); the ports' -1 (the forward's own arg-max) finds the same label."""
    gold, gg = golden
    for m, w, g, A, X, rc in _cases(gold, gg):
        assert int(gold["%s_g%d_label" % (m, g)]) == int(np.argmax(gold[m + "_pred"][0][g]))
        assert GO.grad_graph_torch(A, X, -1, w, return_label=True)[1] == int(gold["%s_g%d_label" % (m, g)]), (m, g)
        assert GO.grad_graph_torch(A, X, -1, w, dtype=np.float64, return_label=True)[1] == int(gold["%s_g%d_label" % (m, g)]), (m, g)


@pytest.mark.parametrize("key", ["", "alt_"])
def test_ports_match_reference_golden(golden, key):
    """fp32 port within 1e-6 relative L2 of the reference on every graph, the fp64 specification within 1e-5, at the predicted label and
    at a label the model does not predict."""
    gold, gg = golden
    for m, w, g, A, X, rc in _cases(gold, gg):
        ref = gold["%s_g%d_%smask" % (m, g, key)].astype(np.float64)
        lab = int(gold["%s_g%d_%slabel" % (m, g, key)])
        f32 = GO.grad_graph_torch(A, X, lab, w)
        f64 = GO.grad_graph_torch(A, X, lab, w, dtype=np.float64)
        assert O.rel_l2(f32[rc], ref) <= 1e-6, (m, g, O.rel_l2(f32[rc], ref))
        assert O.rel_l2(f64[rc], ref) <= 1e-5, (m, g, O.rel_l2(f64[rc], ref))
        assert not f32[A == 0].any() and not f64[A == 0].any()


@pytest.mark.parametrize("key", ["", "alt_"])
def test_closed_form_is_autograd(golden, key):
    """The hand-derived fp64 form (first arg-max routing of the max-pool) equals fp64 autograd to 1e-10, masks and raw gradient on the
    edges."""
    import torch
    gold, gg = golden
    for m, w, g, A, X, rc in _cases(gold, gg):
        lab = int(gold["%s_g%d_%slabel" % (m, g, key)])
        cf, dA = GO.grad_graph_closed_form(A, X, lab, w, return_grad=True)
        ag = GO.grad_graph_torch(A, X, lab, w, dtype=np.float64)
        assert O.rel_l2(cf[rc], ag[rc]) <= 1e-10, (m, g)
        # the raw gradient, through the same autograd graph
        At = torch.tensor(A[None], requires_grad=True)
        xt = torch.tensor(np.asarray(X, np.float64)[None])
        y = O._gcn_forward_torch(xt, At, O.weights_to_torch(w, dtype=torch.float64), True)
        (-torch.log(torch.softmax(y[0], 0)[lab])).backward()
        ref = At.grad[0].numpy()
        assert np.abs(dA - ref)[rc].max() <= 1e-10 * max(np.abs(ref[rc]).max(), 1e-30), (m, g)


def test_non_predicted_label_changes_the_masks(golden):
    gold, gg = golden
    for m, w, g, A, X, rc in _cases(gold, gg):
        a, b = gold["%s_g%d_mask" % (m, g)], gold["%s_g%d_alt_mask" % (m, g)]
        assert int(gold["%s_g%d_label" % (m, g)]) != int(gold["%s_g%d_alt_label" % (m, g)])
        if len(a):
            assert np.abs(a.astype(np.float64) - b).max() > 1e-5, (m, g)


def test_scaled_golden_is_not_near_constant(golden):
    """A freshly initialised model's masks sit within 0.005 of 0.5; the scaled model's spread makes the comparisons above meaningful."""
    gold, gg = golden
    vals = np.concatenate([gold["scaled_g%d_mask" % g] for g in range(int(gg["num_graphs"]))])
    assert vals.max() - vals.min() >= 0.1
    assert len({int(gold["scaled_g%d_label" % g]) for g in range(int(gg["num_graphs"]))}) == 3   # every class is some graph's label
