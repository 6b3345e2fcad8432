"""CPU: the specification of graph-classification mode with the model and optimiser variants, against the masks the UNMODIFIED
reference returned (tests/golden/graph_variants_golden.npz, tools/gen_graph_variants_golden.py; GcnEncoderGraph with
num_gc_layers 2 / 4, --bn, hidden 64 / output 48, and --opt sgd / rmsprop / adagrad / sgd + StepLR; 30 epochs).
The line-by-line torch port reproduces the reference to round-off; the fp64 closed form (Adam) lands within the tolerance rule of
tests/util.py: 1e-4, or 3 x the reference's own spread under +-1 ulp nudges of M0."""
import numpy as np
import pytest

import gnnx_oracle as O
import util

MODEL_TAGS = ["L2", "L4", "bn", "bn_L4", "wide"]
OPT_TAGS = {"sgd": dict(opt="sgd"), "rmsprop": dict(opt="rmsprop"), "adagrad": dict(opt="adagrad"),
            "sgdstep": dict(opt="sgd", opt_scheduler="step", opt_decay_step=10, opt_decay_rate=0.3)}
BASE_KEYS = ["W1", "b1", "W2", "b2", "W3", "b3", "Wp", "bp"]


@pytest.fixture(scope="module")
def gv():
    return np.load(util.GOLDEN + "/graph_variants_golden.npz")


@pytest.fixture(scope="module")
def gg():
    return np.load(util.GOLDEN + "/graphs_golden.npz")


def model_of(gv, tag):
    """(weights, num_layers, bn) of a model-variant tag of the golden file."""
    L = int(gv[tag + "_L"])
    w = {k: gv["%s_%s" % (tag, k)] for k in ["W%d" % l for l in range(1, L + 1)] + ["b%d" % l for l in range(1, L + 1)] + ["Wp", "bp"]}
    return w, L, bool(gv[tag + "_bn"])


def dense_m0(gg, g):
    return O.draw_m0(int(gg["max_nodes"]), seed=int(gg["g%d_seed" % g]))


def test_golden_reuses_the_graph_mode_fixture(gv, gg):
    G = int(gg["num_graphs"])
    for g in range(G):
        ei, ej = np.nonzero(gg["adj"][g])
        assert np.array_equal(dense_m0(gg, g)[ei, ej], gg["g%d_m0" % g])
        for tag in MODEL_TAGS + list(OPT_TAGS):
            assert gv["%s_g%d_mask" % (tag, g)].shape == (len(ei),)
    assert int(gv["num_epochs"]) == 30
    assert [int(gv[t + "_L"]) for t in MODEL_TAGS] == [2, 4, 3, 4, 3]
    assert gv["wide_W1"].shape == (gg["feat"].shape[2], 64) and gv["wide_W3"].shape == (64, 48)


@pytest.mark.parametrize("tag", MODEL_TAGS)
def test_model_variants_port_and_closed_form(gv, gg, tag):
    w, L, bn = model_of(gv, tag)
    hp = O.default_hparams(num_epochs=int(gv["num_epochs"]))
    for g in range(int(gg["num_graphs"])):
        A = gg["adj"][g].astype(np.float64)
        ei, ej = np.nonzero(A)
        ref = gv["%s_g%d_mask" % (tag, g)]
        M0 = dense_m0(gg, g)
        port = O.explain_dense_torch(A, gg["feat"][g], int(gg["label"][g]), None, 0, w, M0, hp=hp, graph_mode=True, bn=bn)
        assert O.rel_l2(port[ei, ej], ref) < 1e-6, (tag, g)
        c64 = O.explain_closed_form(A, gg["feat"][g], int(gg["label"][g]), None, 0, w, M0, hp=hp, graph_mode=True, bn=bn)
        tol = max(1e-4, 3 * float(gv[tag + "_spread"][g]))
        assert O.rel_l2(c64[ei, ej], ref) <= tol, (tag, g, O.rel_l2(c64[ei, ej], ref), tol)


@pytest.mark.parametrize("tag", list(OPT_TAGS))
def test_optimiser_variants_port(gv, gg, tag):
    w = {k: gg[k] for k in BASE_KEYS}
    hp = O.default_hparams(num_epochs=int(gv["num_epochs"]), **OPT_TAGS[tag])
    for g in range(int(gg["num_graphs"])):
        A = gg["adj"][g].astype(np.float64)
        ei, ej = np.nonzero(A)
        port = O.explain_dense_torch(A, gg["feat"][g], int(gg["label"][g]), None, 0, w, dense_m0(gg, g), hp=hp, graph_mode=True)
        assert O.rel_l2(port[ei, ej], gv["%s_g%d_mask" % (tag, g)]) < 1e-6, (tag, g)


def test_edgeless_rows_take_the_bias_constant(gv, gg):
    """Padding rows and the isolated node of graph 3 hold bn(relu(normalize(b_l))) at every hidden layer, whatever the mask: the
    constant the kernel pools instead of those rows."""
    import torch
    w, L, bn = model_of(gv, "bn_L4")
    W = O.weights_to_torch(w, requires_grad=False)
    g = 3
    A = gg["adj"][g].astype(np.float32)
    empty = np.nonzero(A.sum(1) == 0)[0]
    assert 0 in empty and len(empty) < A.shape[0]
    outs = []
    h = torch.tensor(gg["feat"][g][None])
    adj = torch.tensor(A[None] * 0.7)
    for l in range(L):
        y = torch.nn.functional.normalize(torch.matmul(torch.matmul(adj, h), W["conv_w"][l]) + W["conv_b"][l], p=2, dim=2)
        if l < L - 1:
            y = torch.nn.functional.batch_norm(torch.relu(y), None, None, None, None, True, 0.1, 1e-5)
        outs.append(y[0].numpy()); h = y
    for l in range(L):
        b = np.asarray(w["b%d" % (l + 1)], np.float64)
        c = b / max(np.linalg.norm(b), 1e-12)
        if l < L - 1:
            c = np.maximum(c, 0)
            c = (c - c.mean()) / np.sqrt(c.var() + 1e-5)
        assert np.allclose(outs[l][empty], c[None, :], atol=1e-5)
