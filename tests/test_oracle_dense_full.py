"""The WHOLE unconstrained mask on the CPU: the line-by-line port against the unmodified reference's full masked_adj
(tests/golden/unconstrained_full_golden.npz, tools/gen_unconstrained_full_golden.py), bit for bit over all n^2 entries, and the fp64
closed form -- what tests/test_gpu_dense_full.py checks the dense kernel against -- against the port: its full matrix, its per-epoch
regulariser sums (the kernel's trace columns) and its MLP-head path."""
import os

import numpy as np
import pytest
import torch

import dense_oracle as D
import gnnx_oracle as O
import util

UF = np.load(os.path.join(util.GOLDEN, "unconstrained_full_golden.npz"))
GG = np.load(os.path.join(util.GOLDEN, "graphs_golden.npz"))


def graph_weights():
    return {k: GG[k] for k in util.WKEYS}


def node_case(fx, node):
    idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(fx.rowptr, fx.col, fx.feat, fx.label, node, 3)
    A = O.dense_from_csr(srp, scol)
    return A, X, int(lab[idx]), fx.pred_label[nbrs], idx, O.draw_m0(len(nbrs), seed=int(fx.gold["n%d_seed" % node])), nbrs


def graph_case(g):
    A = GG["adj"][g].astype(np.float64)
    return A, GG["feat"][g], int(GG["label"][g]), None, 0, O.draw_m0(int(GG["max_nodes"]), seed=int(GG["g%d_seed" % g]))


def fixture_cases():
    for which in ("syn1", "syn4", "rand"):
        for v in UF[which + "_nodes"]:
            yield which, int(v)
    for g in UF["graphs"]:
        yield "graphs", int(g)


def inputs(which, v):
    """(A, X, gt, y, idx, W, M0, graph_mode, key prefix) of a fixture case."""
    if which == "graphs":
        A, X, gt, y, idx, M0 = graph_case(v)
        return A, X, gt, y, idx, graph_weights(), M0, True, "graphs_g%d" % v
    fx = util.load_fixture(which)
    A, X, gt, y, idx, M0, nbrs = node_case(fx, v)
    assert np.array_equal(nbrs, UF["%s_n%d_nbrs" % (which, v)])
    return A, X, gt, y, idx, fx.weights, M0, False, "%s_n%d" % (which, v)


def test_fixture_has_every_entry_class():
    """Node tasks have edge and non-edge entries; the graphs also padding or isolated rows (the "pad" class)."""
    for which, v in fixture_cases():
        key = ("graphs_g%d" % v if which == "graphs" else "%s_n%d" % (which, v)) + "_e10"
        want = {"edge", "nonedge", "pad"} if which == "graphs" else {"edge", "nonedge"}
        assert {k[len(key) + 8:] for k in UF.files if k.startswith(key + "_spread_")} == want, key


@pytest.mark.parametrize("which,v", list(fixture_cases()))
def test_port_reproduces_reference_full_mask(which, v):
    """Every entry of the reference's masked_adj at 10 and 30 epochs, bit for bit, and the fp64 closed form within the distance the
    fixture recorded for each entry class."""
    A, X, gt, y, idx, W, M0, graph, key = inputs(which, v)
    for E in (int(e) for e in UF["epochs"]):
        hp = O.default_hparams(num_epochs=E)
        port = O.explain_dense_torch(A, X, gt, y, idx, W, M0, hp=hp, graph_mode=graph, full=True, unconstrained=True)
        ref = UF["%s_e%d_full" % (key, E)]
        assert port.shape == ref.shape and np.array_equal(port.astype(np.float32), ref), (key, E, np.abs(port - ref).max())
        assert np.array_equal(port * A, O.explain_dense_torch(A, X, gt, y, idx, W, M0, hp=hp, graph_mode=graph, unconstrained=True))
        cf = D.explain_closed_form(A, X, gt, y, idx, W, M0, hp=hp, graph_mode=graph, full=True)
        for c, (r, k) in D.entry_classes(A).items():
            rec = float(UF["%s_e%d_cfdist_%s" % (key, E, c)])
            got = O.rel_l2(cf[r, k], port[r, k])
            assert got <= 1.1 * rec + 1e-9, (key, E, c, got, rec)
            assert rec <= 1e-5 or which == "graphs", (key, E, c, rec)   # the node fixtures are well conditioned


OPTS = [dict(opt=o, opt_scheduler=s, opt_decay_step=3, opt_decay_rate=0.5, opt_restart=4)
        for o in ("adam", "sgd", "rmsprop", "adagrad") for s in ("none", "step", "cos")]


@pytest.mark.parametrize("over", OPTS + [dict(beta1=0.5, beta2=0.99, eps=1e-3), dict(size=0.05, ent=0.3, lap=4.0, feat_size=0.2)],
                         ids=["%s-%s" % (o["opt"], o["opt_scheduler"]) for o in OPTS] + ["H1", "H2"])
def test_closed_form_full_mask_and_trace_follow_port(over):
    """Every optimiser, scheduler and hyper-parameter set of tests/test_gpu_dense_full.py, 10 epochs: the fp64 closed form's whole
    mask within 1e-5 of the port's per class, and its per-epoch regulariser sums (size, entropy over all n^2 entries, the diagonal
    included; feat_size) equal to the terms of the port's loss to 1e-6."""
    hp = O.default_hparams(num_epochs=10, **over)
    fx = util.load_fixture("rand")
    A, X, gt, y, idx, M0, _ = node_case(fx, 33)
    for graph, (A, X, gt, y, idx, M0), W in ((False, (A, X, gt, y, idx, M0), fx.weights), (True, graph_case(9), graph_weights())):
        n, d = len(A), X.shape[1]
        ptr, ctr = [], []
        port = O.explain_dense_torch(A, X, gt, y, idx, W, M0, hp=hp, graph_mode=graph, trace=ptr, full=True, unconstrained=True)
        cf = D.explain_closed_form(A, X, gt, y, idx, W, M0, hp=hp, graph_mode=graph, full=True, trace=ctr)
        assert len(ctr) == len(ptr) == hp.num_epochs and np.array_equal(ctr[-1]["a"], cf)
        for c, (r, k) in D.entry_classes(A).items():
            assert O.rel_l2(cf[r, k], port[r, k]) <= 1e-5, (over, graph, c, O.rel_l2(cf[r, k], port[r, k]))
        for p, q in zip(ptr, ctr):
            for name, val in (("size", hp.size * q["size"]), ("ent", hp.ent * q["ent"] / (n * n)), ("feat_size", hp.feat_size * q["feat"] / d)):
                assert abs(val - p[name]) <= 1e-6 * abs(p[name]) + 1e-12, (over, graph, name, val, p[name])


@pytest.mark.parametrize("graph", [False, True], ids=["node", "graph"])
def test_closed_form_head_follows_fp64_port(graph):
    """The closed form's MLP-head readout (Linear, ReLU, .., Linear) against the head port in fp64 autograd, 6 epochs, whole mask."""
    rng = np.random.default_rng(11)
    if graph:
        A, X, gt, y, idx, M0 = graph_case(4)
    else:
        fx = util.load_fixture("rand")
        A, X, gt, y, idx, M0, _ = node_case(fx, 149)
    d, C = X.shape[1], 2 if graph else 3
    sc = lambda *s: (rng.normal(size=s) * 0.4).astype(np.float32)
    W = {"W1": sc(d, 20), "b1": sc(20), "W2": sc(20, 20), "b2": sc(20), "W3": sc(20, 20), "b3": sc(20),
         "head": [(sc(24, 60), sc(24)), (sc(10, 24), sc(10))], "Wp": sc(C, 10), "bp": sc(C)}
    hp = O.default_hparams(num_epochs=6)
    cf = D.explain_closed_form(A, X, gt, y, idx, W, M0, hp=hp, graph_mode=graph, full=True)
    ref = O.explain_dense_torch(A, X, gt, y, idx, W, M0, hp=hp, graph_mode=graph, dtype=torch.float64, unconstrained=True, full=True)
    off = ~np.eye(len(A), dtype=bool)
    assert np.abs(cf[off] - ref[off]).max() <= 1e-9
    without = D.explain_closed_form(A, X, gt, y, idx, {k: v for k, v in W.items() if k != "head"} | {"Wp": sc(C, 60)}, M0, hp=hp,
                                    graph_mode=graph, full=True)
    assert np.abs(cf - without).max() > 1e-4    # the head changes the trajectory: the comparison is not vacuous
