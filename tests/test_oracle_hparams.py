"""CPU: the specification off the default hyper-parameters.

  * the line-by-line port reproduces what the UNMODIFIED reference returns under --lr 0.01 / 0.5, --epochs 2 / 300 and Adam with the
    step and cosine schedulers (tests/golden/hparams_golden.npz, tools/gen_hparams_golden.py), node and graph mode;
  * under the Adam betas / eps and loss coefficients of HSETS, the fp64 closed form (gnnx_oracle.explain_closed_form) has torch
    autograd's dL/dM and dL/dF, and it and the edge-list specification (kernel_spec.explain_pruned_edges, whose c_feat / c_lap are
    coef_feat_size / coef_lap) take the fp64 port's Adam steps, node and graph mode, --bn, 2 and 4 layers.  The GPU tests compare the
    kernels with these restatements (tests/test_gpu_hparams.py)."""
import math

import numpy as np
import pytest
import torch

import gnnx_oracle as O
import kernel_spec as KS
import mask_grad_oracle as MG
import util
from test_oracle_graph_variants import dense_m0, model_of
from test_oracle_spec_state import _case

# Hyper-parameter sets, in gnnx_oracle.default_hparams names.  H1: eps large enough to matter against sqrt(v_hat); H2: every loss
# coefficient off its default; H0: the prediction loss alone.
HSETS = {"H1": dict(beta1=0.5, beta2=0.99, eps=1e-3),
         "H2": dict(size=0.05, ent=0.3, lap=4.0, feat_size=0.2),
         "H0": dict(size=0.0, ent=0.0, lap=0.0, feat_size=0.0)}
GX_NAMES = dict(beta1="beta1", beta2="beta2", eps="eps", size="coef_size", ent="coef_ent", lap="coef_lap", feat_size="coef_feat_size")
KS_NAMES = dict(beta1="beta1", beta2="beta2", eps="eps", size="c_size", ent="c_ent", lap="c_lap", feat_size="c_feat")


def gx_over(hset):
    """The gx_hparams fields of a set (engine.make_hparams keywords)."""
    return {GX_NAMES[k]: v for k, v in HSETS[hset].items()}


def golden():
    return np.load(util.GOLDEN + "/hparams_golden.npz")


def case_hparams(H, tag):
    """(epochs, gnnx_oracle hparams) of a fixture case."""
    i = [str(t) for t in H["case_tags"]].index(tag)
    sched = str(H["case_scheduler"][i])
    E = int(H["case_epochs"][i])
    return E, O.default_hparams(num_epochs=E, lr=float(H["case_lr"][i]), opt_scheduler=sched, opt_decay_step=int(H["case_decay_step"][i]),
                                opt_decay_rate=float(H["case_decay_rate"][i]), opt_restart=int(H["case_restart"][i]))


# ------------------------------------------------------------------------------------ the reference fixture
def test_fixture_cases_reach_what_they_are_meant_to():
    H = golden()
    tags = [str(t) for t in H["case_tags"]]
    assert tags == ["lr001", "lr05", "e2", "e300", "step", "cos"]
    _, step = case_hparams(H, "step")
    _, cos = case_hparams(H, "cos")
    assert step.num_epochs // step.opt_decay_step >= 4                     # several decay boundaries inside the run
    assert cos.opt_restart < cos.num_epochs // 2                            # the cosine reaches lr = 0 and rises again
    for tag in tags:
        assert len(H["graphs_%s_gids" % tag]) >= 10
        for which in ("rand", "syn4", "syn1"):
            assert len(H["%s_%s_nodes" % (which, tag)]) >= len(H[which + "_nodes"]) - 1, (which, tag)
            assert np.isfinite(H["%s_%s_spread" % (which, tag)]).all()


@pytest.mark.parametrize("which", ["rand", "syn4", "syn1"])
def test_port_reproduces_the_reference_nodes(which):
    H = golden()
    fx = util.load_fixture(which)
    for tag in (str(t) for t in H["case_tags"]):
        E, hp = case_hparams(H, tag)
        for node in (int(v) for v in H["%s_%s_nodes" % (which, tag)]):
            idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(fx.rowptr, fx.col, fx.feat, fx.label, node, 3)
            A = O.dense_from_csr(srp, scol)
            ei, ej = np.nonzero(A)
            M0 = np.ones(A.shape, np.float32); M0[ei, ej] = fx.gold["n%d_m0" % node]
            port = O.explain_dense_torch(A, X, int(lab[idx]), fx.pred_label[nbrs], idx, fx.weights, M0, hp=hp)
            assert O.rel_l2(port[ei, ej], H["%s_%s_n%d_mask" % (which, tag, node)]) < 1e-6, (tag, node)


def test_port_reproduces_the_reference_graphs():
    H = golden()
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    w = {k: gg[k] for k in util.WKEYS}
    for tag in (str(t) for t in H["case_tags"]):
        E, hp = case_hparams(H, tag)
        for g in (int(v) for v in H["graphs_%s_gids" % tag]):
            A = gg["adj"][g].astype(np.float64)
            ei, ej = np.nonzero(A)
            port = O.explain_dense_torch(A, gg["feat"][g], int(gg["label"][g]), None, 0, w, dense_m0(gg, g), hp=hp, graph_mode=True)
            assert O.rel_l2(port[ei, ej], H["graphs_%s_g%d_mask" % (tag, g)]) < 1e-6, (tag, g)


def test_cases_differ_from_the_defaults():
    """Every case moves the reference's mask away from the default run's: a kernel that ignored the setting would fail."""
    H = golden()
    fx = util.load_fixture("rand")
    node = int(H["rand_nodes"][0])
    gold30 = np.load(util.GOLDEN + "/rand_golden_e30.npz")["n%d_mask" % node]
    for tag in ("lr001", "lr05", "step", "cos"):
        assert O.rel_l2(H["rand_%s_n%d_mask" % (tag, node)], gold30) > 1e-2, tag
    assert fx.gold["n%d_mask" % node].shape == H["rand_e300_n%d_mask" % node].shape


# ------------------------------------------------------------------------------------ the specification under HSETS
def _autograd_grads(A, X, gt, pl, idx, w, M, F, hp, graph_mode, bn):
    """torch autograd's dL/dM and dL/dF of the reference's loss (explain.py:665-808) at (M, F), float64."""
    g = MG.mask_grads(A, X, gt, pl, idx, w, M, F, hp, graph_mode=graph_mode, bn=bn)
    return g.gM, g.gF


def _node_problem(L, bn, node, seed):
    rowptr, col, feat, label, pred_label, w = _case(70, 2, L, 9, 4, L, seed)
    idx, srp, scol, X, lab, nbrs = O.extract_neighborhood(rowptr, col, feat, label, node, L)
    A = O.dense_from_csr(srp, scol)
    M0 = (1 + 0.3 * np.random.default_rng(seed).normal(size=A.shape)).astype(np.float32)
    return dict(A=A, X=X, gt=int(lab[idx]), pl=pred_label[nbrs], idx=idx, w=w, M0=M0, bn=bn, graph_mode=False, srp=srp, scol=scol)


def _graph_problem(tag, g):
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    if tag == "default":
        w, bn = {k: gg[k] for k in util.WKEYS}, False
    else:
        w, _, bn = model_of(np.load(util.GOLDEN + "/graph_variants_golden.npz"), tag)
    return dict(A=gg["adj"][g].astype(np.float64), X=gg["feat"][g], gt=int(gg["label"][g]), pl=None, idx=0, w=w, M0=dense_m0(gg, g), bn=bn,
                graph_mode=True)


PROBLEMS = {"node_L3": lambda: _node_problem(3, False, 11, 1), "node_L2_bn": lambda: _node_problem(2, True, 5, 2),
            "node_L4_bn": lambda: _node_problem(4, True, 40, 3), "node_L4": lambda: _node_problem(4, False, 23, 4),
            "graph_L3": lambda: _graph_problem("default", 3), "graph_L2": lambda: _graph_problem("L2", 5),
            "graph_bn": lambda: _graph_problem("bn", 8), "graph_L4": lambda: _graph_problem("L4", 1)}


def _args(p):
    return (p["A"], p["X"], p["gt"], p["pl"], p["idx"], p["w"])


@pytest.mark.parametrize("hset", list(HSETS))
@pytest.mark.parametrize("prob", list(PROBLEMS))
def test_closed_form_gradient_is_autograds(prob, hset):
    p = PROBLEMS[prob]()
    hp = O.default_hparams(num_epochs=1, **HSETS[hset])
    d = p["X"].shape[1]
    F = 0.7 * np.random.default_rng(9).normal(size=d)          # a feature mask away from its initial 0
    z = np.zeros_like(p["M0"], np.float64)
    init = dict(m=z, v=z, feat=np.stack([F, np.zeros(d), np.zeros(d)]), step=0)
    _, st = O.explain_closed_form(*_args(p), p["M0"], hp=hp, graph_mode=p["graph_mode"], bn=p["bn"], return_state=True, init_state=init)
    gM, gF = _autograd_grads(*_args(p), p["M0"], F, hp, p["graph_mode"], p["bn"])
    assert np.abs(st["gM"] - gM).max() <= 1e-9 * np.abs(gM).max(), (prob, hset)
    assert np.abs(st["gF"] - gF).max() <= 1e-9 * np.abs(gF).max(), (prob, hset)


@pytest.mark.parametrize("hset", list(HSETS))
@pytest.mark.parametrize("prob", list(PROBLEMS))
def test_specification_takes_the_ports_adam_steps(prob, hset):
    """After one and after five updates, the closed form (and, in node mode, the edge-list specification) lands on the fp64 port,
    which runs torch.optim.Adam with the set's betas and eps."""
    p = PROBLEMS[prob]()
    A = p["A"]
    ei, ej = np.nonzero(A)
    for E in (2, 6):
        hp = O.default_hparams(num_epochs=E, **HSETS[hset])
        port, fm = O.explain_dense_torch(*_args(p), p["M0"], hp=hp, graph_mode=p["graph_mode"], bn=p["bn"], dtype=torch.float64,
                                         return_feat=True)
        cf = O.explain_closed_form(*_args(p), p["M0"], hp=hp, graph_mode=p["graph_mode"], bn=p["bn"])
        _, st = O.explain_closed_form(*_args(p), p["M0"], hp=O.default_hparams(num_epochs=E - 1, **HSETS[hset]), graph_mode=p["graph_mode"],
                                      bn=p["bn"], return_state=True)
        assert O.rel_l2(cf[ei, ej], port[ei, ej]) <= 1e-9, (prob, hset, E)
        assert np.abs(1 / (1 + np.exp(-st["F"])) - fm).max() <= 1e-9, (prob, hset, E)
        if not p["graph_mode"]:
            ks = {KS_NAMES[k]: v for k, v in HSETS[hset].items()}
            a, _, F = KS.explain_pruned_edges(p["srp"], p["scol"], p["X"], p["gt"], p["pl"], p["idx"], p["w"], p["M0"][ei, ej], num_epochs=E,
                                              bn=p["bn"], return_F=True, **ks)
            assert O.rel_l2(a, port[ei, ej]) <= 1e-9, (prob, hset, E)
            assert np.abs(1 / (1 + np.exp(-F)) - fm).max() <= 1e-9, (prob, hset, E)


@pytest.mark.parametrize("hset", list(HSETS))
def test_each_set_changes_the_result(hset):
    """The GPU tests compare kernels under each set: the set must move the port far from the default run, or they test nothing."""
    for prob in ("node_L3", "graph_L3"):
        p = PROBLEMS[prob]()
        ei, ej = np.nonzero(p["A"])
        base = O.explain_dense_torch(*_args(p), p["M0"], hp=O.default_hparams(num_epochs=20), graph_mode=p["graph_mode"])
        other = O.explain_dense_torch(*_args(p), p["M0"], hp=O.default_hparams(num_epochs=20, **HSETS[hset]), graph_mode=p["graph_mode"])
        assert O.rel_l2(other[ei, ej], base[ei, ej]) > 1e-2, (prob, hset)


def test_adam_second_moment_with_float_beta2():
    """gx_hparams carries beta2 as a float and the kernels form 1 - fl(beta2) in float, where torch forms fl64(1 - beta2) from the Python
    scalar: exp_avg_sq differs by 1.29e-5 relative at beta2 = 0.999.  The bias correction uses the same fl(beta2), so the kernels run a
    consistent Adam with beta2 = 0.99900001287; after one step the update is the same to far below 1e-6 relative."""
    b2f = float(np.float32(0.999))
    one_minus = float(np.float32(1) - np.float32(0.999))
    torch_one_minus = 1 - 0.999
    assert abs(one_minus / torch_one_minus - 1 - (-1.29e-5)) < 0.01e-5
    g = 0.37
    v_k, v_t = one_minus * g * g, torch_one_minus * g * g
    step_k = g / (math.sqrt(v_k) / math.sqrt(1 - b2f) + 1e-8)
    step_t = g / (math.sqrt(v_t) / math.sqrt(1 - 0.999) + 1e-8)
    assert abs(step_k / step_t - 1) < 1e-6
