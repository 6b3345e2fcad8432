"""GPU (-m gpu): graph-classification mode (SURVEY.md 8 row f1) through the C ABI and the drop-in
Explainer, against golden masks produced by the unmodified reference (oracle/gen_golden.py --only graph:
GcnEncoderGraph, Explainer(graph_mode=True).explain(node_idx=0, graph_idx=g, graph_mode=True))."""
import types

import numpy as np
import pytest
import torch

import gnnx
from gnnx import _abi
import gnnx_oracle as O
import util

pytestmark = pytest.mark.gpu
WK = ["W1", "b1", "W2", "b2", "W3", "b3", "Wp", "bp"]


@pytest.fixture(scope="module")
def gg():
    return np.load(util.GOLDEN + "/graphs_golden.npz")


def _engine(gg):
    eng = gnnx.Engine(0)
    eng.set_model({k: gg[k] for k in WK})
    eng.set_graph_batch(gg["adj"], gg["feat"], gg["label"])
    return eng


@pytest.mark.parametrize("epochs", [10, 100])
def test_graph_masks_match_reference(gg, epochs):
    eng = _engine(gg)
    G = int(gg["num_graphs"])
    gids = list(range(G))
    edge_off = eng.plan_graphs(gids)
    m0 = np.concatenate([gg["g%d_m0" % g] for g in gids])
    assert len(m0) == edge_off[-1]
    out = np.zeros(len(m0), np.float32)
    eng.explain_graphs_host(eng.make_hparams(num_epochs=epochs), m0, out)
    errs = [util.rel_l2(out[edge_off[t]:edge_off[t + 1]], gg["g%d_mask_e%d" % (g, epochs)]) for t, g in enumerate(gids)]
    assert max(errs) <= 1e-4, errs
    # order / batch independence (what makes multi-GPU sharding bit-identical)
    sub = [7, 2, 11]
    eo = eng.plan_graphs(sub)
    o2 = np.zeros(int(eo[-1]), np.float32)
    eng.explain_graphs_host(eng.make_hparams(num_epochs=epochs), np.concatenate([gg["g%d_m0" % g] for g in sub]), o2)
    for t, g in enumerate(sub):
        assert np.array_equal(o2[eo[t]:eo[t + 1]], out[edge_off[g]:edge_off[g + 1]])
    eng.close()


def test_graph_mode_against_oracle_random_weights(gg):
    """Different weights (positive biases => the edge-less constant wins some max-pools), 30 epochs, vs the
    line-by-line torch port."""
    rng = np.random.default_rng(5)
    W = {k: (rng.normal(size=gg[k].shape) * 0.5).astype(np.float32) for k in WK}
    for b in ("b1", "b2", "b3"):
        W[b] = np.abs(W[b]) + 0.2
    eng = gnnx.Engine(0)
    eng.set_model(W)
    eng.set_graph_batch(gg["adj"], gg["feat"], gg["label"])
    gids = [0, 3, 5, 9]
    edge_off = eng.plan_graphs(gids)
    n = int(gg["max_nodes"])
    m0s, dense = [], []
    for t, g in enumerate(gids):
        M0 = O.draw_m0(n, seed=900 + g)
        r, c = eng.graph_rows_cols(g)
        m0s.append(M0[r, c]); dense.append(M0)
    out = np.zeros(int(edge_off[-1]), np.float32)
    fm = np.zeros((len(gids), gg["feat"].shape[2]), np.float32)
    eng.explain_graphs_host(eng.make_hparams(num_epochs=30), np.concatenate(m0s).astype(np.float32), out, fm)
    for t, g in enumerate(gids):
        # edge masks vs the port at 1e-4, feature masks vs the fp64 closed form
        util.check_graph_masks(gg["adj"][g], gg["feat"][g], gg["label"][g], W, dense[t], 30, out[edge_off[t]:edge_off[t + 1]], fm[t],
                               eng.graph_rows_cols(g), edge_tol=1e-4)
    eng.close()


def test_explainer_dropin_graph_mode(gg, tmp_path):
    args = types.SimpleNamespace(num_gc_layers=3, num_epochs=10, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                 mask_bias=False, gpu=False, bias=True, method="base", dataset="graphs", bmname=None,
                                 hidden_dim=20, output_dim=20, name_suffix="", explainer_suffix="", logdir=str(tmp_path))
    model = gnnx.models.GcnEncoderGraph(14, 20, 20, 2, 3, bn=False, args=args)
    sd = {"conv_first.weight": gg["W1"], "conv_first.bias": gg["b1"], "conv_block.0.weight": gg["W2"], "conv_block.0.bias": gg["b2"],
          "conv_last.weight": gg["W3"], "conv_last.bias": gg["b3"], "pred_model.weight": gg["Wp"], "pred_model.bias": gg["bp"]}
    model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    ex = gnnx.Explainer(model=model, adj=torch.tensor(gg["adj"], dtype=torch.float), feat=torch.tensor(gg["feat"]),
                        label=torch.tensor(gg["label"]), pred=gg["pred"], train_idx=[], args=args, writer=None,
                        print_training=False, graph_mode=True, graph_idx=0)
    n = int(gg["max_nodes"])
    for g in (1, 8):
        torch.manual_seed(int(gg["g%d_seed" % g]))
        masked = ex.explain(node_idx=0, graph_idx=g, graph_mode=True)
        assert masked.shape == (n, n) and masked.dtype == np.float64
        ei, ej = np.nonzero(gg["adj"][g])
        assert util.rel_l2(masked[ei, ej], gg["g%d_mask_e10" % g]) <= 1e-4
        off = masked.copy(); off[ei, ej] = 0
        assert np.all(off == 0)
    torch.manual_seed(1)
    a = [ex.explain(0, graph_idx=g, graph_mode=True) for g in (4, 6)]
    torch.manual_seed(1)
    b = ex.explain_graphs([4, 6])
    assert all(np.array_equal(x, y) for x, y in zip(a, b))


def test_graph_mode_other_widths(gg):
    rng = np.random.default_rng(77)
    hid, emb, d, C = 12, 24, 14, 3
    sc = lambda *s: (rng.normal(size=s) * 0.5).astype(np.float32)
    W = dict(W1=sc(d, hid), b1=sc(hid), W2=sc(hid, hid), b2=sc(hid), W3=sc(hid, emb), b3=sc(emb), Wp=sc(C, 2 * hid + emb), bp=sc(C))
    eng = gnnx.Engine(0)
    eng.set_model(W)
    label = gg["label"] % C
    eng.set_graph_batch(gg["adj"], gg["feat"], label)
    gids = [1, 6, 10]
    edge_off = eng.plan_graphs(gids)
    n = int(gg["max_nodes"])
    m0s, dense = [], []
    for g in gids:
        M0 = O.draw_m0(n, seed=40 + g)
        r, c = eng.graph_rows_cols(g)
        m0s.append(M0[r, c]); dense.append(M0)
    out = np.zeros(int(edge_off[-1]), np.float32)
    fm = np.zeros((len(gids), d), np.float32)
    eng.explain_graphs_host(eng.make_hparams(num_epochs=20), np.concatenate(m0s).astype(np.float32), out, fm)
    for t, g in enumerate(gids):
        util.check_graph_masks(gg["adj"][g], gg["feat"][g], label[g], W, dense[t], 20, out[edge_off[t]:edge_off[t + 1]], fm[t],
                               eng.graph_rows_cols(g), edge_tol=1e-4)
    eng.close()
