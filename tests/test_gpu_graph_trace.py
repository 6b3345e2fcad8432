"""GPU (-m gpu): the per-epoch log print_training prints in graph-classification mode.

  * gx_offedge_regularisers_graphs against the fp64 restatement of its recurrence (test_oracle_graph_trace.offedge_sums), host and
    device buffers, on the golden graphs and on graphs of several launch classes;
  * the loss (kernel trace + off-edge sums), mask density and softmax row against what the UNMODIFIED reference printed
    (tests/golden/graph_trace_golden.npz): default hyper-parameters, other loss coefficients, unconstrained=True;
  * the drop-in Explainer(graph_mode=True, print_training=True): the printed lines, last_trace, masks bit-identical to a silent run,
    the device init, the model-variant notice and runs longer than a trace holds."""
import ctypes as C
import os
import re
import types

import numpy as np
import pytest
import torch

import gnnx
from gnnx import _abi
import util
from test_oracle_graph_trace import case_hparams, offedge_sums
from test_oracle_state import dense_m0
from test_gpu_graph_shapes import _ba, _batch, _classes_run
from test_gpu_graph_variants import GX_ERR_UNSUPPORTED, _random_model

pytestmark = pytest.mark.gpu
GX_ERR_INVALID = -1
TG = np.load(os.path.join(util.GOLDEN, "graph_trace_golden.npz"))
GG = np.load(os.path.join(util.GOLDEN, "graphs_golden.npz"))
NG, NMAX, NC = int(GG["num_graphs"]), int(GG["max_nodes"]), GG["Wp"].shape[0]
LINE = re.compile(r"epoch:\s+(\d+)\s+; loss:\s+(\S+)\s+; mask density:\s+(\S+)\s+; pred:\s+tensor\(\[([^\]]*)\]\)")


def _engine():
    eng = gnnx.Engine(0)
    eng.set_model({k: GG[k] for k in util.WKEYS})
    eng.set_graph_batch(GG["adj"], GG["feat"], GG["label"])
    return eng


def _gx_hparams(eng, hp):
    return eng.make_hparams(num_epochs=hp.num_epochs, lr=hp.lr, coef_size=hp.size, coef_ent=hp.ent, coef_feat_size=hp.feat_size)


def _traced_run(eng, gids, hp):
    """Masks, trace, softmax rows and off-edge sums of the tuned kernel on the golden graphs `gids`, M0 drawn from each graph's seed."""
    eo = eng.plan_graphs(gids)
    dense = [dense_m0(NMAX, int(GG["g%d_seed" % g])) for g in gids]
    m0 = np.concatenate([D[eng.graph_rows_cols(g)] for D, g in zip(dense, gids)]).astype(np.float32)
    out = np.zeros(int(eo[-1]), np.float32)
    trace = np.zeros((len(gids), hp.num_epochs, _abi.GX_TRACE_COLS), np.float32)
    pred = np.zeros((len(gids), hp.num_epochs, NC), np.float32)
    eng.explain_nodes_ex(hp, m0, out, trace=trace, trace_pred=pred, graphs=True)
    off = eng.offedge_regularisers_graphs(hp, np.concatenate([D.ravel() for D in dense]))
    plain = np.zeros_like(out)
    eng.explain_graphs_host(hp, m0, plain)
    assert np.array_equal(plain, out), "requesting a trace changed the masks"
    return eo, out, trace, pred, off


def _printed_loss(hp, trace, off):
    return trace[:, :, _abi.TR_LOSS_EDGES].astype(np.float64) + hp.coef_size * off[:, :, 0] + hp.coef_ent * off[:, :, 1] / (NMAX * NMAX)


# ------------------------------------------------------------------------------------ the entry point
def test_offedge_graphs_is_the_restatement():
    eng = _engine()
    gids = [7, 0, 11, 3, 5, 1, 9, 2, 10, 4, 8, 6]
    eng.plan_graphs(gids)
    E = 30
    hp = eng.make_hparams(num_epochs=E, coef_size=0.05, coef_ent=0.3)
    dense = [dense_m0(NMAX, 40 + g) for g in gids]
    flat = np.concatenate([D.ravel() for D in dense])
    off = eng.offedge_regularisers_graphs(hp, flat)
    for t, g in enumerate(gids):
        want = offedge_sums(dense[t], GG["adj"][g] > 0, E, size=0.05, ent=0.3)
        assert np.abs(off[t] / want - 1).max() <= 2e-5, (g, np.abs(off[t] / want - 1).max())
    # device buffers: the same numbers
    dev = torch.device("cuda", 0)
    m0_dev = torch.from_numpy(flat).to(dev)
    out_dev = torch.zeros(len(gids) * E * 2, dtype=torch.float64, device=dev)
    _abi.check(eng._lib.gx_offedge_regularisers_graphs(eng._h, C.byref(hp), _abi.GX_DEVICE, C.c_void_p(m0_dev.data_ptr()),
                                                       C.c_void_p(out_dev.data_ptr())))
    torch.cuda.synchronize()
    assert np.allclose(out_dev.cpu().numpy().reshape(off.shape), off, rtol=1e-12, atol=0)
    eng.close()


def test_offedge_graphs_over_launch_classes():
    """Graphs of several launch classes in one padded batch: most entries of the small graphs are padding."""
    rng = np.random.default_rng(11)
    n = 160
    sizes = [6, 15, 30, 50, 90, 150]
    adj = _batch([_ba(s) for s in sizes], n)
    feat = rng.normal(size=(len(sizes), n, 14)).astype(np.float32)
    eng = gnnx.Engine(0)
    eng.set_model(_random_model(rng, 3, False, 20, 20, 14, 2, "normal"))
    eng.set_graph_batch(adj, feat, rng.integers(0, 2, len(sizes)))
    gids = [5, 2, 0, 4, 1, 3]
    eo = eng.plan_graphs(gids)
    E = 20
    hp = eng.make_hparams(num_epochs=E)
    dense = [dense_m0(n, 90 + g) for g in gids]
    m0 = np.concatenate([D[eng.graph_rows_cols(g)] for D, g in zip(dense, gids)]).astype(np.float32)
    eng.explain_graphs_host(hp, m0, np.zeros(int(eo[-1]), np.float32))
    assert len(_classes_run(eng)) >= 3, _classes_run(eng)
    off = eng.offedge_regularisers_graphs(hp, np.concatenate([D.ravel() for D in dense]))
    for t, g in enumerate(gids):
        want = offedge_sums(dense[t], adj[g] > 0, E)
        assert np.abs(off[t] / want - 1).max() <= 2e-5, g
    eng.close()


def _offedge_call(eng, fn, hp, m0, out):
    """gx_offedge_regularisers(_graphs) through ctypes with host buffers -> status (the Engine wrappers size their output from a plan)."""
    return fn(eng._h, C.byref(hp), _abi.GX_HOST, C.c_void_p(m0.ctypes.data), C.c_void_p(out.ctypes.data))


def test_refusals():
    eng = _engine()
    lib = eng._lib
    m0 = np.ones(NMAX * NMAX, np.float32)
    out = np.zeros(3072 * 2, np.float64)
    hp = eng.make_hparams(num_epochs=10)
    assert _offedge_call(eng, lib.gx_offedge_regularisers_graphs, hp, m0, out) == GX_ERR_INVALID      # no graph plan
    eng.plan_graphs([0])
    for E in (0, 3073):
        assert _offedge_call(eng, lib.gx_offedge_regularisers_graphs, eng.make_hparams(num_epochs=E), m0, out) == GX_ERR_INVALID, E
    sgd = eng.make_hparams(num_epochs=10, opt=_abi.GX_OPT["sgd"])
    assert _offedge_call(eng, lib.gx_offedge_regularisers_graphs, sgd, m0, out) == GX_ERR_UNSUPPORTED
    assert _offedge_call(eng, lib.gx_offedge_regularisers, hp, m0, out) == GX_ERR_INVALID             # a graph plan is not a node plan
    assert eng.offedge_regularisers_graphs(eng.make_hparams(num_epochs=3072), m0).shape == (1, 3072, 2)
    eng.close()


def test_offedge_beyond_the_grid_y_limit():
    """More planned tasks than one launch's gridDim.y holds (65535): every task still gets its own sums, graph and node mode."""
    rng = np.random.default_rng(5)
    E, n, G = 3, 4, 65536 + 9
    adj = np.zeros((G, n, n), np.uint8)
    adj[:, 0, 1] = adj[:, 1, 0] = adj[:, 1, 2] = adj[:, 2, 1] = 1
    adj[1::2, 2, 3] = adj[1::2, 3, 2] = 1                       # odd graphs use all four rows, even graphs leave row 3 padded
    eng = gnnx.Engine(0)
    eng.set_model(_random_model(rng, 3, False, 20, 20, 14, 2, "normal"))
    eng.set_graph_batch(adj, rng.normal(size=(G, n, 14)).astype(np.float32), np.zeros(G, np.int32))
    eng.plan_graphs(np.arange(G))
    dense = rng.normal(1.0, 0.5, size=(G, n, n)).astype(np.float32)
    off = eng.offedge_regularisers_graphs(eng.make_hparams(num_epochs=E), dense.reshape(-1))
    for g in (0, 1, 65534, 65535, 65536, G - 1):
        assert np.abs(off[g] / offedge_sums(dense[g], adj[g] > 0, E) - 1).max() <= 2e-5, g
    eng.close()
    # node mode: the middle node of a 3-node path, explained 65536 + 9 times (its 3-hop set is the whole path)
    fx = util.load_fixture("rand")
    eng = util.make_engine(fx)
    d = fx.feat.shape[1]
    eng.set_graph_csr(np.array([0, 1, 3, 4]), np.array([1, 0, 2, 1]), rng.normal(size=(3, d)).astype(np.float32), np.zeros(3, np.int32),
                      np.zeros(3, np.int32))
    plan = eng.plan_nodes(np.ones(G, np.int32), 3)
    assert all(plan.n(t) == 3 for t in (0, G - 1))
    dense = rng.normal(1.0, 0.5, size=(G, 3, 3)).astype(np.float32)
    off = eng.offedge_regularisers(eng.make_hparams(num_epochs=E), dense.reshape(-1))
    A = np.array([[0, 1, 0], [1, 0, 1], [0, 1, 0]]) > 0
    for t in (0, 65534, 65535, 65536, G - 1):
        assert np.abs(off[t] / offedge_sums(dense[t], A, E) - 1).max() <= 2e-5, t
    eng.close()


# ------------------------------------------------------------------------------------ against the reference
@pytest.mark.parametrize("case", ["a", "b"])
def test_trace_matches_what_the_reference_prints(case):
    eng = _engine()
    gids = [int(g) for g in TG[case + "_gids"]]
    hp = _gx_hparams(eng, case_hparams(TG, case))
    eo, out, trace, pred, off = _traced_run(eng, gids, hp)
    loss = _printed_loss(hp, trace, off)
    for t, g in enumerate(gids):
        ref = TG["%s_g%d" % (case, g)]
        assert np.abs(loss[t] / ref[:, 0] - 1).max() <= 1e-5, (case, g, loss[t, :3], ref[:3, 0])
        assert np.abs(trace[t, :, _abi.TR_DENSITY] - ref[:, 1]).max() <= 1e-5, (case, g)
        assert np.abs(pred[t] - ref[:, 2:]).max() <= 1e-5, (case, g)
    # the batch order changes nothing: masks and trace bit for bit, the off-edge sums to the order of their double additions
    rev = gids[::-1]
    eo2, out2, trace2, pred2, off2 = _traced_run(eng, rev, hp)
    for t, g in enumerate(gids):
        r = rev.index(g)
        assert np.array_equal(out[eo[t]:eo[t + 1]], out2[eo2[r]:eo2[r + 1]])
        assert np.array_equal(trace[t], trace2[r]) and np.array_equal(pred[t], pred2[r])
        assert np.allclose(off[t], off2[r], rtol=1e-12, atol=0)
    eng.close()


def test_unconstrained_trace_matches_what_the_reference_prints():
    eng = _engine()
    gids = [int(g) for g in TG["c_gids"]]
    E = int(TG["c_epochs"])
    eo = eng.plan_graphs(gids)
    hp = eng.make_hparams(num_epochs=E)
    m0 = np.concatenate([dense_m0(NMAX, int(GG["g%d_seed" % g])).ravel() for g in gids])
    out = np.zeros(int(eo[-1]), np.float32)
    trace = np.zeros((len(gids), E, _abi.GX_TRACE_COLS), np.float32)
    pred = np.zeros((len(gids), E, NC), np.float32)
    eng.explain_graphs_unconstrained(hp, m0, out, trace=trace, trace_pred=pred)
    for t, g in enumerate(gids):
        ref = TG["c_g%d" % g]
        assert np.abs(trace[t, :, _abi.TR_LOSS_EDGES] / ref[:, 0] - 1).max() <= 1e-5, g
        assert np.abs(trace[t, :, _abi.TR_DENSITY] - ref[:, 1]).max() <= 1e-5, g
        assert np.abs(pred[t] - ref[:, 2:]).max() <= 1e-5, g
    eng.close()


# ------------------------------------------------------------------------------------ the drop-in
def _args(tmp_path, **over):
    args = types.SimpleNamespace(num_gc_layers=3, num_epochs=30, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                 mask_bias=False, gpu=False, bias=True, bn=False, method="base", dataset="graphs", bmname=None,
                                 hidden_dim=20, output_dim=20, name_suffix="", explainer_suffix="", logdir=str(tmp_path))
    for k, v in over.items():
        setattr(args, k, v)
    return args


def _explainer(args, print_training=True, bn=False):
    model = gnnx.models.GcnEncoderGraph(14, 20, 20, NC, 3, bn=bn, args=args)
    names = {"W1": "conv_first.weight", "b1": "conv_first.bias", "W2": "conv_block.0.weight", "b2": "conv_block.0.bias",
             "W3": "conv_last.weight", "b3": "conv_last.bias", "Wp": "pred_model.weight", "bp": "pred_model.bias"}
    model.load_state_dict({names[k]: torch.tensor(GG[k]) for k in util.WKEYS})
    return gnnx.Explainer(model=model, adj=torch.tensor(GG["adj"], dtype=torch.float), feat=torch.tensor(GG["feat"]),
                          label=torch.tensor(GG["label"]), pred=GG["pred"], train_idx=[], args=args, writer=None,
                          print_training=print_training, graph_mode=True, graph_idx=0)


def _rows(text):
    """(loss, density, printed softmax row) of every epoch line."""
    return [(float(m.group(2)), float(m.group(3)), np.array([float(x) for x in m.group(4).split(",")])) for m in LINE.finditer(text)]


def _check_rows(rows, ref):
    assert len(rows) == len(ref)
    loss = np.array([r[0] for r in rows]); dens = np.array([r[1] for r in rows])
    assert np.abs(loss / ref[:, 0] - 1).max() <= 1e-5, (loss[:3], ref[:3, 0])
    assert np.abs(dens - ref[:, 1]).max() <= 1e-5
    assert np.abs(np.stack([r[2] for r in rows]) - ref[:, 2:]).max() <= 1e-4     # torch prints the row with 4 decimals


def test_dropin_explain_prints_the_reference_lines(tmp_path, capsys):
    ex = _explainer(_args(tmp_path))
    quiet = _explainer(_args(tmp_path), print_training=False)
    E = int(TG["a_epochs"])
    capsys.readouterr()
    for g in range(NG):
        seed = int(GG["g%d_seed" % g])
        torch.manual_seed(seed)
        masked = ex.explain(node_idx=0, graph_idx=g, graph_mode=True)
        text = capsys.readouterr().out
        assert text.count("finished training in") == 1 and "Saved adjacency matrix to" in text
        _check_rows(_rows(text), TG["a_g%d" % g])
        lt = ex.last_trace
        assert lt["loss"].shape == (1, E) and np.abs(lt["loss"][0] / TG["a_g%d" % g][:, 0] - 1).max() <= 1e-5
        assert np.abs(lt["pred"][0] - TG["a_g%d" % g][:, 2:]).max() <= 1e-5
        torch.manual_seed(seed)
        assert np.array_equal(quiet.explain(node_idx=0, graph_idx=g, graph_mode=True), masked)
    # explain_graphs: one block of E lines per graph, in input order, each the lines of that graph explained alone from the same
    # RNG state (the batch draws the graphs' M0 one after another)
    gids = [5, 0, 9, 2]
    torch.manual_seed(7)
    states = []
    for g in gids:
        states.append(torch.get_rng_state())
        torch.FloatTensor(NMAX, NMAX).normal_()
    after = torch.get_rng_state()
    torch.manual_seed(7)
    masks = ex.explain_graphs(gids)
    assert torch.equal(after, torch.get_rng_state())
    text = capsys.readouterr().out
    rows = _rows(text)
    assert len(rows) == E * len(gids) and text.count("finished training in") == len(gids)
    assert ex.last_trace["loss"].shape == (len(gids), E)
    torch.manual_seed(7)
    assert all(np.array_equal(a, b) for a, b in zip(masks, quiet.explain_graphs(gids)))
    for t, g in enumerate(gids):
        torch.set_rng_state(states[t])
        alone = ex.explain(node_idx=0, graph_idx=g, graph_mode=True)
        assert np.array_equal(alone, masks[t])
        one = _rows(capsys.readouterr().out)
        mine = rows[t * E:(t + 1) * E]
        assert np.allclose([r[0] for r in mine], [r[0] for r in one], rtol=1e-12, atol=0)
        assert [r[1] for r in mine] == [r[1] for r in one]


def test_dropin_other_coefficients(tmp_path, capsys):
    """Case b through the drop-in: the Explainer has no setting for the coefficients (the reference fixes them), the engine's
    hyper-parameters are overridden the way a user would patch ExplainModule.coeffs."""
    ex = _explainer(_args(tmp_path))
    hp_of = ex._hparams

    def patched():
        hp, init = hp_of()
        hp.coef_size, hp.coef_ent, hp.coef_feat_size = float(TG["b_size"]), float(TG["b_ent"]), float(TG["b_feat_size"])
        return hp, init
    ex._hparams = patched
    capsys.readouterr()
    for g in [int(x) for x in TG["b_gids"]]:
        torch.manual_seed(int(GG["g%d_seed" % g]))
        ex.explain_graphs([g], save=False)
        _check_rows(_rows(capsys.readouterr().out), TG["b_g%d" % g])


def test_dropin_unconstrained_prints_the_reference_lines(tmp_path, capsys):
    E = int(TG["c_epochs"])
    ex = _explainer(_args(tmp_path, num_epochs=E))
    quiet = _explainer(_args(tmp_path, num_epochs=E), print_training=False)
    capsys.readouterr()
    for g in [int(x) for x in TG["c_gids"]]:
        torch.manual_seed(int(GG["g%d_seed" % g]))
        masked = ex.explain(node_idx=0, graph_idx=g, graph_mode=True, unconstrained=True)
        text = capsys.readouterr().out
        assert "finished training in" in text and "Saved adjacency matrix to" in text
        _check_rows(_rows(text), TG["c_g%d" % g])
        assert ex.last_trace["loss"].shape == (1, E)
        torch.manual_seed(int(GG["g%d_seed" % g]))
        assert np.array_equal(quiet.explain(node_idx=0, graph_idx=g, graph_mode=True, unconstrained=True), masked)


def test_dropin_device_init_prints_the_edge_loss(tmp_path, capsys):
    ex = _explainer(_args(tmp_path, num_epochs=20, gnnx_init="device", gnnx_seed=3))
    quiet = _explainer(_args(tmp_path, num_epochs=20, gnnx_init="device", gnnx_seed=3), print_training=False)

    def refuse(*a, **k):
        raise AssertionError("the device init has no dense M0 to sum over")
    ex.engine.offedge_regularisers_graphs = refuse
    capsys.readouterr()
    masks = ex.explain_graphs([3, 8])
    rows = _rows(capsys.readouterr().out)
    assert len(rows) == 40
    lt = ex.last_trace
    assert np.array_equal(lt["loss"], lt["terms"][:, :, _abi.TR_LOSS_EDGES].astype(np.float64))
    assert np.allclose([r[0] for r in rows], lt["loss"].ravel(), rtol=1e-12, atol=0)
    assert all(np.array_equal(a, b) for a, b in zip(masks, quiet.explain_graphs([3, 8])))


def test_dropin_variant_keeps_the_notice(tmp_path, capsys):
    ex = _explainer(_args(tmp_path, num_epochs=10, bn=True), bn=True)
    capsys.readouterr()
    torch.manual_seed(1)
    ex.explain(node_idx=0, graph_idx=2, graph_mode=True)
    ex.explain_graphs([1, 4])
    text = capsys.readouterr().out
    assert "per-epoch trace is not built for --bn" in text and not _rows(text) and "finished training in" not in text


def test_dropin_wide_layers_keep_the_notice(tmp_path, capsys):
    """Hidden / output widths above 32 run the variant kernel, which logs no trace: the notice, and the masks of a silent run."""
    args = _args(tmp_path, num_epochs=10, hidden_dim=64, output_dim=64)
    torch.manual_seed(0)
    model = gnnx.models.GcnEncoderGraph(14, 64, 64, NC, 3, bn=False, args=args)
    make = lambda pt: gnnx.Explainer(model=model, adj=torch.tensor(GG["adj"], dtype=torch.float), feat=torch.tensor(GG["feat"]),
                                     label=torch.tensor(GG["label"]), pred=GG["pred"], train_idx=[], args=args, writer=None,
                                     print_training=pt, graph_mode=True, graph_idx=0)
    ex, quiet = make(True), make(False)
    capsys.readouterr()
    torch.manual_seed(3)
    a = ex.explain_graphs([1, 4]) + [ex.explain(node_idx=0, graph_idx=6, graph_mode=True)]
    text = capsys.readouterr().out
    assert "per-epoch trace is not built" in text and "widths above 32" in text and not _rows(text)
    torch.manual_seed(3)
    b = quiet.explain_graphs([1, 4]) + [quiet.explain(node_idx=0, graph_idx=6, graph_mode=True)]
    assert all(np.array_equal(x, y) for x, y in zip(a, b)) and all(np.isfinite(x).all() for x in a)
    # node mode the same
    fx = util.load_fixture("rand")
    d, Cn = fx.feat.shape[1], fx.weights["Wp"].shape[0]
    torch.manual_seed(1)
    node_model = gnnx.models.GcnEncoderNode(d, 64, 48, Cn, 3, bn=False, args=args)
    A = np.zeros((fx.N, fx.N)); A[np.repeat(np.arange(fx.N), np.diff(fx.rowptr)), fx.col] = 1
    make = lambda pt: gnnx.Explainer(model=node_model, adj=A[None], feat=fx.feat[None].astype(np.float64), label=fx.label[None],
                                     pred=fx.pred[None], train_idx=list(range(fx.N)), args=args, writer=None, print_training=pt,
                                     graph_idx=-1)
    ex, quiet = make(True), make(False)
    capsys.readouterr()
    torch.manual_seed(5)
    a = ex.explain(33, graph_idx=0)
    text = capsys.readouterr().out
    assert "widths above 32" in text and not _rows(text)
    torch.manual_seed(5)
    assert np.array_equal(a, quiet.explain(33, graph_idx=0))


def test_dropin_beyond_the_trace_limit(tmp_path, capsys):
    ex = _explainer(_args(tmp_path, num_epochs=1537))
    quiet = _explainer(_args(tmp_path, num_epochs=1537), print_training=False)
    capsys.readouterr()
    torch.manual_seed(2)
    masks = ex.explain_graphs([0, 6])
    text = capsys.readouterr().out
    assert "per-epoch trace is not built for more than 1536 epochs" in text and not _rows(text)
    assert len(masks) == 2 and all(np.isfinite(m).all() for m in masks)
    torch.manual_seed(2)
    assert all(np.array_equal(a, b) for a, b in zip(masks, quiet.explain_graphs([0, 6])))
