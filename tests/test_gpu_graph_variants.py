"""GPU (-m gpu): graph-classification mode with the model and optimiser variants (explain_var.cu in graph mode, through the C ABI and the
drop-in Explainer), against the masks the UNMODIFIED reference returned (tests/golden/graph_variants_golden.npz, 30 epochs) and
against the line-by-line torch port on random models, a graph larger than the tuned kernel's shared memory, and the tuned kernel."""
import os
import types

import numpy as np
import pytest
import torch

import gnnx
import gnnx_oracle as O
import util
from gnnx import _abi
from test_oracle_graph_variants import BASE_KEYS, MODEL_TAGS, OPT_TAGS, dense_m0, model_of

pytestmark = pytest.mark.gpu
OPT_CASES = {"sgd": dict(opt=1), "rmsprop": dict(opt=2), "adagrad": dict(opt=3),
             "sgdstep": dict(opt=1, opt_scheduler=1, opt_decay_step=10, opt_decay_rate=0.3)}
GX_ERR_UNSUPPORTED = -3


@pytest.fixture(scope="module")
def gv():
    return np.load(util.GOLDEN + "/graph_variants_golden.npz")


@pytest.fixture(scope="module")
def gg():
    return np.load(util.GOLDEN + "/graphs_golden.npz")


def _engine(w, L, bn, adj, feat, label):
    eng = gnnx.Engine(0)
    eng.set_model(w, num_layers=L, bn=bn)
    eng.set_graph_batch(adj, feat, label)
    return eng


def _run(eng, gids, m0_of, epochs, with_feat=False, **over):
    edge_off = eng.plan_graphs(gids)
    m0 = np.concatenate([m0_of(g) for g in gids]).astype(np.float32)
    assert len(m0) == edge_off[-1]
    out = np.zeros(len(m0), np.float32)
    fm = np.zeros((len(gids), eng.input_dim), np.float32) if with_feat else None
    eng.explain_graphs_host(eng.make_hparams(num_epochs=epochs, **over), m0, out, fm)
    return (edge_off, out, fm) if with_feat else (edge_off, out)


@pytest.mark.parametrize("tag", MODEL_TAGS + list(OPT_CASES))
def test_graph_variants_match_reference_golden(gv, gg, tag):
    if tag in OPT_CASES:
        w, L, bn, over = {k: gg[k] for k in BASE_KEYS}, 3, False, OPT_CASES[tag]
    else:
        (w, L, bn), over = model_of(gv, tag), {}
    eng = _engine(w, L, bn, gg["adj"], gg["feat"], gg["label"])
    gids = list(range(int(gg["num_graphs"])))
    E = int(gv["num_epochs"])
    edge_off, out, fm = _run(eng, gids, lambda g: gg["g%d_m0" % g], E, with_feat=True, **over)
    eng.close()
    for t, g in enumerate(gids):
        err = util.rel_l2(out[edge_off[t]:edge_off[t + 1]], gv["%s_g%d_mask" % (tag, g)])
        tol = max(1e-4, 3 * float(gv[tag + "_spread"][g]))
        assert err <= tol, (tag, g, err, tol)
        A, M0 = gg["adj"][g].astype(np.float64), dense_m0(gg, g)
        args = (A, gg["feat"][g], int(gg["label"][g]), None, 0, w, M0)
        if tag in OPT_CASES:   # no closed form for these optimisers: the port's feature mask, at 30 x the reference's own spread
            _, ref_fm = O.explain_dense_torch(*args, hp=O.default_hparams(num_epochs=E, **OPT_TAGS[tag]), graph_mode=True, return_feat=True)
            assert np.abs(ref_fm - 0.5).max() > 1e-3
            ferr = np.abs(fm[t] - ref_fm).max()
            assert ferr <= max(2e-4, 30 * float(gv[tag + "_spread"][g])), (tag, g, ferr)
        else:
            util.check_graph_masks(A, gg["feat"][g], gg["label"][g], w, M0, E, None, fm[t], np.nonzero(A), bn=bn)


def _random_model(rng, L, bn, hid, emb, d, C, bias):
    sc = lambda *s: (rng.normal(size=s) * 0.5).astype(np.float32)
    dims = [d] + [hid] * (L - 1) + [emb]
    w = {}
    for l in range(1, L + 1):
        w["W%d" % l] = sc(dims[l - 1], dims[l])
        if bias == "positive":
            w["b%d" % l] = np.abs(sc(dims[l])) + 0.2      # the edge-less rows' constant wins some max-pools
        elif bias == "normal":
            w["b%d" % l] = sc(dims[l])
    w["Wp"] = sc(C, hid * (L - 1) + emb); w["bp"] = sc(C)
    return w


def _check_against_port(eng, w, L, bn, adj, feat, label, gids, epochs, seed):
    n = adj.shape[1]
    dense = {g: O.draw_m0(n, seed=seed + g) for g in gids}
    rc = {g: eng.graph_rows_cols(g) for g in gids}
    fm = np.zeros((len(gids), feat.shape[2]), np.float32)
    edge_off = eng.plan_graphs(gids)
    out = np.zeros(int(edge_off[-1]), np.float32)
    eng.explain_graphs_host(eng.make_hparams(num_epochs=epochs), np.concatenate([dense[g][rc[g]] for g in gids]).astype(np.float32), out, fm)
    for t, g in enumerate(gids):
        util.check_graph_masks(adj[g], feat[g], label[g], w, dense[g], epochs, out[edge_off[t]:edge_off[t + 1]], fm[t], rc[g], bn=bn)


@pytest.mark.parametrize("seed,L,bn,hid,emb,d,C,bias", [(1, 3, True, 64, 48, 14, 3, "positive"), (2, 2, False, 33, 40, 100, 4, "none"),
                                                       (6, 4, True, 128, 128, 128, 5, "positive"), (4, 4, False, 96, 33, 7, 3, "normal"),
                                                       (5, 2, True, 20, 20, 14, 4, "none")])
def test_random_models_match_torch_port(gg, seed, L, bn, hid, emb, d, C, bias):
    rng = np.random.default_rng(seed)
    w = _random_model(rng, L, bn, hid, emb, d, C, bias)
    adj = gg["adj"]
    feat = rng.normal(size=(adj.shape[0], adj.shape[1], d)).astype(np.float32) * (adj.sum(2, keepdims=True) > 0)
    label = gg["label"] % C
    eng = _engine(w, L, bn, adj, feat, label)
    _check_against_port(eng, w, L, bn, adj, feat, label, [0, 3, 5, 9, 11], 20, 300 * seed)
    eng.close()


def test_graph_larger_than_shared_memory(gv):
    """One graph with 1500 active nodes (the tuned kernel refuses it: its state does not fit 226 KB of shared memory) next to a small
    one, a 3-layer --bn model, against the torch port."""
    import networkx as nx
    rng = np.random.default_rng(8)
    n, d = 1520, 14
    adj = np.zeros((2, n, n), np.uint8)
    adj[0, :1500, :1500] = nx.to_numpy_array(nx.barabasi_albert_graph(1500, 2, seed=3))
    adj[1, :30, :30] = nx.to_numpy_array(nx.cycle_graph(30))
    feat = (rng.normal(size=(2, n, d)) * (adj.sum(2, keepdims=True) > 0)).astype(np.float32)
    label = np.array([1, 0])
    w, L, bn = model_of(gv, "bn")
    default = gnnx.Engine(0)
    default.set_model({k: np.asarray(v) for k, v in _random_model(rng, 3, False, 20, 20, d, 2, "normal").items()})
    default.set_graph_batch(adj, feat, label)
    with pytest.raises(_abi.GnnxError) as e:
        default.plan_graphs([0])
    assert e.value.status == GX_ERR_UNSUPPORTED
    default.close()
    eng = _engine(w, L, bn, adj, feat, label)
    _check_against_port(eng, w, L, bn, adj, feat, label, [0, 1], 10, 77)
    eng.close()


def test_order_and_batch_independence(gv, gg):
    w, L, bn = model_of(gv, "bn_L4")
    eng = _engine(w, L, bn, gg["adj"], gg["feat"], gg["label"])
    m0_of = lambda g: gg["g%d_m0" % g]
    gids = list(range(int(gg["num_graphs"])))
    eo, out = _run(eng, gids, m0_of, 30)
    for sub in ([7, 2, 11], [11, 10, 9, 8, 7, 6, 5, 4, 3, 2, 1, 0], [3]):
        so, o2 = _run(eng, sub, m0_of, 30)
        for t, g in enumerate(sub):
            assert np.array_equal(o2[so[t]:so[t + 1]], out[eo[g]:eo[g + 1]]), (sub, g)
    eng.close()


def test_philox_init_equals_the_tuned_kernel(gg):
    """GX_INIT_PHILOX in both graph kernels draws the M0 of its host restatement (gnnx_oracle.philox_m0: key = graph id, slot = position
    in the graph's CSR, std sqrt(2 / max_nodes)): at num_epochs = 1 (the mask before any update) an SGD run (variant kernel) and an Adam
    run (tuned kernel) both return (sigmoid(M0_ij) + sigmoid(M0_ji)) / 2."""
    eng = _engine({k: gg[k] for k in BASE_KEYS}, 3, False, gg["adj"], gg["feat"], gg["label"])
    gids = list(range(int(gg["num_graphs"])))
    edge_off = eng.plan_graphs(gids)
    n, seed = int(gg["max_nodes"]), 1234 + (3 << 32)      # the seed's high word keys the generator too
    want = []
    for t, g in enumerate(gids):
        r, c = eng.graph_rows_cols(g)
        S = np.full((n, n), np.nan)
        S[r, c] = 1 / (1 + np.exp(-O.philox_m0(seed, g, len(r), n)))
        want.append((S[r, c] + S[c, r]) / 2)
    want = np.concatenate(want)
    res = []
    for opt in (0, 1):
        out = np.zeros(int(edge_off[-1]), np.float32)
        eng.explain_graphs_host(eng.make_hparams(num_epochs=1, init=_abi.GX_INIT_PHILOX, seed=seed, opt=opt), None, out)
        res.append(out)
    eng.close()
    assert np.abs(res[0] - res[1]).max() <= 1e-6
    assert np.abs(res[0] - want).max() <= 1e-6 and np.abs(res[1] - want).max() <= 1e-6
    assert np.isfinite(res[0]).all() and 0.3 < res[0].mean() < 0.95


def test_variant_path_refuses_trace_and_state(gv, gg):
    w, L, bn = model_of(gv, "bn")
    eng = _engine(w, L, bn, gg["adj"], gg["feat"], gg["label"])
    edge_off = eng.plan_graphs([0, 1])
    te = int(edge_off[-1])
    m0 = np.concatenate([gg["g0_m0"], gg["g1_m0"]]).astype(np.float32)
    out = np.zeros(te, np.float32)
    hp = eng.make_hparams(num_epochs=3)
    calls = [dict(trace=np.zeros((2, 3, _abi.GX_TRACE_COLS), np.float32)),
             dict(state_out=dict(M=np.zeros(te, np.float32), m=np.zeros(te, np.float32), v=np.zeros(te, np.float32)))]
    for kw in calls:
        with pytest.raises(_abi.GnnxError) as e:
            eng.explain_nodes_ex(hp, m0, out, graphs=True, **kw)
        assert e.value.status == GX_ERR_UNSUPPORTED
    with pytest.raises(_abi.GnnxError) as e:
        eng.explain_nodes_ex(eng.make_hparams(num_epochs=3, init=_abi.GX_INIT_STATE, start_step=2), m0, out, graphs=True,
                             state_in=dict(m=np.zeros(te, np.float32), v=np.zeros(te, np.float32)))
    assert e.value.status == GX_ERR_UNSUPPORTED
    eng.explain_nodes_ex(hp, m0, out, graphs=True)        # edge_mask / feat_mask only: fine
    assert np.isfinite(out).all()
    eng.close()


def test_explainer_dropin_bn_4_layers(gv, gg, tmp_path, capsys):
    args = types.SimpleNamespace(num_gc_layers=4, num_epochs=int(gv["num_epochs"]), lr=0.1, opt="adam", opt_scheduler="none",
                                 mask_act="sigmoid", mask_bias=False, gpu=False, bias=True, bn=True, method="base", dataset="graphs",
                                 bmname=None, hidden_dim=20, output_dim=20, name_suffix="", explainer_suffix="", logdir=str(tmp_path))
    d, C = gg["feat"].shape[2], gg["Wp"].shape[0]
    model = gnnx.models.GcnEncoderGraph(d, 20, 20, C, 4, bn=True, args=args)
    keys = ["conv_first", "conv_block.0", "conv_block.1", "conv_last"]
    sd = {}
    for l, k in enumerate(keys, 1):
        sd[k + ".weight"] = gv["bn_L4_W%d" % l]; sd[k + ".bias"] = gv["bn_L4_b%d" % l]
    sd["pred_model.weight"] = gv["bn_L4_Wp"]; sd["pred_model.bias"] = gv["bn_L4_bp"]
    model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    ex = gnnx.Explainer(model=model, adj=torch.tensor(gg["adj"], dtype=torch.float), feat=torch.tensor(gg["feat"]),
                        label=torch.tensor(gg["label"]), pred=None, train_idx=[], args=args, writer=None,
                        print_training=True, graph_mode=True, graph_idx=0)
    n = int(gg["max_nodes"])
    for g in (1, 3, 8):
        torch.manual_seed(int(gg["g%d_seed" % g]))
        masked = ex.explain(node_idx=0, graph_idx=g, graph_mode=True)
        assert masked.shape == (n, n) and masked.dtype == np.float64
        ei, ej = np.nonzero(gg["adj"][g])
        tol = max(1e-4, 3 * float(gv["bn_L4_spread"][g]))
        assert util.rel_l2(masked[ei, ej], gv["bn_L4_g%d_mask" % g]) <= tol
        off = masked.copy(); off[ei, ej] = 0
        assert np.all(off == 0)
    printed = capsys.readouterr().out
    assert "trace is not built" in printed and "Saved adjacency matrix to" in printed
    assert any(f.startswith("masked_adj_") and f.endswith(".npy") for f in os.listdir(tmp_path))
    torch.manual_seed(1)
    a = [ex.explain(0, graph_idx=g, graph_mode=True) for g in (4, 6)]
    torch.manual_seed(1)
    b = ex.explain_graphs([4, 6])
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
