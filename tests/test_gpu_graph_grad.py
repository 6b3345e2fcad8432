"""GPU (-m gpu): the gradient baseline in graph-classification mode (gx_grad_graphs, explain_graph.cu's mode 1; the drop-in's
explain(..., graph_mode=True, model="grad"), explain_graphs(model="grad") and gnnx.dist.explain_graphs_sharded(model="grad")).

Every mask is judged per graph at 1e-5, relative L2 and max abs, against the fp64 specification (tests/graph_grad_oracle.py) and, on the
golden graphs, against the unmodified reference's adj_feat_grad (graph_grad_golden.npz).  A max-pool column whose best two rows lie within
2 fp32 ulps is a near tie: there the mask may follow either routing, judged as tests/test_gpu_pool_ties.py does with
tests/pool_oracle.py's flips."""
import os
import socket
import types

import numpy as np
import pytest
import torch

import gnnx
from gnnx import _abi
import gnnx_oracle as O
import graph_grad_oracle as GO
import pool_oracle as PO
import util
from test_gpu_graph_shapes import (CLASS_SIZES, FAMILY, MAXN_C, _accepted, _active, _ba, _batch, _bench_module, _classes_run,
                                   _tree)
from test_gpu_graph_variants import GX_ERR_UNSUPPORTED, _random_model

pytestmark = pytest.mark.gpu
TOL = 1e-5
GX_ERR_INVALID = -1
WKEYS = ("W1", "b1", "W2", "b2", "W3", "b3", "Wp", "bp")


def _grad_pool(A, X, lab, w, dtype, flips=None):
    """The port with pool_oracle's readout: (mask, record of the one forward's arg-max choices)."""
    pool = PO._Pool(flips, True, 2)
    prev = O.set_pool(pool)
    try:
        m = GO.grad_graph_torch(A, X, lab, w, dtype=dtype)
    finally:
        O.set_pool(prev)
    return m, pool.rec


def _errs(got, want):
    return O.rel_l2(got, want), float(np.abs(np.asarray(got, np.float64) - want).max(initial=0.0))


def check(got, A, X, lab, w, rc, ref=None):
    """got (the graph's slots) within TOL of the fp64 specification (and of `ref`, the reference's mask), or -- where the forward has a
    max-pool near tie -- of the fp32 port with that column's arg-max on the other row."""
    A = np.asarray(A, np.float64)
    spec = GO.grad_graph_closed_form(A, X, lab, w)[rc]
    e = _errs(got, spec)
    if ref is not None:
        e = max(e, _errs(got, ref))
    if max(e) <= TOL:
        return
    _, r64 = _grad_pool(A, X, lab, w, np.float64)
    _, r32 = _grad_pool(A, X, lab, w, np.float32)
    alts = []
    for _, l, c, win, run, _ in PO.near_ties(r64):
        row = run if int(r32[0][l][0][c]) == win else win
        alts.append(max(_errs(got, _grad_pool(A, X, lab, w, np.float32, flips={0: [(l, c, row)]})[0][rc])))
    assert alts and min(alts) <= TOL, ("no admissible routing within %g" % TOL, e, alts)


def _labels_of(adj, feat, w, gids):
    """The model's own prediction per graph (fp64 forward): what pred_label = -1 resolves to unless the logits nearly tie."""
    return np.asarray([GO.grad_graph_torch(adj[g], feat[g], -1, w, dtype=np.float64, return_label=True)[1] for g in gids], np.int32)


def _run(eng, gids, labels):
    eo = eng.plan_graphs(gids)
    out = np.zeros(max(int(eo[-1]), 1), np.float32)
    eng.grad_graphs_host(np.asarray(labels, np.int32), out)
    return eo, out


# ------------------------------------------------------------------------------------------------ golden graphs, both models
@pytest.mark.parametrize("model", ["base", "scaled"])
def test_golden_graphs_match_reference(model):
    gold = np.load(util.GOLDEN + "/graph_grad_golden.npz")
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    w = {k: gold["%s_w_%s" % (model, k)].astype(np.float32) for k in WKEYS}
    eng = gnnx.Engine(0)
    eng.set_model(w)
    eng.set_graph_batch(gg["adj"], gg["feat"], gg["label"])
    G = int(gg["num_graphs"])
    gids = list(range(G))
    for key in ("", "alt_"):
        labels = [int(gold["%s_g%d_%slabel" % (model, g, key)]) for g in gids]
        eo, out = _run(eng, gids, labels)
        for t, g in enumerate(gids):
            rc = eng.graph_rows_cols(g)
            check(out[eo[t]:eo[t + 1]], gg["adj"][g], gg["feat"][g], labels[t], w, rc, ref=gold["%s_g%d_%smask" % (model, g, key)])
        if key == "":
            # pred_label = -1: the kernel's own arg-max of the same logits is the golden (predicted) label -> the same bits
            eo1, out1 = _run(eng, gids, [-1] * G)
            assert np.array_equal(out1, out)
    eng.close()


# ------------------------------------------------------------------------------------------------ every footprint class
@pytest.fixture(scope="module")
def class_engine():
    rng = np.random.default_rng(3)
    sizes = CLASS_SIZES + FAMILY
    adj = _batch([_ba(s) for s in sizes], MAXN_C)
    feat = rng.normal(size=(len(sizes), MAXN_C, 14)).astype(np.float32)
    w = _random_model(rng, 3, False, 20, 20, 14, 3, "normal")
    w["Wp"] = w["Wp"] * 8     # a readout with a gradient well away from 0 (the layers normalise, so only pred_model sets its scale)
    eng = gnnx.Engine(0)
    eng.set_model(w)
    eng.set_graph_batch(adj, feat, rng.integers(0, 3, len(sizes)))
    b = types.SimpleNamespace(eng=eng, adj=adj, feat=feat, w=w, gid={s: g for g, s in enumerate(sizes)})
    yield b
    eng.close()


def test_every_launch_class_alone_and_together(class_engine):
    b = class_engine
    lo, hi = b.gid[FAMILY[0]], b.gid[FAMILY[-1]]
    assert _accepted(b, lo) and not _accepted(b, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if _accepted(b, mid) else (lo, mid)
    gids = [b.gid[s] for s in CLASS_SIZES] + [lo]                  # lo: the largest graph the tuned kernel accepts
    assert _active(b.adj[b.gid[300]]) > 256
    labels = np.array([0, 1, 2, -1, 1, 0, 2], np.int32)
    eo, out = _run(b.eng, gids, labels)
    ran = []
    for t, g in enumerate(gids):
        eo1, o1 = _run(b.eng, [g], labels[t:t + 1])
        r = _classes_run(b.eng)
        assert len(r) == 1
        ran.append(r[0])
        assert np.array_equal(o1[:eo1[-1]], out[eo[t]:eo[t + 1]]), g        # alone == in the mixed batch
    assert ran == [0, 1, 2, 3, 4, 5, 5], ran
    own = _labels_of(b.adj, b.feat, b.w, gids)
    for t, g in enumerate(gids):
        lab = int(labels[t]) if labels[t] >= 0 else int(own[t])
        check(out[eo[t]:eo[t + 1]], b.adj[g], b.feat[g], lab, b.w, b.eng.graph_rows_cols(g))
    # batch order: the reversed list gives the same bits per graph
    eo2, out2 = _run(b.eng, gids[::-1], labels[::-1])
    for t, g in enumerate(gids[::-1]):
        assert np.array_equal(out2[eo2[t]:eo2[t + 1]], out[eo[len(gids) - 1 - t]:eo[len(gids) - t]]), g
    # -1 == the explicit arg-max, bit for bit
    eo3, out3 = _run(b.eng, gids, own)
    eo4, out4 = _run(b.eng, gids, np.full(len(gids), -1, np.int32))
    assert np.array_equal(out3, out4)


# ------------------------------------------------------------------------------------------------ structure: padding, isolated rows, no edge
def test_structure_edge_cases():
    rng = np.random.default_rng(31)
    n, d, C = 48, 14, 3
    w = _random_model(rng, 3, False, 20, 20, d, C, "positive")
    w["Wp"] = w["Wp"] * 8
    star = np.zeros((6, 6), np.uint8)
    star[0, 1:] = star[1:, 0] = 1
    parts = [_tree(rng, n, 12),            # 0: every row active: no padding row, no edge-less constant in the pools
             (6, _tree(rng, 34, 6)),       # 1: rows 0..5 isolated, below the active rows
             star,                         # 2: a star, padded
             np.zeros((n, n), np.uint8),   # 3: no edge at all
             (20, _tree(rng, 25, 4))]      # 4: padding on both sides
    adj = _batch(parts, n)
    feat = rng.normal(size=(len(parts), n, d)).astype(np.float32)
    eng = gnnx.Engine(0)
    eng.set_model(w)
    eng.set_graph_batch(adj, feat, rng.integers(0, C, len(parts)))
    gids = [0, 1, 2, 3, 4]
    own = _labels_of(adj, feat, w, gids)
    eo, out = _run(eng, gids, own)
    assert eo[4] == eo[3]                                          # graph 3 has no edge slot
    for t, g in enumerate(gids):
        check(out[eo[t]:eo[t + 1]], adj[g], feat[g], int(own[t]), w, eng.graph_rows_cols(g))
    eo1, out1 = _run(eng, gids, np.full(len(gids), -1, np.int32))
    assert np.array_equal(out1, out)
    alt = (own + 1) % C
    eo2, out2 = _run(eng, gids, alt)
    for t, g in enumerate(gids):
        check(out2[eo2[t]:eo2[t + 1]], adj[g], feat[g], int(alt[t]), w, eng.graph_rows_cols(g))
    sub = [4, 2, 0, 1]                                             # batch composition and order: the edge-less graph changes nothing
    eo3, out3 = _run(eng, sub, own[sub])
    for t3, g in enumerate(sub):
        assert np.array_equal(out3[eo3[t3]:eo3[t3 + 1]], out[eo[g]:eo[g + 1]]), g
    # labels outside [-1, C) and a label list of the wrong length are refused
    eng.plan_graphs(gids)
    buf = np.zeros(max(int(eo[-1]), 1), np.float32)
    for bad in (C, -2):
        with pytest.raises(_abi.GnnxError) as e:
            eng.grad_graphs_host(np.array([0, 0, bad, 0, 0], np.int32), buf)
        assert e.value.status == GX_ERR_INVALID
    with pytest.raises(ValueError):
        eng.grad_graphs_host(np.zeros(4, np.int32), buf)
    eng.close()


# ------------------------------------------------------------------------------------------------ more graphs than resident CTAs
def test_benchmarked_batch_past_the_resident_grid():
    """bench.py --workload graphs (4337 graphs, max_nodes 100): some launch class holds more graphs than it has resident CTAs
    (tests/test_gpu_graph_shapes.py asserts that for this batch), so CTAs take further graphs from the queue.  Graphs of every class
    against the specification; a shuffled sub-batch, and the device-memory entry, give the same bits."""
    bench = _bench_module()
    adj, feat, label, W = bench.make_graph_batch()
    G, n = adj.shape[:2]
    eng = gnnx.Engine(0)
    eng.set_model(W)
    eng.set_graph_batch(adj, feat, label)
    gids = list(range(G))
    labels = np.full(G, -1, np.int32)
    eo, out = _run(eng, gids, labels)
    cls = {}
    for g in range(0, G, 97):
        _run(eng, [g], labels[:1])
        cls.setdefault(_classes_run(eng)[0], []).append(g)
    assert sorted(cls) == [0, 1, 2, 3, 4], sorted(cls)
    picks = sorted({g for v in cls.values() for g in v[:2]} | {1279})
    own = _labels_of(adj, feat, W, picks)
    for g, lab in zip(picks, own):
        check(out[eo[g]:eo[g + 1]], adj[g], feat[g], int(lab), W, eng.graph_rows_cols(g))
    sub = np.random.default_rng(0).permutation(G)[:2500].tolist()
    eo2, out2 = _run(eng, sub, labels[:len(sub)])
    for t, g in enumerate(sub):
        assert np.array_equal(out2[eo2[t]:eo2[t + 1]], out[eo[g]:eo[g + 1]]), g
    eng.plan_graphs(gids)
    dev = eng.grad_graphs_device(labels)
    torch.cuda.synchronize()
    assert np.array_equal(dev.cpu().numpy(), out[:int(eo[-1])])
    eng.close()


# ------------------------------------------------------------------------------------------------ the drop-in
def _args(tmp_path, **over):
    a = dict(num_gc_layers=3, num_epochs=20, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid", mask_bias=False, gpu=False,
             bias=True, method="base", dataset="graphs", bmname=None, hidden_dim=20, output_dim=20, name_suffix="", explainer_suffix="",
             logdir=str(tmp_path))
    a.update(over)
    return types.SimpleNamespace(**a)


def _explainer(gg, args, pred, bn=False, L=3):
    model = gnnx.models.GcnEncoderGraph(14, 20, 20, 2, L, bn=bn, args=args)
    if not bn and L == 3:
        sd = {"conv_first.weight": gg["W1"], "conv_first.bias": gg["b1"], "conv_block.0.weight": gg["W2"], "conv_block.0.bias": gg["b2"],
              "conv_last.weight": gg["W3"], "conv_last.bias": gg["b3"], "pred_model.weight": gg["Wp"], "pred_model.bias": gg["bp"]}
        model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    return gnnx.Explainer(model=model, adj=torch.tensor(gg["adj"], dtype=torch.float), feat=torch.tensor(gg["feat"]),
                          label=torch.tensor(gg["label"]), pred=pred, train_idx=[], args=args, writer=None, print_training=False,
                          graph_mode=True, graph_idx=0)


def _normals_after(seed, n, count):
    torch.manual_seed(seed)
    for _ in range(count):
        O.draw_m0(n)
    return torch.get_rng_state()


@pytest.mark.parametrize("with_pred", [True, False])
def test_dropin_explain_and_explain_graphs(tmp_path, with_pred):
    gold = np.load(util.GOLDEN + "/graph_grad_golden.npz")
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    n = int(gg["max_nodes"])
    ex = _explainer(gg, _args(tmp_path), gg["pred"] if with_pred else None)
    gids = [3, 0, 8, 11]
    singles = []
    for g in gids:
        torch.manual_seed(5)
        masked = ex.explain(0, graph_idx=g, graph_mode=True, model="grad")
        assert torch.equal(torch.get_rng_state(), _normals_after(5, n, 1))      # one ExplainModule's n^2 normals (explain.py:645-652)
        assert masked.shape == (n, n) and masked.dtype == np.float64
        rc = ex.engine.graph_rows_cols(g)
        off = masked.copy(); off[rc] = 0
        assert not off.any()
        # the plan result densified
        eo = ex.engine.plan_graphs([g])
        packed = np.zeros(max(int(eo[-1]), 1), np.float32)
        ex.engine.grad_graphs_host([int(gold["base_g%d_label" % g])], packed)
        assert np.array_equal(masked[rc], packed[:int(eo[-1])].astype(np.float64))
        check(masked[rc], gg["adj"][g], gg["feat"][g], int(gold["base_g%d_label" % g]), {k: gg[k] for k in WKEYS}, rc,
              ref=gold["base_g%d_mask" % g])
        singles.append(masked)
    files = os.listdir(tmp_path)
    assert any(f.startswith("masked_adj_") and f.endswith(".npy") for f in files), files
    saved = np.load(os.path.join(tmp_path, [f for f in files if f.startswith("masked_adj_")][0]))
    assert np.array_equal(saved, singles[-1])
    torch.manual_seed(5)
    many = ex.explain_graphs(gids, save=False, model="grad")
    assert torch.equal(torch.get_rng_state(), _normals_after(5, n, len(gids)))
    assert all(np.array_equal(a, b) for a, b in zip(many, singles))
    # the device init draws nothing on the host
    exd = _explainer(gg, _args(tmp_path, gnnx_init="device"), None)
    torch.manual_seed(5)
    state = torch.get_rng_state()
    assert all(np.array_equal(a, b) for a, b in zip(exd.explain_graphs(gids, save=False, model="grad"), singles))
    assert torch.equal(torch.get_rng_state(), state)
    ex.engine.close()
    exd.engine.close()


def test_variants_are_refused_before_any_rng(tmp_path):
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    for bn, L in ((True, 3), (False, 4)):
        ex = _explainer(gg, _args(tmp_path, num_gc_layers=L, bn=bn), None, bn=bn, L=L)
        ex.engine.plan_graphs([0, 1])
        with pytest.raises(_abi.GnnxError) as e:
            ex.engine.grad_graphs_host([0, 1], np.zeros(256, np.float32))
        assert e.value.status == GX_ERR_UNSUPPORTED and "gradient baseline" in str(e.value)
        torch.manual_seed(9)
        state = torch.get_rng_state()
        with pytest.raises(NotImplementedError):
            ex.explain(0, graph_idx=1, graph_mode=True, model="grad")
        with pytest.raises(NotImplementedError):
            ex.explain_graphs([0, 1], model="grad")
        assert torch.equal(torch.get_rng_state(), state)
        ex.engine.close()


# ------------------------------------------------------------------------------------------------ sharded
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def test_explain_graphs_sharded_grad_one_rank(tmp_path):
    import torch.distributed as dist
    from gnnx.dist import explain_graphs_sharded
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    gids = [4, 1, 9, 1, 0, 11, 6]
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % _free_port(), rank=0, world_size=1)
    try:
        ex = _explainer(gg, _args(tmp_path), gg["pred"])
        torch.manual_seed(21)
        want = ex.explain_graphs(gids, save=False, model="grad")
        rng_after = torch.get_rng_state()
        for use_engine_comm in (False, True):
            torch.manual_seed(21)
            values, offsets, _, dense = explain_graphs_sharded(ex, gids, dense=True, model="grad", use_engine_comm=use_engine_comm)
            torch.cuda.synchronize()
            assert torch.equal(torch.get_rng_state(), rng_after)
            assert np.array_equal(dense.cpu().numpy(), np.stack(want))
            packed = np.concatenate([D[ex.engine.graph_rows_cols(g)] for D, g in zip(want, gids)]).astype(np.float32)
            assert np.array_equal(values.cpu().numpy(), packed)
        ex.engine.close()
    finally:
        dist.destroy_process_group()


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import conftest  # noqa: F401
    import torch.distributed as dist
    import util
    import gnnx
    from gnnx.dist import explain_graphs_sharded
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    gg = np.load(util.GOLDEN + "/graphs_golden.npz")
    args = _args("/tmp/gnnx_dist_graph_grad_%d" % rank)
    model = gnnx.models.GcnEncoderGraph(14, 20, 20, 2, 3, bn=False, args=args)
    sd = {"conv_first.weight": gg["W1"], "conv_first.bias": gg["b1"], "conv_block.0.weight": gg["W2"], "conv_block.0.bias": gg["b2"],
          "conv_last.weight": gg["W3"], "conv_last.bias": gg["b3"], "pred_model.weight": gg["Wp"], "pred_model.bias": gg["bp"]}
    model.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    ex = gnnx.Explainer(model=model, adj=torch.tensor(gg["adj"], dtype=torch.float), feat=torch.tensor(gg["feat"]),
                        label=torch.tensor(gg["label"]), pred=gg["pred"], train_idx=[], args=args, writer=None, print_training=False,
                        graph_mode=True, graph_idx=0, device=rank)
    gids = [5, 0, 11, 3, 3, 8, 1, 10, 2, 9, 7]
    torch.manual_seed(8)
    _, _, (_, pos), dense = explain_graphs_sharded(ex, gids, dense=True, model="grad")
    if rank == 0:
        torch.manual_seed(8)
        full = ex.explain_graphs(gids, save=False, model="grad")
        q.put((dense.cpu().numpy(), np.stack(full), len(pos)))
    dist.barrier()
    ex.engine.close()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_explain_graphs_sharded_grad_two_ranks():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    try:
        dense, full, owned = q.get(timeout=300)
    finally:
        for p in procs:
            p.join(120)
            if p.is_alive():
                p.terminate()
                p.join(10)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    assert 0 < owned < 11
    assert np.array_equal(dense, full)
