"""GPU (-m gpu): the narrow instantiation of the shared-memory node kernel (explain_node.cu, kNarrow).  Inputs no wider than the
hidden width (4 * ceil(d / 4) <= HID == EMB) run with the lane-group shape fixed at compile time; the arithmetic and its order are
those of the run-time-shape code, so every output must be the same bits as with GNNX_NODE_GENERIC=1:

  * syn1 (all 700 nodes) and syn4 (all 871) with Philox init: masks, feature masks, trace rows and optimiser-state outputs;
  * random graphs with d in {1, 3, 10, 17, 20} at widths 20 / 20, and d in {20, 32} at widths 24 / 28 (zero-padded to 32 / 32);
  * every shared-memory launch class, each asserting the instantiation and thread count it reached (debug dump);
  * the gradient baseline (model="grad");
  * d = 21 at widths 20 / 20 stays on the run-time-shape code;
  * the per-node reference goldens at their tolerances, and the same bits in reversed batch order."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import gnnx
from gnnx import _abi
import gnnx_oracle as O
import util

pytestmark = pytest.mark.gpu

SMEM = 5   # launch classes 0..4 of gx_plan_class_counts: the shared-memory kernel
THREADS = [128, 256, 256, 512, 512]   # threads per CTA of classes 0..4 (host.cuh, kNodeClasses)
DUMP = 1 << 19


def _engine(weights, rowptr, col, feat, label, pred_label, generic):
    old = os.environ.get("GNNX_NODE_GENERIC")
    os.environ["GNNX_NODE_GENERIC"] = "1" if generic else "0"
    try:
        eng = gnnx.Engine(0)
    finally:
        if old is None:
            del os.environ["GNNX_NODE_GENERIC"]
        else:
            os.environ["GNNX_NODE_GENERIC"] = old
    eng.set_model(weights)
    eng.set_graph_csr(rowptr, col, feat, label, pred_label)
    return eng


def _pair(g):
    """(narrow-enabled engine, generic engine) on the same graph and model"""
    return [_engine(g.weights, g.rowptr, g.col, g.feat, g.label, g.pred_label, generic) for generic in (False, True)]


def _rand_graph(d, hid, emb, seed, N=240, C=4):
    rng = np.random.default_rng(seed)
    edges = set()
    for i in range(1, N):   # preferential-attachment-like: a few hubs, many short rows
        for j in rng.integers(0, i, size=min(i, 2)):
            edges.add((int(j), i))
    for _ in range(N // 3):
        i, j = rng.integers(0, N, size=2)
        if i != j:
            edges.add((int(min(i, j)), int(max(i, j))))
    edges = np.array(sorted(edges), np.int64)
    rowptr, col = O.csr_from_edges(N, edges)
    f = lambda *s: (rng.standard_normal(s) * 0.4).astype(np.float32)
    w = {"W1": f(d, hid), "b1": f(hid), "W2": f(hid, hid), "b2": f(hid), "W3": f(hid, emb), "b3": f(emb),
         "Wp": f(C, 2 * hid + emb), "bp": f(C)}
    label = rng.integers(0, C, size=N).astype(np.int32)
    return type("G", (), dict(weights=w, rowptr=rowptr, col=col, feat=f(N, d), label=label,
                             pred_label=rng.integers(0, C, size=N).astype(np.int32), N=N, d=d))


def _fixture(name):
    fx = util.load_fixture(name)
    fx.d = fx.feat.shape[1]
    return fx


def _outputs(eng, nodes, hp, d, C, m0=None):
    """masks, feature masks, trace rows and optimiser-state outputs of one batch, plus its launch-class counts"""
    plan = eng.plan_nodes(nodes, 3)
    cnt = len(plan.nodes)
    o = dict(mask=np.zeros(plan.total_edges, np.float32), feat=np.zeros((cnt, d), np.float32),
             trace=np.zeros((cnt, hp.num_epochs, 8), np.float32), trace_pred=np.zeros((cnt, hp.num_epochs, C), np.float32))
    so = dict(M=np.zeros(plan.total_edges, np.float32), m=np.zeros(plan.total_edges, np.float32),
              v=np.zeros(plan.total_edges, np.float32), feat=np.zeros((cnt, 3, d), np.float32))
    eng.explain_nodes_ex(hp, m0(plan) if m0 else None, o["mask"], o["feat"], trace=o["trace"], trace_pred=o["trace_pred"], state_out=so)
    o.update({"state_" + k: v for k, v in so.items()})
    # and the production path (no trace / state buffers: the other instantiation)
    o["mask_plain"] = np.zeros(plan.total_edges, np.float32)
    o["feat_plain"] = np.zeros((cnt, d), np.float32)
    eng.explain_nodes_host(hp, m0(plan) if m0 else None, o["mask_plain"], o["feat_plain"])
    return o, eng.plan_class_counts()[0], plan


def _assert_same(a, b, what):
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), (what, k)


def _which(eng, node, hp):
    """(1 if the narrow instantiation ran else 0, threads of the CTA) for a batch of one node, from the kernel's debug dump"""
    dbg = torch.zeros(DUMP + 64 + 16, dtype=torch.float32, device="cuda")   # + the timeline record of task 0
    lib = _abi.lib()
    lib.gx_debug_set_dump.argtypes = [C.c_void_p, C.c_void_p]
    lib.gx_debug_set_dump(eng._h, C.c_void_p(dbg.data_ptr()))
    try:
        plan = eng.plan_nodes([node], 3)
        eng.explain_nodes_host(hp, None, np.zeros(plan.total_edges, np.float32))
    finally:
        lib.gx_debug_set_dump(eng._h, None)
    o = dbg[DUMP:DUMP + 13].cpu().numpy()
    return int(o[12]), int(o[11])


def _class_of(eng, node):
    eng.plan_nodes([node], 3)
    return int(np.argmax(eng.plan_class_counts()[0]))


HP = dict(num_epochs=100, init=_abi.GX_INIT_PHILOX, seed=5)


@pytest.mark.parametrize("name", ["syn1", "syn4"])
def test_fixture_batch_is_bit_identical(name):
    fx = _fixture(name)
    nar, gen = _pair(fx)
    nodes = list(range(fx.N))
    hp = nar.make_hparams(**HP)
    a, ca, _ = _outputs(nar, nodes, hp, fx.d, fx.weights["Wp"].shape[0])
    b, cb, _ = _outputs(gen, nodes, gen.make_hparams(**HP), fx.d, fx.weights["Wp"].shape[0])
    assert np.array_equal(ca, cb) and ca[SMEM:].sum() == 0, (ca, cb)
    if name == "syn1":
        assert (ca[:SMEM] > 0).all(), ca
    _assert_same(a, b, name)
    nar.close(); gen.close()


def test_every_class_reaches_the_narrow_instantiation():
    seen = {}
    for name in ("rand", "syn4", "syn1"):
        fx = _fixture(name)
        nar, gen = _pair(fx)
        hp = nar.make_hparams(num_epochs=3, init=_abi.GX_INIT_PHILOX, seed=1)
        for v in fx.nodes:
            c = _class_of(nar, v)
            if c in seen:
                continue
            kn, tn = _which(nar, v, hp)
            kg, tg = _which(gen, v, hp)
            assert (kn, kg) == (1, 0) and tn == tg == THREADS[c], (name, v, c, kn, kg, tn, tg)
            seen[c] = v
        nar.close(); gen.close()
    assert sorted(seen) == list(range(SMEM)), seen


@pytest.mark.parametrize("d,hid,emb", [(1, 20, 20), (3, 20, 20), (10, 20, 20), (17, 20, 20), (20, 20, 20), (20, 24, 28), (32, 24, 28)])
def test_random_widths_are_bit_identical(d, hid, emb):
    g = _rand_graph(d, hid, emb, seed=100 + d + hid)
    nar, gen = _pair(g)
    nodes = list(range(0, g.N, 3))
    a, ca, plan = _outputs(nar, nodes, nar.make_hparams(**HP), d, 4)
    b, cb, _ = _outputs(gen, nodes, gen.make_hparams(**HP), d, 4)
    assert np.array_equal(ca, cb) and ca[SMEM:].sum() == 0, (ca, cb)
    _assert_same(a, b, (d, hid, emb))
    hp = nar.make_hparams(num_epochs=2, init=_abi.GX_INIT_PHILOX, seed=1)
    assert _which(nar, nodes[0], hp)[0] == 1 and _which(gen, nodes[0], hp)[0] == 0
    nar.close(); gen.close()


def test_wider_input_takes_the_generic_code():
    g = _rand_graph(21, 20, 20, seed=7)
    nar, gen = _pair(g)
    hp = nar.make_hparams(num_epochs=2, init=_abi.GX_INIT_PHILOX, seed=1)
    assert _which(nar, 0, hp)[0] == 0 and _which(gen, 0, hp)[0] == 0
    nodes = list(range(0, g.N, 5))
    a, _, _ = _outputs(nar, nodes, nar.make_hparams(**HP), 21, 4)
    b, _, _ = _outputs(gen, nodes, gen.make_hparams(**HP), 21, 4)
    _assert_same(a, b, "d=21")
    nar.close(); gen.close()


@pytest.mark.parametrize("name", ["syn1", "rand"])
def test_gradient_baseline_is_bit_identical(name):
    fx = _fixture(name)
    nar, gen = _pair(fx)
    outs = []
    for eng in (nar, gen):
        plan = eng.plan_nodes(list(range(fx.N)) if name == "syn1" else fx.nodes, 3)
        out = np.zeros(plan.total_edges, np.float32)
        eng.grad_nodes_host(out)
        outs.append(out)
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32))
    nar.close(); gen.close()


@pytest.mark.parametrize("name", ["syn1", "syn4", "rand"])
def test_goldens_and_batch_order(name):
    fx = _fixture(name)
    eng = util.make_engine(fx)
    assert _which(eng, fx.nodes[0], eng.make_hparams(num_epochs=2, init=_abi.GX_INIT_PHILOX, seed=1))[0] == 1
    tol = util.node_tolerances(name, 100)
    m0 = lambda plan: util.golden_m0(fx, plan)
    res = []
    for order in (fx.nodes, fx.nodes[::-1]):
        plan = eng.plan_nodes(order, 3)
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_host(eng.make_hparams(), m0(plan), out)
        res.append({v: out[plan.edge_off[t]:plan.edge_off[t + 1]] for t, v in enumerate(plan.nodes)})
    fwd, rev = res
    bad = {v: (util.rel_l2(fwd[v], fx.gold["n%d_mask" % v]), tol[v]) for v in fx.nodes
           if not util.rel_l2(fwd[v], fx.gold["n%d_mask" % v]) <= tol[v]}
    assert not bad, bad
    for v in fx.nodes:
        assert np.array_equal(fwd[v], rev[v]), v
    eng.close()
