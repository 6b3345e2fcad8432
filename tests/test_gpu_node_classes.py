"""GPU (-m gpu): every launch class of the shared-memory node kernel (explain_node.cu).  The pair indices of a task live in its
L2-resident pair slab next to the pair's optimiser state, so every class, the cluster class and the trace / state paths read them
from there.

  * each of the classes 0..4 is reached by the fixtures' golden nodes and by the full syn1 batch;
  * per class: masks against the reference golden at the per-node tolerances, and bit for bit the same alone, in reversed order and
    inside the full 700-node syn1 batch (a task's class depends on the task alone);
  * tasks of the 2-per-SM class (the large syn1 tasks) on thread-block clusters of 2 and 4 CTAs, against the golden and the single-CTA run;
  * trace and optimiser-state I/O on tasks of the 2-per-SM class: a trace leaves the masks unchanged and agrees with the slab kernel's,
    a split run resumed from its state equals the straight run bit for bit."""
import numpy as np
import pytest

from gnnx import _abi
import util

pytestmark = pytest.mark.gpu

SMEM = 5           # launch classes 0..4 of gx_plan_class_counts: the shared-memory kernel
TWO = 3            # the 2-per-SM class


def _class_of(eng, nodes):
    """Launch class of each node, planned alone."""
    out = {}
    for v in nodes:
        eng.plan_nodes([v], 3)
        out[v] = int(np.argmax(eng.plan_class_counts()[0]))
    return out


def _run(eng, nodes, hp, m0=None):
    plan = eng.plan_nodes(nodes, 3)
    out = np.zeros(plan.total_edges, np.float32)
    eng.explain_nodes_host(hp, m0(plan) if m0 else None, out)
    return {v: out[plan.edge_off[t]:plan.edge_off[t + 1]] for t, v in enumerate(plan.nodes)}


def _two_nodes(fx, eng, k):
    cls = _class_of(eng, fx.nodes)
    nodes = [v for v in fx.nodes if cls[v] == TWO][:k]
    assert len(nodes) == k, cls
    return nodes


def test_every_class_is_reached():
    seen = set()
    for which in ("rand", "syn4", "syn1"):
        fx = util.load_fixture(which)
        eng = util.make_engine(fx)
        seen |= set(_class_of(eng, fx.nodes).values())
        eng.close()
    assert set(range(SMEM)) <= seen, sorted(seen)
    fx = util.load_fixture("syn1")
    eng = util.make_engine(fx)
    eng.plan_nodes(np.arange(fx.rowptr.shape[0] - 1, dtype=np.int32), 3)
    counts, cs = eng.plan_class_counts()
    eng.close()
    assert (counts[:SMEM] > 0).all() and counts[SMEM:].sum() == 0 and cs == 1, counts


@pytest.mark.parametrize("which", ["syn1", "syn4", "rand"])
def test_classes_match_golden_and_are_batch_independent(which):
    fx = util.load_fixture(which)
    eng = util.make_engine(fx)
    cls = _class_of(eng, fx.nodes)
    tol = util.node_tolerances(which, 100)
    m0 = lambda plan: util.golden_m0(fx, plan)
    full = _run(eng, fx.nodes, eng.make_hparams(), m0)
    bad = {v: (util.rel_l2(full[v], fx.gold["n%d_mask" % v]), tol[v]) for v in fx.nodes
           if not util.rel_l2(full[v], fx.gold["n%d_mask" % v]) <= tol[v]}
    assert not bad, bad
    hp = eng.make_hparams(num_epochs=10, init=_abi.GX_INIT_PHILOX, seed=7)   # Philox streams are keyed by node id
    whole = _run(eng, list(range(fx.rowptr.shape[0] - 1)) if which == "syn1" else fx.nodes, hp)
    for c in sorted(set(cls.values())):
        nodes = [v for v in fx.nodes if cls[v] == c]
        alone = _run(eng, nodes, hp)
        rev = _run(eng, nodes[::-1], hp)
        for v in nodes:
            assert np.array_equal(alone[v], whole[v]) and np.array_equal(rev[v], whole[v]), (which, c, v)
    eng.close()


@pytest.mark.parametrize("cs", [2, 4])
def test_two_per_sm_tasks_on_clusters(cs):
    fx = util.load_fixture("syn1")
    eng = util.make_engine(fx)
    nodes = _two_nodes(fx, eng, 4)
    m0 = lambda plan: util.golden_m0(fx, plan)
    one = _run(eng, nodes, eng.make_hparams(num_epochs=10), m0)
    eng.debug_cluster(cs, 1)
    plan = eng.plan_nodes(nodes, 3)
    counts, csz = eng.plan_class_counts()
    assert counts[6] == len(nodes) and csz == cs, (counts, csz)
    ten = _run(eng, nodes, eng.make_hparams(num_epochs=10), m0)
    full = _run(eng, nodes, eng.make_hparams(), m0)
    eng.close()
    tol = util.node_tolerances("syn1", 100)
    for v in nodes:
        assert util.rel_l2(ten[v], one[v]) < 2e-6, v
        assert util.rel_l2(full[v], fx.gold["n%d_mask" % v]) <= tol[v], v


def test_two_per_sm_trace_and_state_io():
    fx = util.load_fixture("syn1")
    d = fx.feat.shape[1]
    C = fx.weights["Wp"].shape[0]
    res = {}
    for stream in (False, True):
        eng = util.make_engine(fx)
        nodes = _two_nodes(fx, eng, 3)
        eng.debug_force_stream(stream)
        plan = eng.plan_nodes(nodes, 3)
        assert eng.plan_class_counts()[0][SMEM if stream else TWO] == len(nodes)
        hp = eng.make_hparams(num_epochs=8)
        m0 = util.golden_m0(fx, plan)
        out = np.zeros(plan.total_edges, np.float32)
        tr = np.zeros((plan.count, 8, _abi.GX_TRACE_COLS), np.float32)
        pred = np.zeros((plan.count, 8, C), np.float32)
        eng.explain_nodes_ex(hp, m0, out, trace=tr, trace_pred=pred)
        plain = np.zeros_like(out)
        eng.explain_nodes_host(hp, m0, plain)
        assert np.array_equal(plain, out), "requesting a trace changed the masks"
        res[stream] = (tr, pred)
        if not stream:   # 30 epochs straight == 12 epochs, state out, 18 more from the state
            te = plan.total_edges
            full = np.zeros(te, np.float32); fm_full = np.zeros((plan.count, d), np.float32)
            eng.explain_nodes_host(eng.make_hparams(num_epochs=30), m0, full, fm_full)
            so = dict(M=np.zeros(te, np.float32), m=np.zeros(te, np.float32), v=np.zeros(te, np.float32),
                      feat=np.zeros((plan.count, 3, d), np.float32))
            eng.explain_nodes_ex(eng.make_hparams(num_epochs=12), m0, np.zeros(te, np.float32), state_out=so)
            rest = np.zeros(te, np.float32); fm = np.zeros((plan.count, d), np.float32)
            eng.explain_nodes_ex(eng.make_hparams(num_epochs=19, init=_abi.GX_INIT_STATE, start_step=11), so["M"], rest, feat_mask_out=fm,
                                 state_in=dict(m=so["m"], v=so["v"], feat=so["feat"]))
            assert np.array_equal(rest, full) and np.array_equal(fm, fm_full)
        eng.close()
    assert np.allclose(res[False][0], res[True][0], rtol=1e-4, atol=1e-5)
    assert np.allclose(res[False][1], res[True][1], rtol=1e-4, atol=1e-5)
