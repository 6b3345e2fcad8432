"""gen_unconstrained_full_golden.py -- tests/golden/unconstrained_full_golden.npz by EXECUTING THE UNMODIFIED REFERENCE.

Explainer.explain(..., unconstrained=True) returns masked_adj[0] * sub_adj (explain.py:209-211): the sub-adjacency slots only.  The
optimisation moves every one of the n^2 entries (ExplainModule.forward, explain.py:688-692), so this fixture keeps the WHOLE
masked_adj[0] the last epoch's forward built, read from the ExplainModule instance explain() creates (its __init__ is wrapped while explain() runs
to record the instance; nothing in the reference is modified).  Needs the reference tree (oracle/ref_harness.py);
deterministic:
    python tools/gen_unconstrained_full_golden.py

Keys (full masks float32 (n, n), row-major as the reference's; spreads float64):
  epochs, <fx>_nodes, graphs                    fixtures syn1 / syn4 / rand (their weights and M0 seeds) and graphs_golden.npz
  <fx>_n<node>_nbrs                             the node's 3-hop set, ascending (the reference's extract_neighborhood)
  <fx>_n<node>_e<E>_full, graphs_g<g>_e<E>_full E = 10, 30 epochs
  <case>_e<E>_spread_<cls>, _cfdist_<cls>       per entry class cls (tests/dense_oracle.entry_classes: edge, nonedge, pad)
The spread of a class is the reproducibility of the reference itself, as oracle/gen_sensitivity.py measures it: the largest rel-L2,
over the class's entries, of the line-by-line port from the reference's mask when every M0 entry is nudged by +-1 ulp (twelve random
sign patterns; four more that also nudge every model weight).  cfdist is the rel-L2 of the fp64 closed form from the port.  The port
(oracle/gnnx_oracle.explain_dense_torch, unconstrained=True) must reproduce every full reference mask bit for bit.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import dense_oracle as D  # noqa: E402
import gnnx_oracle as O  # noqa: E402
import ref_harness  # noqa: E402
from gen_golden import OUT, _load_fixture_model, train_args  # noqa: E402

NODES = {"syn1": [301, 313, 343, 403], "syn4": [0, 1, 100, 511], "rand": [33, 77, 149]}
GRAPHS = [0, 4, 7, 9]
EPOCHS = (10, 30)
NUDGES = 16          # the first 12 nudge M0 only, the last 4 also every weight (oracle/gen_sensitivity.py)


def _nudge(x, rng):
    x = np.asarray(x, np.float32)
    up = rng.integers(0, 2, x.shape).astype(bool)
    return np.where(up, np.nextafter(x, np.float32(np.inf)), np.nextafter(x, np.float32(-np.inf))).astype(np.float32)


class _Recorder:
    """Wraps ExplainModule.__init__ (the reference calls super(ExplainModule, self), so the class itself must stay) to remember the
    last instance: explain() builds one per call."""

    def __init__(self, R):
        self.cls, self.last = R.explain.ExplainModule, None

    def __enter__(self):
        self.orig = self.cls.__init__
        orig, rec = self.orig, self

        def init(module, *a, **k):
            orig(module, *a, **k)
            rec.last = module
        self.cls.__init__ = init
        return self

    def __exit__(self, *exc):
        self.cls.__init__ = self.orig

    def full(self):
        return self.last.masked_adj[0].detach().numpy().astype(np.float32).copy()


def _record(out, key, A, ref_full, port_fn, cf_fn, M0, W, salt):
    """Checks the port reproduces ref_full bit for bit, then stores the full mask, the spread and the closed form's distance per class."""
    mine = port_fn(M0, W)
    assert np.array_equal(mine.astype(np.float32), ref_full), (key, np.abs(mine - ref_full).max())
    cls = D.entry_classes(A)
    cf = cf_fn(M0)
    spread = {c: 0.0 for c in cls}
    for s in range(NUDGES):
        rng = np.random.default_rng(1000 * s + salt)
        Ws = W if s < 12 else {k: _nudge(v, rng) for k, v in W.items()}
        res = port_fn(_nudge(M0, rng), Ws)
        for c, (r, k) in cls.items():
            spread[c] = max(spread[c], O.rel_l2(res[r, k], ref_full[r, k]))
    out[key + "_full"] = ref_full
    for c, (r, k) in cls.items():
        out[key + "_spread_" + c] = np.float64(spread[c])
        out[key + "_cfdist_" + c] = np.float64(O.rel_l2(cf[r, k], mine[r, k]))
    return spread


def gen(R):
    out = {"epochs": np.asarray(EPOCHS, np.int64), "graphs": np.asarray(GRAPHS, np.int64)}
    for fx, nodes in NODES.items():
        out[fx + "_nodes"] = np.asarray(nodes, np.int64)
        for E in EPOCHS:
            make, g, gold = _load_fixture_model(R, fx, num_epochs=E)
            ex = make()
            W = {k: g[k] for k in ("W1", "b1", "W2", "b2", "W3", "b3", "Wp", "bp")}
            hp = O.default_hparams(num_epochs=E)
            for node in nodes:
                with ref_harness.quiet():
                    idx, sub_adj, sub_feat, sub_label, nbrs = ex.extract_neighborhood(node, 0)
                seed = int(gold["n%d_seed" % node])
                torch.manual_seed(seed)
                with ref_harness.quiet(), _Recorder(R) as rec:
                    masked = np.asarray(ex.explain(node, graph_idx=0, unconstrained=True))
                full = rec.full()
                A = np.asarray(sub_adj, np.float64)
                assert np.array_equal(masked, full * A)     # what explain() returns is this matrix at the sub-adjacency slots
                pl = np.argmax(np.asarray(ex.pred[0])[nbrs], axis=1)
                gt = int(np.asarray(sub_label)[idx])
                M0 = O.draw_m0(len(nbrs), seed=seed)
                key = "%s_n%d_e%d" % (fx, node, E)
                sp = _record(out, key, A, full,
                             lambda M, Wx: O.explain_dense_torch(A, sub_feat, gt, pl, idx, Wx, M, hp=hp, full=True, unconstrained=True),
                             lambda M: D.explain_closed_form(A, sub_feat, gt, pl, idx, W, M, hp=hp, full=True), M0, W, node)
                out["%s_n%d_nbrs" % (fx, node)] = np.asarray(nbrs, np.int32)
                print("  %s n=%d: %s" % (key, len(nbrs), {c: "%.1e" % v for c, v in sp.items()}), flush=True)
    gg = np.load(os.path.join(OUT, "graphs_golden.npz"))
    G_n, n = int(gg["num_graphs"]), int(gg["max_nodes"])
    d, C = gg["feat"].shape[2], gg["Wp"].shape[0]
    model = R.models.GcnEncoderGraph(d, 20, 20, C, 3, bn=False, args=train_args(input_dim=d))
    model.load_state_dict({k: torch.tensor(gg[w]) for k, w in (("conv_first.weight", "W1"), ("conv_first.bias", "b1"),
                           ("conv_block.0.weight", "W2"), ("conv_block.0.bias", "b2"), ("conv_last.weight", "W3"),
                           ("conv_last.bias", "b3"), ("pred_model.weight", "Wp"), ("pred_model.bias", "bp"))})
    model.eval()
    W = {k: gg[k] for k in ("W1", "b1", "W2", "b2", "W3", "b3", "Wp", "bp")}
    adj, feat, label = gg["adj"].astype(np.float64), gg["feat"].astype(np.float32), gg["label"].astype(np.int64)
    with torch.no_grad():
        pred = np.stack([model(torch.tensor(feat[g:g + 1]), torch.tensor(adj[g:g + 1], dtype=torch.float))[0][0].numpy()
                         for g in range(G_n)])[None]
    for E in EPOCHS:
        eargs = ref_harness.explainer_args(dataset="uncon", num_epochs=E)
        with ref_harness.quiet():
            ex = R.explain.Explainer(model=model, adj=torch.tensor(adj, dtype=torch.float), feat=torch.tensor(feat),
                                     label=torch.tensor(label), pred=pred, train_idx=list(range(G_n)), args=eargs,
                                     writer=None, print_training=False, graph_mode=True, graph_idx=0)
        hp = O.default_hparams(num_epochs=E)
        for g in GRAPHS:
            seed = int(gg["g%d_seed" % g])
            torch.manual_seed(seed)
            with ref_harness.quiet(), _Recorder(R) as rec:
                masked = np.asarray(ex.explain(node_idx=0, graph_idx=g, graph_mode=True, unconstrained=True))
            full = rec.full()
            assert np.array_equal(masked, full * adj[g])
            M0 = O.draw_m0(n, seed=seed)
            key = "graphs_g%d_e%d" % (g, E)
            sp = _record(out, key, adj[g], full,
                         lambda M, Wx: O.explain_dense_torch(adj[g], feat[g], int(label[g]), None, 0, Wx, M, hp=hp, graph_mode=True,
                                                             full=True, unconstrained=True),
                         lambda M: D.explain_closed_form(adj[g], feat[g], int(label[g]), None, 0, W, M, hp=hp, graph_mode=True, full=True),
                         M0, W, 100 + g)
            print("  %s: %s" % (key, {c: "%.1e" % v for c, v in sp.items()}), flush=True)
    np.savez_compressed(os.path.join(OUT, "unconstrained_full_golden.npz"), **out)
    print("  unconstrained full golden written")


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen(ref_harness.load())
