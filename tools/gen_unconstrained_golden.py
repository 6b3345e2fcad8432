"""gen_unconstrained_golden.py -- tests/golden/unconstrained_golden.npz by EXECUTING THE UNMODIFIED REFERENCE.

Explainer.explain(..., unconstrained=True) (explain.py:688-692: the dense mask sym(sigmoid(M)) * (1 - I) drives the forward, the
features are not masked) in node mode on the syn1 / syn4 / rand fixtures and in graph mode on the 12 graphs of graphs_golden.npz.
Needs the reference tree (oracle/ref_harness.py); deterministic:
    python tools/gen_unconstrained_golden.py

Keys (masks at the sub-adjacency entries, row-major, float32; spreads float64):
  <fx>_nodes, <fx>_n<node>_nbrs                       node fixtures syn1 / syn4 / rand (weights and seeds of <fx>_graph / _golden)
  <fx>_n<node>_e<E>_mask, _e<E>_spread               E = 10, 30, 100 epochs
  graphs_g<g>_e<E>_mask, _e<E>_spread                 graph mode
  var_<tag>_W<l> / _b<l> / _Wp / _bp / _L / _bn        random models of the variants (rand: GcnEncoderNode, graphs: GcnEncoderGraph)
  var_<tag>_rand_n<node>_mask / _spread / _nbrs, var_<tag>_graphs_g<g>_mask / _spread   at var_epochs, tag = bn / L4 / sgd
  trace_<fx>_n<node>                                   (epoch, loss, mask density, softmax row) printed by print_training=True
The spread of a case is the reproducibility of the reference itself: how far the line-by-line port moves from the reference's mask
when every M0 entry is nudged by +-1 ulp (nudges draws), and how far the fp64 and fp32 closed forms (the same trajectory restated in
another summation order) land from it.  Some dense trajectories are insensitive to M0 noise but not to the order of the sums (a
graph whose fp32 closed form lands 0.14 away at 100 epochs), hence both.  The port (gnnx_oracle.explain_dense_torch,
unconstrained=True) must reproduce every reference mask to below 1e-6.
"""
import contextlib
import io
import os
import re
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import dense_oracle as D  # noqa: E402
import ref_harness  # noqa: E402
from gen_golden import OUT, _load_fixture_model, train_args  # noqa: E402

NODES = {"syn1": [0, 3, 23, 33, 163, 293, 300, 313, 343], "syn4": [0, 1, 4, 100, 511], "rand": [0, 1, 7, 33, 77, 100, 149]}
EPOCHS = (10, 30, 100)
VAR_EPOCHS = 30
VARIANTS = (("bn", 3, True, {}), ("L4", 4, False, {}), ("sgd", 3, False, dict(opt="sgd")))
TRACE = {"syn1": [300, 13], "rand": [0, 33]}
TRACE_EPOCHS = 12


def _nudged(M0, s, salt):
    rng = np.random.default_rng(1000 * s + salt)
    up = rng.integers(0, 2, M0.shape).astype(bool)
    return np.where(up, np.nextafter(M0, np.float32(np.inf)), np.nextafter(M0, np.float32(-np.inf))).astype(np.float32)


def _check(O, port_fn, cf_fn, M0, ref, ei, ej, nudges, salt, what):
    mine = port_fn(M0)
    err = O.rel_l2(mine[ei, ej], ref)
    assert err < 1e-6, (what, err)
    spread = max(O.rel_l2(cf_fn(M0, dt)[ei, ej], ref) for dt in (np.float64, np.float32))
    for s in range(nudges):
        spread = max(spread, O.rel_l2(port_fn(_nudged(M0, s, salt))[ei, ej], ref))
    return spread


def _weights_of(model, L):
    sd = model.state_dict()
    keys = ["conv_first"] + ["conv_block.%d" % i for i in range(L - 2)] + ["conv_last"]
    W = {}
    for l, k in enumerate(keys, 1):
        W["W%d" % l] = sd[k + ".weight"].numpy().astype(np.float32)
        W["b%d" % l] = sd[k + ".bias"].numpy().astype(np.float32)
    W["Wp"] = sd["pred_model.weight"].numpy().astype(np.float32)
    W["bp"] = sd["pred_model.bias"].numpy().astype(np.float32)
    return W


def _random_model(cls, d, C, L, bn, seed):
    torch.manual_seed(seed)
    model = cls(d, 20, 20, C, L, bn=bn, args=train_args(input_dim=d, num_gc_layers=L, bn=bn))
    with torch.no_grad():
        for name, p_ in model.named_parameters():
            if name.endswith("bias"):
                p_.normal_(0.0, 0.3)
    model.eval()
    return model


def _explain_nodes(R, O, out, key, ex, nodes, seeds, W, hp_over, epochs, bn, nudges, with_nbrs=False):
    """The reference's explain(node, unconstrained=True) on `nodes` and the port on the same inputs."""
    hp = O.default_hparams(num_epochs=epochs, **hp_over)
    for node in nodes:
        with ref_harness.quiet():
            idx, sub_adj, sub_feat, sub_label, nbrs = ex.extract_neighborhood(node, 0)
        n = len(nbrs)
        M0 = O.draw_m0(n, seed=seeds[node])
        torch.manual_seed(seeds[node])
        with ref_harness.quiet():
            masked = np.asarray(ex.explain(node, graph_idx=0, unconstrained=True))
        ei, ej = np.nonzero(sub_adj)
        off = masked.copy(); off[ei, ej] = 0
        assert np.all(off == 0)
        ref = masked[ei, ej]
        pl = np.argmax(np.asarray(ex.pred[0])[nbrs], axis=1)
        gt = int(np.asarray(sub_label)[idx])
        A = np.asarray(sub_adj, np.float64)
        port = lambda M: O.explain_dense_torch(A, sub_feat, gt, pl, idx, W, M, hp=hp, bn=bn, unconstrained=True)
        cf = lambda M, dt: D.explain_closed_form(A, sub_feat, gt, pl, idx, W, M, hp=hp, bn=bn, dtype=dt)
        out[key % node + "_mask"] = ref.astype(np.float32)
        out[key % node + "_spread"] = np.float64(_check(O, port, cf, M0, ref, ei, ej, nudges, node, (key % node)))
        if with_nbrs:
            out[key % node + "_nbrs"] = np.asarray(nbrs, np.int32)


def _explain_graphs(R, O, out, key, model, gg, W, L, bn, hp_over, epochs, nudges):
    G_n, n = int(gg["num_graphs"]), int(gg["max_nodes"])
    adj, feat, label = gg["adj"].astype(np.float64), gg["feat"].astype(np.float32), gg["label"].astype(np.int64)
    with torch.no_grad():
        pred = np.stack([model(torch.tensor(feat[g:g + 1]), torch.tensor(adj[g:g + 1], dtype=torch.float))[0][0].numpy()
                         for g in range(G_n)])[None]
    eargs = ref_harness.explainer_args(dataset="uncon", num_epochs=epochs, num_gc_layers=L, bn=bn, **hp_over)
    with ref_harness.quiet():
        ex = R.explain.Explainer(model=model, adj=torch.tensor(adj, dtype=torch.float), feat=torch.tensor(feat),
                                 label=torch.tensor(label), pred=pred, train_idx=list(range(G_n)), args=eargs,
                                 writer=None, print_training=False, graph_mode=True, graph_idx=0)
    hp = O.default_hparams(num_epochs=epochs, **hp_over)
    for g in range(G_n):
        seed = int(gg["g%d_seed" % g])
        M0 = O.draw_m0(n, seed=seed)
        torch.manual_seed(seed)
        with ref_harness.quiet():
            masked = np.asarray(ex.explain(node_idx=0, graph_idx=g, graph_mode=True, unconstrained=True))
        ei, ej = np.nonzero(adj[g])
        off = masked.copy(); off[ei, ej] = 0
        assert np.all(off == 0)
        ref = masked[ei, ej]
        port = lambda M: O.explain_dense_torch(adj[g], feat[g], int(label[g]), None, 0, W, M, hp=hp, graph_mode=True, bn=bn,
                                               unconstrained=True)
        cf = lambda M, dt: D.explain_closed_form(adj[g], feat[g], int(label[g]), None, 0, W, M, hp=hp, graph_mode=True, bn=bn, dtype=dt)
        out[key % g + "_mask"] = ref.astype(np.float32)
        out[key % g + "_spread"] = np.float64(_check(O, port, cf, M0, ref, ei, ej, nudges, 100 + g, key % g))


def gen(R, nudges=4):
    import gnnx_oracle as O
    out = {"epochs": np.asarray(EPOCHS, np.int64), "var_epochs": np.int64(VAR_EPOCHS), "trace_epochs": np.int64(TRACE_EPOCHS)}
    # ---- node mode on the committed fixtures (their weights, and the M0 seeds of <fx>_golden.npz)
    for fx, nodes in NODES.items():
        out[fx + "_nodes"] = np.asarray(nodes, np.int64)
        for E in EPOCHS:
            make, g, gold = _load_fixture_model(R, fx, num_epochs=E)
            W = {k: g[k] for k in ("W1", "b1", "W2", "b2", "W3", "b3", "Wp", "bp")}
            seeds = {node: int(gold["n%d_seed" % node]) for node in nodes}
            _explain_nodes(R, O, out, fx + "_n%d" + "_e%d" % E, make(), nodes, seeds, W, {}, E, False, nudges, with_nbrs=False)
        print("  %s: %d nodes, spreads e100 %s" % (fx, len(nodes), ["%.1e" % out["%s_n%d_e100_spread" % (fx, v)] for v in nodes]), flush=True)
    # ---- graph mode on graphs_golden.npz (its model and seeds)
    gg = np.load(os.path.join(OUT, "graphs_golden.npz"))
    d, C = gg["feat"].shape[2], gg["Wp"].shape[0]
    base = R.models.GcnEncoderGraph(d, 20, 20, C, 3, bn=False, args=train_args(input_dim=d))
    base.load_state_dict({k: torch.tensor(gg[w]) for k, w in (("conv_first.weight", "W1"), ("conv_first.bias", "b1"),
                          ("conv_block.0.weight", "W2"), ("conv_block.0.bias", "b2"), ("conv_last.weight", "W3"),
                          ("conv_last.bias", "b3"), ("pred_model.weight", "Wp"), ("pred_model.bias", "bp"))})
    base.eval()
    Wg = _weights_of(base, 3)
    for E in EPOCHS:
        _explain_graphs(R, O, out, "graphs_g%d" + "_e%d" % E, base, gg, Wg, 3, False, {}, E, nudges)
    print("  graphs: spreads e100 %s" % ["%.1e" % out["graphs_g%d_e100_spread" % g] for g in range(int(gg["num_graphs"]))], flush=True)
    # ---- variants: --bn, 4 layers (random models) and SGD (the fixture models), rand nodes and the graphs
    make_r, gr, gold_r = _load_fixture_model(R, "rand", num_epochs=VAR_EPOCHS)
    seeds_r = {node: int(gold_r["n%d_seed" % node]) for node in NODES["rand"]}
    N = int(gr["N"]); dr = gr["feat"].shape[1]; Cr = gr["Wp"].shape[0]
    adj_r = np.zeros((1, N, N)); e = gr["edges"]; adj_r[0, e[:, 0], e[:, 1]] = 1; adj_r[0, e[:, 1], e[:, 0]] = 1
    for tag, L, bn, over in VARIANTS:
        if over:
            model_n, Wn = None, {k: gr[k] for k in ("W1", "b1", "W2", "b2", "W3", "b3", "Wp", "bp")}
            ex = make_r(**over)
            model_g, Wgv = base, Wg
        else:
            model_n = _random_model(R.models.GcnEncoderNode, dr, Cr, L, bn, 300 + 10 * L + int(bn))
            Wn = _weights_of(model_n, L)
            with torch.no_grad():
                pred, _ = model_n(torch.tensor(gr["feat"][None], dtype=torch.float), torch.tensor(adj_r, dtype=torch.float))
            eargs = ref_harness.explainer_args(dataset="rand", num_epochs=VAR_EPOCHS, num_gc_layers=L, bn=bn)
            with ref_harness.quiet():
                ex = R.explain.Explainer(model=model_n, adj=adj_r, feat=gr["feat"][None].astype(np.float64), label=gr["label"][None],
                                         pred=pred.numpy(), train_idx=list(range(N)), args=eargs, writer=None, print_training=False,
                                         graph_idx=-1)
            out.update({"var_%s_rand_%s" % (tag, k): v for k, v in Wn.items()})
            model_g = _random_model(R.models.GcnEncoderGraph, d, C, L, bn, 400 + 10 * L + int(bn))
            Wgv = _weights_of(model_g, L)
            out.update({"var_%s_graphs_%s" % (tag, k): v for k, v in Wgv.items()})
        out["var_%s_L" % tag] = np.int64(L); out["var_%s_bn" % tag] = np.int64(bn)
        _explain_nodes(R, O, out, "var_" + tag + "_rand_n%d", ex, NODES["rand"], seeds_r, Wn, over, VAR_EPOCHS, bn, nudges, with_nbrs=True)
        _explain_graphs(R, O, out, "var_" + tag + "_graphs_g%d", model_g, gg, Wgv, L, bn, over, VAR_EPOCHS, nudges)
        print("  variant %s done" % tag, flush=True)
    # ---- what print_training prints every epoch (oracle/gen_golden.py:gen_trace), node mode
    for fx, nodes in TRACE.items():
        make, g, gold = _load_fixture_model(R, fx, num_epochs=TRACE_EPOCHS)
        ex = make(print_training=True)
        for node in nodes:
            buf = io.StringIO()
            torch.manual_seed(int(gold["n%d_seed" % node]))
            torch.set_printoptions(precision=8, sci_mode=False)
            with contextlib.redirect_stdout(buf):
                ex.explain(node, graph_idx=0, unconstrained=True)
            rows = []
            for mt in re.finditer(r"epoch:\s+(\d+)\s+; loss:\s+(\S+)\s+; mask density:\s+(\S+)\s+; pred:\s+tensor\(\[([^\]]*)\]", buf.getvalue()):
                rows.append([float(mt.group(2)), float(mt.group(3))] + [float(x) for x in mt.group(4).replace("\n", " ").split(",")])
            assert len(rows) == TRACE_EPOCHS, (fx, node, len(rows))
            out["trace_%s_n%d" % (fx, node)] = np.asarray(rows, np.float64)
        out["trace_%s_nodes" % fx] = np.asarray(nodes, np.int64)
    torch.set_printoptions(profile="default")
    np.savez_compressed(os.path.join(OUT, "unconstrained_golden.npz"), **out)
    print("  unconstrained golden written")


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen(ref_harness.load())
