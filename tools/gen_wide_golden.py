"""gen_wide_golden.py -- tests/golden/wide_golden.npz by EXECUTING THE UNMODIFIED REFERENCE on models whose input is wider than 128
features (the wide path of csrc/explain_var.cu).

The reference's GcnEncoderNode / GcnEncoderGraph (models.py, reference init), biases redrawn from N(0, 0.3) so that they matter,
explained with Explainer.explain (model="exp"):
  * node mode on the rand fixture graph with d = 300 random N(0, 1) features: 3 layers at 30 and 100 epochs, --bn with 2 layers, SGD;
  * graph mode on the 12 graphs of graphs_golden.npz with one-hot features over 190 node labels: 3 layers, --bn with 4 layers.
Needs the reference tree (oracle/ref_harness.py); deterministic:
    python tools/gen_wide_golden.py

Keys (masks at the sub-adjacency entries, row-major, float32; spreads float64):
  cases                                            the case names
  <case>_mode / _L / _bn / _opt / _epochs          node (0) or graph (1) mode, the model, the optimiser, the epochs
  <case>_w_<W1 .. WL, b1 .., Wp, bp>               the model's weights (reference state_dict, renamed)
  <case>_feat                                      the features the case used: (N, 300) node mode, (G, max_nodes, 190) graph mode
  <case>_pred                                      the model's forward on the graph (node mode) or on each padded graph (graph mode)
  <case>_nodes, <case>_n<node>_seed / _nbrs / _mask / _spread   node mode
  <case>_g<g>_mask / _spread                       graph mode (M0 seeds: graphs_golden.npz g<g>_seed)
The spread of a mask is the reproducibility of the reference itself: the largest distance from the reference's mask of the torch port
(gnnx_oracle.explain_dense_torch) run with every M0 entry nudged by +-1 ulp (NUDGES draws), and of the same port in fp64.  The port
must land within max(1e-6, 3 x spread) of every reference mask.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import gnnx_oracle as O  # noqa: E402
import ref_harness  # noqa: E402
from gen_golden import OUT, train_args  # noqa: E402

NUDGES = 3
D_NODE, D_GRAPH = 300, 190
NODES = [0, 7, 33, 100]
# name: (L, bn, opt, epochs)
NODE_CASES = {"rand_L3_e30": (3, False, "adam", 30), "rand_L3_e100": (3, False, "adam", 100), "rand_bn_L2": (2, True, "adam", 30),
              "rand_sgd": (3, False, "sgd", 30)}
GRAPH_CASES = {"graphs_L3": (3, False, "adam", 30), "graphs_bn_L4": (4, True, "adam", 30)}


def _nudged(M0, s, salt):
    rng = np.random.default_rng(1000 * s + salt)
    up = rng.integers(0, 2, M0.shape).astype(bool)
    return np.where(up, np.nextafter(M0, np.float32(np.inf)), np.nextafter(M0, np.float32(-np.inf))).astype(np.float32)


def _spread(port, M0, ref, ei, ej, salt, what):
    spread = O.rel_l2(port(M0, torch.float64)[ei, ej], ref)
    for s in range(NUDGES):
        spread = max(spread, O.rel_l2(port(_nudged(M0, s, salt), torch.float)[ei, ej], ref))
    err = O.rel_l2(port(M0, torch.float)[ei, ej], ref)
    assert err <= max(1e-6, 3 * spread), (what, err, spread)
    return spread


def _model(cls, d, C, L, bn, seed):
    torch.manual_seed(seed)
    model = cls(d, 20, 20, C, L, bn=bn, args=train_args(input_dim=d, hidden_dim=20, output_dim=20, num_gc_layers=L, bn=bn))
    with torch.no_grad():
        for name, p_ in model.named_parameters():
            if name.endswith("bias"):
                p_.normal_(0.0, 0.3)
    model.eval()
    sd = model.state_dict()
    keys = ["conv_first"] + ["conv_block.%d" % i for i in range(L - 2)] + ["conv_last"]
    W = {}
    for l, k in enumerate(keys, 1):
        W["W%d" % l] = sd[k + ".weight"].numpy().astype(np.float32)
        W["b%d" % l] = sd[k + ".bias"].numpy().astype(np.float32)
    W["Wp"] = sd["pred_model.weight"].numpy().astype(np.float32)
    W["bp"] = sd["pred_model.bias"].numpy().astype(np.float32)
    return model, W


def _meta(out, name, mode, L, bn, opt, epochs, W, feat, pred):
    out.update({"%s_w_%s" % (name, k): v for k, v in W.items()})
    out.update({name + "_mode": np.int64(mode), name + "_L": np.int64(L), name + "_bn": np.int64(bn), name + "_opt": np.str_(opt),
                name + "_epochs": np.int64(epochs), name + "_feat": feat, name + "_pred": pred})


def gen_node_case(R, out, name, L, bn, opt, epochs, seed):
    g = np.load(os.path.join(OUT, "rand_graph.npz"))
    gold = np.load(os.path.join(OUT, "rand_golden.npz"))
    N, C = int(g["N"]), g["Wp"].shape[0]
    feat = np.random.default_rng(seed).normal(size=(N, D_NODE)).astype(np.float32)
    adj = np.zeros((1, N, N)); e = g["edges"]; adj[0, e[:, 0], e[:, 1]] = 1; adj[0, e[:, 1], e[:, 0]] = 1
    model, W = _model(R.models.GcnEncoderNode, D_NODE, C, L, bn, seed)
    with torch.no_grad():
        pred, _ = model(torch.tensor(feat[None]), torch.tensor(adj, dtype=torch.float))
    eargs = ref_harness.explainer_args(dataset="rand", num_epochs=epochs, num_gc_layers=L, bn=bn, opt=opt)
    with ref_harness.quiet():
        ex = R.explain.Explainer(model=model, adj=adj, feat=feat[None].astype(np.float64), label=g["label"][None], pred=pred.numpy(),
                                 train_idx=list(range(N)), args=eargs, writer=None, print_training=False, graph_idx=-1)
    _meta(out, name, 0, L, bn, opt, epochs, W, feat, pred[0].numpy())
    out[name + "_nodes"] = np.asarray(NODES, np.int64)
    hp = O.default_hparams(num_epochs=epochs, opt=opt)
    for node in NODES:
        seed_n = int(gold["n%d_seed" % node])
        with ref_harness.quiet():
            idx, sub_adj, sub_feat, sub_label, nbrs = ex.extract_neighborhood(node, 0)
        M0 = O.draw_m0(len(nbrs), seed=seed_n)
        torch.manual_seed(seed_n)
        with ref_harness.quiet():
            masked = np.asarray(ex.explain(node, graph_idx=0))
        ei, ej = np.nonzero(sub_adj)
        ref = masked[ei, ej]
        pl = np.argmax(pred[0].numpy()[nbrs], axis=1)
        gt = int(np.asarray(sub_label)[idx])
        A = np.asarray(sub_adj, np.float64)
        port = lambda M, dt: O.explain_dense_torch(A, np.asarray(sub_feat, np.float32), gt, pl, idx, W, M, hp, bn=bn, dtype=dt)
        key = "%s_n%d" % (name, node)
        out[key + "_seed"] = np.int64(seed_n)
        out[key + "_nbrs"] = np.asarray(nbrs, np.int32)
        out[key + "_mask"] = ref.astype(np.float32)
        out[key + "_spread"] = np.float64(_spread(port, M0, ref, ei, ej, node, key))
    print("  %s: spreads %s" % (name, ["%.1e" % out["%s_n%d_spread" % (name, v)] for v in NODES]), flush=True)


def gen_graph_case(R, out, name, L, bn, opt, epochs, seed):
    gg = np.load(os.path.join(OUT, "graphs_golden.npz"))
    G_n, n = int(gg["num_graphs"]), int(gg["max_nodes"])
    adj, label = gg["adj"].astype(np.float64), gg["label"].astype(np.int64)
    labels = np.random.default_rng(seed).integers(0, D_GRAPH, size=(G_n, n))
    feat = (np.eye(D_GRAPH, dtype=np.float32)[labels] * (adj.sum(2, keepdims=True) > 0)).astype(np.float32)   # one-hot node labels
    C = gg["Wp"].shape[0]
    model, W = _model(R.models.GcnEncoderGraph, D_GRAPH, C, L, bn, seed)
    with torch.no_grad():
        pred = np.stack([model(torch.tensor(feat[g:g + 1]), torch.tensor(adj[g:g + 1], dtype=torch.float))[0][0].numpy()
                         for g in range(G_n)])
    eargs = ref_harness.explainer_args(dataset="graphs", num_epochs=epochs, num_gc_layers=L, bn=bn, opt=opt)
    with ref_harness.quiet():
        ex = R.explain.Explainer(model=model, adj=torch.tensor(adj, dtype=torch.float), feat=torch.tensor(feat),
                                 label=torch.tensor(label), pred=pred[None], train_idx=list(range(G_n)), args=eargs,
                                 writer=None, print_training=False, graph_mode=True, graph_idx=0)
    _meta(out, name, 1, L, bn, opt, epochs, W, feat, pred)
    hp = O.default_hparams(num_epochs=epochs, opt=opt)
    for g in range(G_n):
        seed_g = int(gg["g%d_seed" % g])
        M0 = O.draw_m0(n, seed=seed_g)
        torch.manual_seed(seed_g)
        with ref_harness.quiet():
            masked = np.asarray(ex.explain(node_idx=0, graph_idx=g, graph_mode=True))
        ei, ej = np.nonzero(adj[g])
        ref = masked[ei, ej]
        port = lambda M, dt: O.explain_dense_torch(adj[g], feat[g], int(label[g]), None, 0, W, M, hp, graph_mode=True, bn=bn, dtype=dt)
        out["%s_g%d_mask" % (name, g)] = ref.astype(np.float32)
        out["%s_g%d_spread" % (name, g)] = np.float64(_spread(port, M0, ref, ei, ej, 100 + g, "%s_g%d" % (name, g)))
    print("  %s: spreads %s" % (name, ["%.1e" % out["%s_g%d_spread" % (name, g)] for g in range(G_n)]), flush=True)


def gen(R):
    out = {"cases": np.asarray(list(NODE_CASES) + list(GRAPH_CASES))}
    for k, (name, c) in enumerate(NODE_CASES.items()):
        gen_node_case(R, out, name, *c, seed=800 + k)
    for k, (name, c) in enumerate(GRAPH_CASES.items()):
        gen_graph_case(R, out, name, *c, seed=900 + k)
    np.savez_compressed(os.path.join(OUT, "wide_golden.npz"), **out)
    print("  wide golden written")


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen(ref_harness.load())
