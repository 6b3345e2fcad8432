"""gen_deep_golden.py -- tests/golden/deep_golden.npz by EXECUTING THE UNMODIFIED REFERENCE on GCNs with five to seven graph-convolution
layers (--num-gc-layers 5 .. 7, explain.py:64: n_hops = num_gc_layers).

The reference's GcnEncoderNode / GcnEncoderGraph (models.py, reference init), biases redrawn from N(0, 0.3) so that they matter,
explained with Explainer.explain (model="exp"):
  * node mode on the rand fixture graph (its own features), 4 nodes each: 5, 6 and 7 layers at 30 epochs, 5 layers at 100 epochs,
    --bn with 6 layers, hidden / output 64 / 48 with 5 layers, SGD with 5 layers, an attention model (--method att) with 5 layers;
  * graph mode on the 12 graphs of graphs_golden.npz: 5 layers, --bn with 7 layers.
Needs the reference tree (oracle/ref_harness.py); deterministic:
    python tools/gen_deep_golden.py

Keys (masks at the sub-adjacency entries, row-major, float32; spreads float64):
  cases                                                 the case names
  <case>_mode / _L / _bn / _att / _hid / _emb / _opt / _epochs   node (0) or graph (1) mode, the model, the optimiser, the epochs
  <case>_w_<W1 .. WL, b1 .., Wa1 .. (att), Wp, bp>      the model's weights (reference state_dict, renamed)
  <case>_pred                                           the model's forward on the rand graph (node mode) or on each padded graph
  <case>_nodes, <case>_n<node>_seed / _nbrs / _mask / _spread   node mode (M0 seeds: rand_golden.npz n<node>_seed)
  <case>_g<g>_mask / _spread                            graph mode (M0 seeds: graphs_golden.npz g<g>_seed)
The spread of a mask is the reproducibility of the reference itself: the largest distance from the reference's mask of the torch port
(oracle/gnnx_oracle.explain_dense_torch) run with every M0 entry nudged by +-1 ulp (NUDGES draws), and of the same port in fp64.
The port must land within max(1e-6, 3 x spread) of every reference mask.
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
NODES = [0, 7, 33, 100]
# name: (L, bn, att, hid, emb, opt, epochs)
NODE_CASES = {"rand_L5_e30": (5, False, False, 20, 20, "adam", 30), "rand_L6_e30": (6, False, False, 20, 20, "adam", 30),
              "rand_L7_e30": (7, False, False, 20, 20, "adam", 30), "rand_L5_e100": (5, False, False, 20, 20, "adam", 100),
              "rand_bn_L6": (6, True, False, 20, 20, "adam", 30), "rand_L5_h64_o48": (5, False, False, 64, 48, "adam", 30),
              "rand_L5_sgd": (5, False, False, 20, 20, "sgd", 30), "rand_L5_att": (5, False, True, 20, 20, "adam", 30)}
GRAPH_CASES = {"graphs_L5": (5, False, False, 20, 20, "adam", 30), "graphs_bn_L7": (7, True, False, 20, 20, "adam", 30)}


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


def _model(cls, d, C, L, bn, att, hid, emb, seed):
    torch.manual_seed(seed)
    over = dict(method="att") if att else {}
    model = cls(d, hid, emb, C, L, bn=bn, args=train_args(input_dim=d, hidden_dim=hid, output_dim=emb, num_gc_layers=L, bn=bn, **over))
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
        if att:
            W["Wa%d" % l] = sd[k + ".att_weight"].numpy().astype(np.float32)
    W["Wp"] = sd["pred_model.weight"].numpy().astype(np.float32)
    W["bp"] = sd["pred_model.bias"].numpy().astype(np.float32)
    return model, W


def _meta(out, name, mode, L, bn, att, hid, emb, opt, epochs, W, pred):
    out.update({"%s_w_%s" % (name, k): v for k, v in W.items()})
    out.update({name + "_mode": np.int64(mode), name + "_L": np.int64(L), name + "_bn": np.int64(bn), name + "_att": np.int64(att),
                name + "_hid": np.int64(hid), name + "_emb": np.int64(emb), name + "_opt": np.str_(opt), name + "_epochs": np.int64(epochs),
                name + "_pred": pred})


def gen_node_case(R, out, name, L, bn, att, hid, emb, opt, epochs, seed):
    g = np.load(os.path.join(OUT, "rand_graph.npz"))
    gold = np.load(os.path.join(OUT, "rand_golden.npz"))
    N, C = int(g["N"]), g["Wp"].shape[0]
    feat = g["feat"].astype(np.float32)
    adj = np.zeros((1, N, N)); e = g["edges"]; adj[0, e[:, 0], e[:, 1]] = 1; adj[0, e[:, 1], e[:, 0]] = 1
    model, W = _model(R.models.GcnEncoderNode, feat.shape[1], C, L, bn, att, hid, emb, seed)
    with torch.no_grad():
        pred, _ = model(torch.tensor(feat[None]), torch.tensor(adj, dtype=torch.float))
    over = dict(method="att") if att else {}
    eargs = ref_harness.explainer_args(dataset="rand", num_epochs=epochs, num_gc_layers=L, bn=bn, opt=opt, hidden_dim=hid, output_dim=emb,
                                       **over)
    with ref_harness.quiet():
        ex = R.explain.Explainer(model=model, adj=adj, feat=feat[None].astype(np.float64), label=g["label"][None], pred=pred.numpy(),
                                 train_idx=list(range(N)), args=eargs, writer=None, print_training=False, graph_idx=-1)
    _meta(out, name, 0, L, bn, att, hid, emb, opt, epochs, W, pred[0].numpy())
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
    print("  %s: n %s, spreads %s" % (name, [len(out["%s_n%d_nbrs" % (name, v)]) for v in NODES],
                                      ["%.1e" % out["%s_n%d_spread" % (name, v)] for v in NODES]), flush=True)


def gen_graph_case(R, out, name, L, bn, att, hid, emb, opt, epochs, seed):
    gg = np.load(os.path.join(OUT, "graphs_golden.npz"))
    G_n, n = int(gg["num_graphs"]), int(gg["max_nodes"])
    adj, feat, label = gg["adj"].astype(np.float64), gg["feat"].astype(np.float32), gg["label"].astype(np.int64)
    C = gg["Wp"].shape[0]
    model, W = _model(R.models.GcnEncoderGraph, feat.shape[2], C, L, bn, att, hid, emb, seed)
    with torch.no_grad():
        pred = np.stack([model(torch.tensor(feat[g:g + 1]), torch.tensor(adj[g:g + 1], dtype=torch.float))[0][0].numpy()
                         for g in range(G_n)])
    eargs = ref_harness.explainer_args(dataset="graphs", num_epochs=epochs, num_gc_layers=L, bn=bn, opt=opt, hidden_dim=hid, output_dim=emb)
    with ref_harness.quiet():
        ex = R.explain.Explainer(model=model, adj=torch.tensor(adj, dtype=torch.float), feat=torch.tensor(feat),
                                 label=torch.tensor(label), pred=pred[None], train_idx=list(range(G_n)), args=eargs,
                                 writer=None, print_training=False, graph_mode=True, graph_idx=0)
    _meta(out, name, 1, L, bn, att, hid, emb, opt, epochs, W, pred)
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
        gen_node_case(R, out, name, *c, seed=1100 + k)
    for k, (name, c) in enumerate(GRAPH_CASES.items()):
        gen_graph_case(R, out, name, *c, seed=1200 + k)
    np.savez_compressed(os.path.join(OUT, "deep_golden.npz"), **out)
    print("  deep golden written")


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen(ref_harness.load())
