"""gen_head_golden.py -- tests/golden/head_golden.npz by EXECUTING THE UNMODIFIED REFERENCE on GCNs with an MLP prediction head
(GcnEncoderNode / GcnEncoderGraph(pred_hidden_dims=[..]), models.py:193-207).

The reference's models (reference init, biases redrawn from N(0, 0.3) so that they matter, then every parameter rounded to the nearest
float16 value so that the fixture stores each model in half the bytes), explained with Explainer.explain (model="exp"):
  * node mode on the rand fixture graph, 4 nodes each: head [50] with 3 layers at 30 and 100 epochs, [64, 32] with --bn, [50] with 2
    layers and SGD, an attention model (--method att) with [20], d = 300 random N(0, 1) features (float16-rounded) with [50];
  * graph mode on the 12 graphs of graphs_golden.npz: [50] with 3 layers, --bn with 4 layers and [32, 16];
  * unconstrained=True: node mode ([50], 3 layers, --bn) and graph mode ([32, 16], 4 layers).
Needs the reference tree (oracle/ref_harness.py); deterministic:
    python tools/gen_head_golden.py

Keys (masks at the sub-adjacency entries, row-major, float32; spreads float64):
  cases                                                   the case names
  <case>_mode / _L / _bn / _att / _hid / _emb / _opt / _epochs / _unc   node (0) or graph (1) mode, the model, the optimiser, the epochs,
                                                          unconstrained (1) or not
  <case>_head                                             the hidden head widths
  <case>_w_<W1 .. WL, b1 .., Wa1 .. (att), Wh1 .., bh1 .., Wp, bp>   the weights, float16 (exact); Wh<j> / bh<j> = pred_model.<2j-2>,
                                                          Wp / bp = the last Linear; torch's (out, in) layout for the head
  <case>_feat                                             node mode with d = 300 only: the features (float16, exact)
  <case>_pred                                             the model's forward on the rand graph (node mode) or on each padded graph
  <case>_nodes, <case>_n<node>_seed / _nbrs / _mask / _spread   node mode (M0 seeds: rand_golden.npz n<node>_seed)
  <case>_g<g>_mask / _spread                              graph mode (M0 seeds: graphs_golden.npz g<g>_seed)
  init_<state_dict key>, init_seed                        a GcnEncoderNode(10, 20, 20, 3, 3, pred_hidden_dims=[50, 7], bn=True) as the
                                                          reference constructs it under torch.manual_seed(init_seed) (float32)
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gnnx_oracle as O  # noqa: E402
import ref_harness  # noqa: E402
from gen_deep_golden import NODES, _spread  # noqa: E402
from gen_golden import OUT, train_args  # noqa: E402

# name: (L, bn, att, head widths, opt, epochs, d (None: the rand graph's features), unconstrained, seed)
NODE_CASES = {"rand_h50_e30": (3, False, False, [50], "adam", 30, None, False, 1500),
              "rand_h50_e100": (3, False, False, [50], "adam", 100, None, False, 1500),
              "rand_bn_h64_32": (3, True, False, [64, 32], "adam", 30, None, False, 1501),
              "rand_L2_h50_sgd": (2, False, False, [50], "sgd", 30, None, False, 1502),
              "rand_att_h20": (3, False, True, [20], "adam", 30, None, False, 1503),
              "rand_d300_h50": (3, False, False, [50], "adam", 30, 300, False, 1504),
              "rand_unc_bn_h50": (3, True, False, [50], "adam", 30, None, True, 1505)}
GRAPH_CASES = {"graphs_h50": (3, False, False, [50], "adam", 30, None, False, 1600),
               "graphs_bn_L4_h32_16": (4, True, False, [32, 16], "adam", 30, None, False, 1601),
               "graphs_unc_L4_h32_16": (4, False, False, [32, 16], "adam", 30, None, True, 1602)}
HID = EMB = 20
INIT_SEED = 1700


def _model(cls, d, C, L, bn, att, widths, seed):
    """The reference's model with pred_hidden_dims = widths, biases N(0, 0.3), every parameter rounded to float16; -> (model, weights)."""
    torch.manual_seed(seed)
    over = dict(method="att") if att else {}
    model = cls(d, HID, EMB, C, L, pred_hidden_dims=list(widths), bn=bn,
                args=train_args(input_dim=d, hidden_dim=HID, output_dim=EMB, num_gc_layers=L, bn=bn, **over))
    with torch.no_grad():
        for name, p_ in model.named_parameters():
            if name.endswith("bias"):
                p_.normal_(0.0, 0.3)
        for p_ in model.parameters():
            p_.copy_(p_.half().float())
    model.eval()
    sd = {k: v.numpy().astype(np.float32) for k, v in model.state_dict().items()}
    keys = ["conv_first"] + ["conv_block.%d" % i for i in range(L - 2)] + ["conv_last"]
    W = {}
    for l, k in enumerate(keys, 1):
        W["W%d" % l], W["b%d" % l] = sd[k + ".weight"], sd[k + ".bias"]
        if att:
            W["Wa%d" % l] = sd[k + ".att_weight"]
    for j in range(len(widths)):
        W["Wh%d" % (j + 1)], W["bh%d" % (j + 1)] = sd["pred_model.%d.weight" % (2 * j)], sd["pred_model.%d.bias" % (2 * j)]
    W["Wp"], W["bp"] = sd["pred_model.%d.weight" % (2 * len(widths))], sd["pred_model.%d.bias" % (2 * len(widths))]
    assert set(sd) == {k for k in sd if not k.startswith("pred_model")} | {"pred_model.%d.%s" % (2 * j, s) for j in range(len(widths) + 1)
                                                                            for s in ("weight", "bias")}
    return model, W


def _meta(out, name, mode, L, bn, att, widths, opt, epochs, unc, W, pred):
    for k, v in W.items():
        h = v.astype(np.float16)
        assert np.array_equal(h.astype(np.float32), v), k
        out["%s_w_%s" % (name, k)] = h
    out.update({name + "_mode": np.int64(mode), name + "_L": np.int64(L), name + "_bn": np.int64(bn), name + "_att": np.int64(att),
                name + "_hid": np.int64(HID), name + "_emb": np.int64(EMB), name + "_opt": np.str_(opt), name + "_epochs": np.int64(epochs),
                name + "_unc": np.int64(unc), name + "_head": np.asarray(widths, np.int64), name + "_pred": pred})


def gen_node_case(R, out, name, L, bn, att, widths, opt, epochs, d, unc, seed):
    g = np.load(os.path.join(OUT, "rand_graph.npz"))
    gold = np.load(os.path.join(OUT, "rand_golden.npz"))
    N, C = int(g["N"]), g["Wp"].shape[0]
    feat = g["feat"].astype(np.float32)
    if d is not None:
        feat = np.random.default_rng(seed).normal(size=(N, d)).astype(np.float16).astype(np.float32)
        out[name + "_feat"] = feat.astype(np.float16)
    adj = np.zeros((1, N, N)); e = g["edges"]; adj[0, e[:, 0], e[:, 1]] = 1; adj[0, e[:, 1], e[:, 0]] = 1
    model, W = _model(R.models.GcnEncoderNode, feat.shape[1], C, L, bn, att, widths, seed)
    with torch.no_grad():
        pred, _ = model(torch.tensor(feat[None]), torch.tensor(adj, dtype=torch.float))
    over = dict(method="att") if att else {}
    eargs = ref_harness.explainer_args(dataset="rand", num_epochs=epochs, num_gc_layers=L, bn=bn, opt=opt, hidden_dim=HID, output_dim=EMB,
                                       **over)
    with ref_harness.quiet():
        ex = R.explain.Explainer(model=model, adj=adj, feat=feat[None].astype(np.float64), label=g["label"][None], pred=pred.numpy(),
                                 train_idx=list(range(N)), args=eargs, writer=None, print_training=False, graph_idx=-1)
    _meta(out, name, 0, L, bn, att, widths, opt, epochs, unc, W, pred[0].numpy())
    out[name + "_nodes"] = np.asarray(NODES, np.int64)
    hp = O.default_hparams(num_epochs=epochs, opt=opt)
    for node in NODES:
        seed_n = int(gold["n%d_seed" % node])
        with ref_harness.quiet():
            idx, sub_adj, sub_feat, sub_label, nbrs = ex.extract_neighborhood(node, 0)
        M0 = O.draw_m0(len(nbrs), seed=seed_n)
        torch.manual_seed(seed_n)
        with ref_harness.quiet():
            masked = np.asarray(ex.explain(node, graph_idx=0, unconstrained=unc))
        ei, ej = np.nonzero(sub_adj)
        ref = masked[ei, ej]
        pl = np.argmax(pred[0].numpy()[nbrs], axis=1)
        gt = int(np.asarray(sub_label)[idx])
        A = np.asarray(sub_adj, np.float64)
        port = lambda M, dt: O.explain_dense_torch(A, np.asarray(sub_feat, np.float32), gt, pl, idx, W, M, hp, bn=bn, dtype=dt,
                                                   unconstrained=unc)
        key = "%s_n%d" % (name, node)
        out[key + "_seed"] = np.int64(seed_n)
        out[key + "_nbrs"] = np.asarray(nbrs, np.int32)
        out[key + "_mask"] = ref.astype(np.float32)
        out[key + "_spread"] = np.float64(_spread(port, M0, ref, ei, ej, node, key))
    print("  %s: spreads %s" % (name, ["%.1e" % out["%s_n%d_spread" % (name, v)] for v in NODES]), flush=True)


def gen_graph_case(R, out, name, L, bn, att, widths, opt, epochs, d, unc, seed):
    gg = np.load(os.path.join(OUT, "graphs_golden.npz"))
    G_n, n = int(gg["num_graphs"]), int(gg["max_nodes"])
    adj, feat, label = gg["adj"].astype(np.float64), gg["feat"].astype(np.float32), gg["label"].astype(np.int64)
    C = gg["Wp"].shape[0]
    model, W = _model(R.models.GcnEncoderGraph, feat.shape[2], C, L, bn, att, widths, seed)
    with torch.no_grad():
        pred = np.stack([model(torch.tensor(feat[g:g + 1]), torch.tensor(adj[g:g + 1], dtype=torch.float))[0][0].numpy()
                         for g in range(G_n)])
    eargs = ref_harness.explainer_args(dataset="graphs", num_epochs=epochs, num_gc_layers=L, bn=bn, opt=opt, hidden_dim=HID, output_dim=EMB)
    with ref_harness.quiet():
        ex = R.explain.Explainer(model=model, adj=torch.tensor(adj, dtype=torch.float), feat=torch.tensor(feat),
                                 label=torch.tensor(label), pred=pred[None], train_idx=list(range(G_n)), args=eargs,
                                 writer=None, print_training=False, graph_mode=True, graph_idx=0)
    _meta(out, name, 1, L, bn, att, widths, opt, epochs, unc, W, pred)
    hp = O.default_hparams(num_epochs=epochs, opt=opt)
    for g in range(G_n):
        seed_g = int(gg["g%d_seed" % g])
        M0 = O.draw_m0(n, seed=seed_g)
        torch.manual_seed(seed_g)
        with ref_harness.quiet():
            masked = np.asarray(ex.explain(node_idx=0, graph_idx=g, graph_mode=True, unconstrained=unc))
        ei, ej = np.nonzero(adj[g])
        ref = masked[ei, ej]
        port = lambda M, dt: O.explain_dense_torch(adj[g], feat[g], int(label[g]), None, 0, W, M, hp, graph_mode=True, bn=bn, dtype=dt,
                                              unconstrained=unc)
        out["%s_g%d_mask" % (name, g)] = ref.astype(np.float32)
        out["%s_g%d_spread" % (name, g)] = np.float64(_spread(port, M0, ref, ei, ej, 100 + g, "%s_g%d" % (name, g)))
    print("  %s: spreads %s" % (name, ["%.1e" % out["%s_g%d_spread" % (name, g)] for g in range(G_n)]), flush=True)


def gen(R):
    out = {"cases": np.asarray(list(NODE_CASES) + list(GRAPH_CASES))}
    torch.manual_seed(INIT_SEED)
    init = R.models.GcnEncoderNode(10, 20, 20, 3, 3, pred_hidden_dims=[50, 7], bn=True,
                                   args=train_args(input_dim=10, hidden_dim=20, output_dim=20, num_gc_layers=3, bn=True))
    out.update({"init_" + k: v.numpy().astype(np.float32) for k, v in init.state_dict().items()})
    out["init_seed"] = np.int64(INIT_SEED)
    for name, c in NODE_CASES.items():
        gen_node_case(R, out, name, *c)
    for name, c in GRAPH_CASES.items():
        gen_graph_case(R, out, name, *c)
    path = os.path.join(OUT, "head_golden.npz")
    np.savez_compressed(path, **out)
    print("  head golden written (%d bytes)" % os.path.getsize(path))


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen(ref_harness.load())
