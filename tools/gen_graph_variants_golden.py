"""gen_graph_variants_golden.py -- tests/golden/graph_variants_golden.npz by EXECUTING THE UNMODIFIED REFERENCE.

Graph-classification mode with the model and optimiser variants, on the graphs, features, labels and seeds of
tests/golden/graphs_golden.npz.  Needs the reference tree (oracle/ref_harness.py); deterministic:
    python tools/gen_graph_variants_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_harness  # noqa: E402
from gen_golden import OUT, train_args  # noqa: E402


GRAPH_MODEL_VARIANTS = (("L2", 2, False, 20, 20), ("L4", 4, False, 20, 20), ("bn", 3, True, 20, 20), ("bn_L4", 4, True, 20, 20),
                        ("wide", 3, True, 64, 48))
GRAPH_OPT_VARIANTS = (("sgd", dict(opt="sgd")), ("rmsprop", dict(opt="rmsprop")), ("adagrad", dict(opt="adagrad")),
                      ("sgdstep", dict(opt="sgd", opt_scheduler="step", opt_decay_step=10, opt_decay_rate=0.3)))


def gen_graph_variants(R, epochs=30, nudges=4):
    """Graph-classification mode with the model and optimiser variants (explainer_main.py:209-219 passes --num-gc-layers, --bn,
    --hidden-dim, --output-dim to GcnEncoderGraph; utils/train_utils.py:7-23 serves both modes): the unmodified reference's
    Explainer(graph_mode=True) on the graphs, features, labels and seeds of graphs_golden.npz, 30 epochs ->
    tests/golden/graph_variants_golden.npz.
      * model variants (random weights, non-zero biases): <tag>_W<l> / _b<l> / _Wp / _bp, <tag>_L, <tag>_bn
      * optimisers on graphs_golden's default model: sgd / rmsprop / adagrad / sgd + StepLR
      * per graph g: <tag>_g<g>_mask (the returned mask at the edges, row-major) and <tag>_spread[g]: how far the line-by-line port
        moves from the reference's mask when every M0 entry is nudged by +-1 ulp (the reproducibility of the reference itself)
    The port (gnnx_oracle.explain_dense_torch) must reproduce every reference mask to below 1e-6."""
    import gnnx_oracle as O
    gg = np.load(os.path.join(OUT, "graphs_golden.npz"))
    G_n, n, d, C = int(gg["num_graphs"]), int(gg["max_nodes"]), gg["feat"].shape[2], gg["Wp"].shape[0]
    adj, feat, label = gg["adj"].astype(np.float64), gg["feat"].astype(np.float32), gg["label"].astype(np.int64)
    out = dict(num_epochs=np.int64(epochs))
    runs = []
    for tag, L, bn, hid, emb in GRAPH_MODEL_VARIANTS:
        torch.manual_seed(200 + 10 * L + int(bn) + hid)
        model = R.models.GcnEncoderGraph(d, hid, emb, C, L, bn=bn, args=train_args(input_dim=d, num_gc_layers=L, bn=bn))
        with torch.no_grad():
            for name, p_ in model.named_parameters():
                if name.endswith("bias"):
                    p_.normal_(0.0, 0.3)
        runs.append((tag, model, L, bn, hid, emb, {}))
    base = R.models.GcnEncoderGraph(d, 20, 20, C, 3, bn=False, args=train_args(input_dim=d))
    base.load_state_dict({k: torch.tensor(gg[w]) for k, w in (("conv_first.weight", "W1"), ("conv_first.bias", "b1"),
                          ("conv_block.0.weight", "W2"), ("conv_block.0.bias", "b2"), ("conv_last.weight", "W3"),
                          ("conv_last.bias", "b3"), ("pred_model.weight", "Wp"), ("pred_model.bias", "bp"))})
    for tag, over in GRAPH_OPT_VARIANTS:
        runs.append((tag, base, 3, False, 20, 20, over))
    for tag, model, L, bn, hid, emb, over in runs:
        model.eval()
        sd = model.state_dict()
        keys = ["conv_first"] + ["conv_block.%d" % i for i in range(L - 2)] + ["conv_last"]
        W = {}
        for l, k in enumerate(keys, 1):
            W["W%d" % l] = sd[k + ".weight"].numpy().astype(np.float32)
            W["b%d" % l] = sd[k + ".bias"].numpy().astype(np.float32)
        W["Wp"] = sd["pred_model.weight"].numpy().astype(np.float32)
        W["bp"] = sd["pred_model.bias"].numpy().astype(np.float32)
        if not over:
            out.update({"%s_%s" % (tag, k): v for k, v in W.items()})
            out.update({tag + "_L": np.int64(L), tag + "_bn": np.int64(bn)})
        with torch.no_grad():
            pred = np.stack([model(torch.tensor(feat[g:g + 1]), torch.tensor(adj[g:g + 1], dtype=torch.float))[0][0].numpy()
                             for g in range(G_n)])[None]
        eargs = ref_harness.explainer_args(dataset="graphvar", num_epochs=epochs, num_gc_layers=L, bn=bn, hidden_dim=hid, output_dim=emb,
                                           **over)
        with ref_harness.quiet():
            ex = R.explain.Explainer(model=model, adj=torch.tensor(adj, dtype=torch.float), feat=torch.tensor(feat),
                                     label=torch.tensor(label), pred=pred, train_idx=list(range(G_n)), args=eargs,
                                     writer=None, print_training=False, graph_mode=True, graph_idx=0)
        hp = O.default_hparams(num_epochs=epochs, **over)
        spread = np.zeros(G_n)
        for g in range(G_n):
            seed = int(gg["g%d_seed" % g])
            M0 = O.draw_m0(n, seed=seed)
            ei, ej = np.nonzero(adj[g])
            assert np.array_equal(M0[ei, ej], gg["g%d_m0" % g])
            torch.manual_seed(seed)
            with ref_harness.quiet():
                masked = np.asarray(ex.explain(node_idx=0, graph_idx=g, graph_mode=True))
            off = masked.copy(); off[ei, ej] = 0
            assert np.all(off == 0)
            ref = masked[ei, ej]
            out["%s_g%d_mask" % (tag, g)] = ref.astype(np.float32)
            mine = O.explain_dense_torch(adj[g], feat[g], int(label[g]), None, 0, W, M0, hp=hp, graph_mode=True, bn=bn)
            err = O.rel_l2(mine[ei, ej], ref)
            assert err < 1e-6, (tag, g, err)
            for s in range(nudges):
                rng = np.random.default_rng(1000 * s + g)
                up = rng.integers(0, 2, M0.shape).astype(bool)
                Mn = np.where(up, np.nextafter(M0, np.float32(np.inf)), np.nextafter(M0, np.float32(-np.inf))).astype(np.float32)
                res = O.explain_dense_torch(adj[g], feat[g], int(label[g]), None, 0, W, Mn, hp=hp, graph_mode=True, bn=bn)
                spread[g] = max(spread[g], O.rel_l2(res[ei, ej], ref))
        out[tag + "_spread"] = spread
        print("  %s: %d graphs, spread > 3e-5: %s" % (tag, G_n, {g: "%.1e" % s for g, s in enumerate(spread) if s > 3e-5}), flush=True)
    np.savez_compressed(os.path.join(OUT, "graph_variants_golden.npz"), **out)
    print("  graph-mode variants golden written")


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_graph_variants(ref_harness.load())
