"""gen_graph_grad_golden.py -- tests/golden/graph_grad_golden.npz: the gradient baseline in graph-classification mode, by EXECUTING THE
UNMODIFIED REFERENCE's ExplainModule.adj_feat_grad (explain.py:717-738, graph branch) on the 12 padded graphs of graphs_golden.npz.

The reference's Explainer.explain(0, graph_idx=g, graph_mode=True, model="grad") cannot produce this itself: explain.py:102 makes the
graph's predicted label a numpy scalar and explain.py:129 indexes it (pred_label[node_idx_new]), which raises
"IndexError: invalid index to scalar variable" for every graph (checked below on every graph); explain.py:130 would also index the
(1, n, n) gradient with graph_idx.  Its computation is sound, so this script builds the ExplainModule exactly as explain.py:97-119 does,
calls adj_feat_grad(0, argmax(pred[0][g])) and applies explain.py:128-133 with batch entry 0:
    sigmoid(|dL/dA| + |dL/dA|^T) * adj.
Needs the reference tree (oracle/ref_harness.py); deterministic:
    python tools/gen_graph_grad_golden.py

Models:
  base     the GcnEncoderGraph(14, 20, 20, 2, 3) of graphs_golden.npz, its stored pred
  scaled   a GcnEncoderGraph(14, 20, 20, 3, 3) as the reference initialises it under torch.manual_seed(SCALED_SEED), pred_model's
           weight times PRED_SCALE, biases N(0, 0.1), every parameter rounded to the nearest float16 value.  A freshly initialised model
           gives masks of 0.500-0.505; the layers normalise their outputs, so only pred_model's scale moves the gradient, and this one
           spreads the masks over more than 0.1 with all three classes predicted
Keys (masks at the adjacency entries of the graph in row-major order, float32 -- the reference's float32 sigmoid):
  models                                         the model names
  <m>_w_<W1 b1 W2 b2 W3 b3 Wp bp>                the weights (float32; scaled: float16-exact)
  <m>_pred                                       (1, G, C) the model's forward on every padded graph (the Explainer's pred)
  <m>_g<g>_label, <m>_g<g>_mask                  argmax(pred[0][g]) and the mask at that label
  <m>_g<g>_alt_label, <m>_g<g>_alt_mask          the same at a label the model does not predict ((label + 1) % C)
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_harness  # noqa: E402
from gen_golden import OUT, state_to_np, train_args  # noqa: E402

SCALED_SEED, PRED_SCALE = 1803, 16.0
WKEYS = ("W1", "b1", "W2", "b2", "W3", "b3", "Wp", "bp")
SD_KEYS = (("conv_first.weight", "W1"), ("conv_first.bias", "b1"), ("conv_block.0.weight", "W2"), ("conv_block.0.bias", "b2"),
           ("conv_last.weight", "W3"), ("conv_last.bias", "b3"), ("pred_model.weight", "Wp"), ("pred_model.bias", "bp"))


def _models(R, gg):
    d = gg["feat"].shape[2]
    base = R.models.GcnEncoderGraph(d, 20, 20, 2, 3, bn=False, args=train_args(input_dim=d))
    base.load_state_dict({k: torch.tensor(gg[w]) for k, w in SD_KEYS})
    torch.manual_seed(SCALED_SEED)
    scaled = R.models.GcnEncoderGraph(d, 20, 20, 3, 3, bn=False, args=train_args(input_dim=d, num_classes=3))
    with torch.no_grad():
        for name, p_ in scaled.named_parameters():
            if name.endswith("bias"):
                p_.normal_(0.0, 0.1)
            elif name == "pred_model.weight":
                p_.mul_(PRED_SCALE)
        for p_ in scaled.parameters():
            p_.copy_(p_.half().float())
    return [("base", base, gg["pred"]), ("scaled", scaled, None)]


def _grad_mask(R, model, adj_g, feat_g, label_g, pred_label):
    """explain.py:97-119 (ExplainModule as explain() builds it) + :125-133 with batch entry 0."""
    eargs = ref_harness.explainer_args(dataset="graphs", graph_mode=True)
    adj = torch.tensor(adj_g[None], dtype=torch.float)
    x = torch.tensor(feat_g[None], requires_grad=True, dtype=torch.float)
    label = torch.tensor(np.asarray(label_g), dtype=torch.long)
    explainer = R.explain.ExplainModule(adj=adj, x=x, model=model, label=label, args=eargs, writer=None, graph_idx=0, graph_mode=True)
    model.eval()
    explainer.zero_grad()
    adj_grad = torch.abs(explainer.adj_feat_grad(0, pred_label)[0])[0]
    masked = torch.sigmoid(adj_grad + adj_grad.t())
    return masked.cpu().detach().numpy() * adj_g


def main():
    R = ref_harness.load()
    gg = np.load(os.path.join(OUT, "graphs_golden.npz"))
    adj, feat, label = gg["adj"].astype(np.float64), gg["feat"].astype(np.float64), gg["label"]
    G = int(gg["num_graphs"])
    out = dict(models=np.asarray(["base", "scaled"]))
    for name, model, pred in _models(R, gg):
        model.eval()
        if pred is None:
            with torch.no_grad():
                pred = np.stack([model(torch.tensor(feat[g:g + 1], dtype=torch.float), torch.tensor(adj[g:g + 1], dtype=torch.float))[0][0].numpy()
                                 for g in range(G)])[None].astype(np.float32)
        W = {w: v for w, v in state_to_np(model).items() if w in WKEYS}
        for k, v in W.items():
            if name == "scaled":
                assert np.array_equal(v.astype(np.float16).astype(np.float32), v), k
            out["%s_w_%s" % (name, k)] = v
        out[name + "_pred"] = pred
        C = pred.shape[2]
        # the unmodified explain() on this path: IndexError on the scalar predicted label (explain.py:129), every graph
        eargs = ref_harness.explainer_args(dataset="graphs")
        with ref_harness.quiet():
            ex = R.explain.Explainer(model=model, adj=torch.tensor(adj, dtype=torch.float), feat=torch.tensor(feat, dtype=torch.float),
                                     label=torch.tensor(label), pred=pred, train_idx=list(range(G)), args=eargs, writer=None,
                                     print_training=False, graph_mode=True, graph_idx=0)
            for g in range(G):
                try:
                    ex.explain(node_idx=0, graph_idx=g, graph_mode=True, model="grad")
                    raise AssertionError("the reference's explain(model='grad') ran in graph mode")
                except IndexError:
                    pass
        rng_state = torch.get_rng_state()
        for g in range(G):
            rows, cols = np.nonzero(adj[g])
            pl = int(np.argmax(pred[0][g], axis=0))                                    # explain.py:102
            alt = (pl + 1) % C
            for key, lab in (("", pl), ("alt_", alt)):
                m = _grad_mask(R, model, adj[g], feat[g], label[g], lab)
                assert not m[adj[g] == 0].any()
                out["%s_g%d_%slabel" % (name, g, key)] = np.int64(lab)
                out["%s_g%d_%smask" % (name, g, key)] = m[rows, cols].astype(np.float32)
        torch.set_rng_state(rng_state)
        vals = np.concatenate([out["%s_g%d_mask" % (name, g)] for g in range(G)])
        print("%s: C=%d labels %s, masks in [%.4f, %.4f]" % (name, C, [int(out["%s_g%d_label" % (name, g)]) for g in range(G)],
                                                             vals.min(), vals.max()))
    path = os.path.join(OUT, "graph_grad_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path)


if __name__ == "__main__":
    main()
