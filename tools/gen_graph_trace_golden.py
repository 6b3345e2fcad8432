"""gen_graph_trace_golden.py -- tests/golden/graph_trace_golden.npz by EXECUTING THE UNMODIFIED REFERENCE.

What Explainer(print_training=True) prints every epoch in graph-classification mode (explain.py:137-159: loss, mask density,
softmax row), parsed from the reference's stdout, on the 12 graphs of golden/graphs_golden.npz (its model and its per-graph M0 seeds).
The printed loss sums size and entropy over all max_nodes^2 mask entries (explain.py:755-770), so it holds the off-edge part
gx_offedge_regularisers_graphs computes.  Three cases:
  a   default hyper-parameters, A_EPOCHS epochs, every graph;
  b   the loss coefficients size 0.05, entropy 0.3, feature size 0.2 (set H2 of tests/test_oracle_hparams.py; graph mode has no
      Laplacian term), B_EPOCHS epochs, graphs B_GIDS: the off-edge part scales with c_size and c_ent / max_nodes^2;
  c   unconstrained=True, C_EPOCHS epochs, graphs C_GIDS.
The reference has no setting for its loss coefficients (ExplainModule.__init__ fixes self.coeffs, explain.py:624-631): case b
updates that dict right after the reference's own constructor has run, and restores the constructor afterwards.  The epoch counts
stay short: dense trajectories of some graphs are chaotic at 100 epochs (DESIGN.md section 11).  M0 is not stored; tests redraw
it from the seed.  Needs the reference tree (oracle/ref_harness.py); deterministic:
    python tools/gen_graph_trace_golden.py

Keys: a_epochs / b_epochs / c_epochs, a_gids / b_gids / c_gids, b_size / b_ent / b_feat_size, and <case>_g<g> = float64
[epoch] (loss, mask density, softmax row) as printed.
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
import ref_harness  # noqa: E402
from gen_golden import OUT, train_args  # noqa: E402

A_EPOCHS = 30
B_EPOCHS, B_GIDS, B_COEFFS = 30, (0, 5, 9), dict(size=0.05, ent=0.3, feat_size=0.2)
C_EPOCHS, C_GIDS = 12, (1, 4, 7)
LINE = re.compile(r"epoch:\s+(\d+)\s+; loss:\s+(\S+)\s+; mask density:\s+(\S+)\s+; pred:\s+tensor\(\[([^\]]*)\]")


@contextlib.contextmanager
def coefficients(R, over):
    """ExplainModule instances built inside the block carry `over` in their coeffs dict."""
    init = R.explain.ExplainModule.__init__

    def patched(self, *a, **k):
        init(self, *a, **k)
        self.coeffs.update(over)
    R.explain.ExplainModule.__init__ = patched
    try:
        yield
    finally:
        R.explain.ExplainModule.__init__ = init


def printed(ex, g, seed, unconstrained, epochs):
    """Rows (loss, density, softmax row) the reference prints while it explains graph g."""
    buf = io.StringIO()
    torch.manual_seed(seed)
    with contextlib.redirect_stdout(buf):
        ex.explain(node_idx=0, graph_idx=g, graph_mode=True, unconstrained=unconstrained)
    rows = [[float(m.group(2)), float(m.group(3))] + [float(x) for x in m.group(4).replace("\n", " ").split(",")]
            for m in LINE.finditer(buf.getvalue())]
    assert len(rows) == epochs, (g, len(rows), buf.getvalue()[:300])
    return np.asarray(rows, np.float64)


def main():
    R = ref_harness.load()
    gg = np.load(os.path.join(OUT, "graphs_golden.npz"))
    G_n, d, C = int(gg["num_graphs"]), gg["feat"].shape[2], gg["Wp"].shape[0]
    adj, feat, label = gg["adj"].astype(np.float64), gg["feat"].astype(np.float32), gg["label"].astype(np.int64)
    model = R.models.GcnEncoderGraph(d, 20, 20, C, 3, bn=False, args=train_args(input_dim=d))
    model.load_state_dict({k: torch.tensor(gg[w]) for k, w in (("conv_first.weight", "W1"), ("conv_first.bias", "b1"),
                           ("conv_block.0.weight", "W2"), ("conv_block.0.bias", "b2"), ("conv_last.weight", "W3"),
                           ("conv_last.bias", "b3"), ("pred_model.weight", "Wp"), ("pred_model.bias", "bp"))})
    model.eval()
    with torch.no_grad():
        pred = np.stack([model(torch.tensor(feat[g:g + 1]), torch.tensor(adj[g:g + 1], dtype=torch.float))[0][0].numpy()
                         for g in range(G_n)])[None]

    def explainer(epochs):
        eargs = ref_harness.explainer_args(dataset="graph_trace", num_epochs=epochs)
        return R.explain.Explainer(model=model, adj=torch.tensor(adj, dtype=torch.float), feat=torch.tensor(feat),
                                   label=torch.tensor(label), pred=pred, train_idx=list(range(G_n)), args=eargs,
                                   writer=None, print_training=True, graph_mode=True, graph_idx=0)

    out = dict(a_epochs=np.int64(A_EPOCHS), b_epochs=np.int64(B_EPOCHS), c_epochs=np.int64(C_EPOCHS),
               a_gids=np.arange(G_n, dtype=np.int64), b_gids=np.asarray(B_GIDS, np.int64), c_gids=np.asarray(C_GIDS, np.int64),
               b_size=np.float64(B_COEFFS["size"]), b_ent=np.float64(B_COEFFS["ent"]), b_feat_size=np.float64(B_COEFFS["feat_size"]))
    seed = lambda g: int(gg["g%d_seed" % g])
    torch.set_printoptions(precision=8, sci_mode=False)
    try:
        ex = explainer(A_EPOCHS)
        for g in range(G_n):
            out["a_g%d" % g] = printed(ex, g, seed(g), False, A_EPOCHS)
        with coefficients(R, B_COEFFS):
            ex = explainer(B_EPOCHS)
            for g in B_GIDS:
                out["b_g%d" % g] = printed(ex, g, seed(g), False, B_EPOCHS)
        ex = explainer(C_EPOCHS)
        for g in C_GIDS:
            out["c_g%d" % g] = printed(ex, g, seed(g), True, C_EPOCHS)
    finally:
        torch.set_printoptions(profile="default")
    np.savez_compressed(os.path.join(OUT, "graph_trace_golden.npz"), **out)
    print("  graph trace golden written: %d + %d + %d graphs" % (G_n, len(B_GIDS), len(C_GIDS)))


if __name__ == "__main__":
    torch.set_num_threads(8)
    main()
