"""gen_hparams_golden.py -- tests/golden/hparams_golden.npz by EXECUTING THE UNMODIFIED REFERENCE.

The learning rate, the epoch count and the Adam schedulers, off the defaults, through the reference's own CLI settings (--lr, --epochs,
--opt-scheduler step / cos with --opt-decay-step, --opt-decay-rate, --opt-restart), in node mode (the rand and syn4 fixtures and the
reproducible syn1 nodes of golden/syn1_sens.npz) and graph mode (the 12 graphs of golden/graphs_golden.npz).  Needs the reference tree
(oracle/ref_harness.py); deterministic:
    python tools/gen_hparams_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_harness  # noqa: E402
from gen_golden import OUT, _load_fixture_model, train_args  # noqa: E402

# tag -> (epochs, reference settings); the step boundaries fall at epochs 6, 12, 18, 24; the cosine reaches lr = 0 at epoch 8 and
# rises again to lr at epoch 16 (CosineAnnealingLR is periodic in 2 T_max)
CASES = (("lr001", 30, dict(lr=0.01)), ("lr05", 30, dict(lr=0.5)), ("e2", 2, {}), ("e300", 300, dict(lr=0.01)),
         ("step", 30, dict(opt_scheduler="step", opt_decay_step=6, opt_decay_rate=0.5)),
         ("cos", 30, dict(opt_scheduler="cos", opt_restart=8)))
NODES = dict(rand=[0, 1, 7, 33, 77, 100, 149], syn4=[0, 1, 8, 164, 404, 511, 870], syn1=[0, 5, 300, 350, 400, 620])
NUDGES = 4


def case_hparams(epochs, over):
    import gnnx_oracle as O
    return O.default_hparams(num_epochs=epochs, **over)


def _spread(run, M0, ei, ej, ref, salt):
    """How far the port moves from the reference's mask when every M0 entry is nudged by +-1 ulp."""
    import gnnx_oracle as O
    worst = 0.0
    for s in range(NUDGES):
        rng = np.random.default_rng(1000 * s + salt)
        up = rng.integers(0, 2, M0.shape).astype(bool)
        Mn = np.where(up, np.nextafter(M0, np.float32(np.inf)), np.nextafter(M0, np.float32(-np.inf))).astype(np.float32)
        worst = max(worst, O.rel_l2(run(Mn)[ei, ej], ref))
    return worst


def gen_nodes(R, out):
    import gnnx_oracle as O
    for which, nodes in NODES.items():
        out[which + "_nodes"] = np.asarray(nodes, np.int64)
        for tag, epochs, over in CASES:
            make, g, gold = _load_fixture_model(R, which, num_epochs=epochs, **over)
            ex = make()
            W = {k: g[k] for k in ["W1", "b1", "W2", "b2", "W3", "b3", "Wp", "bp"]}
            hp = case_hparams(epochs, over)
            kept, spread = [], []
            for node in nodes:
                seed = int(gold["n%d_seed" % node])
                torch.manual_seed(seed)
                with ref_harness.quiet():
                    idx, sub_adj, sub_feat, sub_label, nbrs = ex.extract_neighborhood(node, 0)
                    masked = np.asarray(ex.explain(node, graph_idx=0))
                ei, ej = np.nonzero(sub_adj)
                ref = masked[ei, ej]
                if not np.isfinite(ref).all():      # the reference's entropy term is NaN once sigmoid(M) rounds to 1
                    print("  %s %s n%d: the reference returns NaN, case dropped" % (which, tag, node))
                    continue
                M0 = np.ones(sub_adj.shape, np.float32); M0[ei, ej] = gold["n%d_m0" % node]
                pl = np.argmax(g["pred"][nbrs], 1)
                run = lambda M: O.explain_dense_torch(sub_adj, sub_feat, int(g["label"][node]), pl, idx, W, M, hp=hp)
                err = O.rel_l2(run(M0)[ei, ej], ref)
                assert err < 1e-6, (which, tag, node, err)
                out["%s_%s_n%d_mask" % (which, tag, node)] = ref.astype(np.float32)
                kept.append(node)
                spread.append(_spread(run, M0, ei, ej, ref, node))
            out["%s_%s_nodes" % (which, tag)] = np.asarray(kept, np.int64)
            out["%s_%s_spread" % (which, tag)] = np.asarray(spread)
            print("  %s %s: %d nodes, largest spread %.1e" % (which, tag, len(kept), max(spread)), flush=True)


def gen_graphs(R, out):
    import gnnx_oracle as O
    gg = np.load(os.path.join(OUT, "graphs_golden.npz"))
    G_n, n, d, C = int(gg["num_graphs"]), int(gg["max_nodes"]), gg["feat"].shape[2], gg["Wp"].shape[0]
    adj, feat, label = gg["adj"].astype(np.float64), gg["feat"].astype(np.float32), gg["label"].astype(np.int64)
    model = R.models.GcnEncoderGraph(d, 20, 20, C, 3, bn=False, args=train_args(input_dim=d))
    model.load_state_dict({k: torch.tensor(gg[w]) for k, w in (("conv_first.weight", "W1"), ("conv_first.bias", "b1"),
                           ("conv_block.0.weight", "W2"), ("conv_block.0.bias", "b2"), ("conv_last.weight", "W3"),
                           ("conv_last.bias", "b3"), ("pred_model.weight", "Wp"), ("pred_model.bias", "bp"))})
    model.eval()
    W = {k: gg[k] for k in ["W1", "b1", "W2", "b2", "W3", "b3", "Wp", "bp"]}
    with torch.no_grad():
        pred = np.stack([model(torch.tensor(feat[g:g + 1]), torch.tensor(adj[g:g + 1], dtype=torch.float))[0][0].numpy()
                         for g in range(G_n)])[None]
    for tag, epochs, over in CASES:
        eargs = ref_harness.explainer_args(dataset="hparams", num_epochs=epochs, **over)
        with ref_harness.quiet():
            ex = R.explain.Explainer(model=model, adj=torch.tensor(adj, dtype=torch.float), feat=torch.tensor(feat),
                                     label=torch.tensor(label), pred=pred, train_idx=list(range(G_n)), args=eargs,
                                     writer=None, print_training=False, graph_mode=True, graph_idx=0)
        hp = case_hparams(epochs, over)
        kept, spread = [], []
        for g in range(G_n):
            seed = int(gg["g%d_seed" % g])
            M0 = O.draw_m0(n, seed=seed)
            ei, ej = np.nonzero(adj[g])
            assert np.array_equal(M0[ei, ej], gg["g%d_m0" % g])
            torch.manual_seed(seed)
            with ref_harness.quiet():
                masked = np.asarray(ex.explain(node_idx=0, graph_idx=g, graph_mode=True))
            ref = masked[ei, ej]
            if not np.isfinite(ref).all():
                print("  graphs %s g%d: the reference returns NaN, case dropped" % (tag, g))
                continue
            run = lambda M: O.explain_dense_torch(adj[g], feat[g], int(label[g]), None, 0, W, M, hp=hp, graph_mode=True)
            err = O.rel_l2(run(M0)[ei, ej], ref)
            assert err < 1e-6, (tag, g, err)
            out["graphs_%s_g%d_mask" % (tag, g)] = ref.astype(np.float32)
            kept.append(g)
            spread.append(_spread(run, M0, ei, ej, ref, g))
        out["graphs_%s_gids" % tag] = np.asarray(kept, np.int64)
        out["graphs_%s_spread" % tag] = np.asarray(spread)
        print("  graphs %s: %d graphs, largest spread %.1e" % (tag, len(kept), max(spread)), flush=True)


def main():
    """case_* = the settings of every case, in CASES order.  Per case <tag>: <fixture>_<tag>_nodes / graphs_<tag>_gids (the cases kept: the reference
    returned a finite mask), <fixture>_<tag>_n<node>_mask / graphs_<tag>_g<g>_mask (the reference's mask at the sub-adjacency's edges,
    row-major; M0 and its seed are the fixture's, golden/<fixture>_golden.npz and graphs_golden.npz) and <...>_<tag>_spread (how far the
    line-by-line port moves from it when every M0 entry is nudged by +-1 ulp).  The port (gnnx_oracle.explain_dense_torch) must
    reproduce every reference mask to below 1e-6."""
    R = ref_harness.load()
    hps = [case_hparams(e, over) for _, e, over in CASES]
    out = dict(case_tags=np.array([c[0] for c in CASES]), case_epochs=np.array([c[1] for c in CASES], np.int64),
               case_lr=np.array([h.lr for h in hps]), case_scheduler=np.array([h.opt_scheduler for h in hps]),
               case_decay_step=np.array([h.opt_decay_step for h in hps], np.int64), case_decay_rate=np.array([h.opt_decay_rate for h in hps]),
               case_restart=np.array([h.opt_restart for h in hps], np.int64))
    gen_nodes(R, out)
    gen_graphs(R, out)
    np.savez_compressed(os.path.join(OUT, "hparams_golden.npz"), **out)
    print("  hyper-parameter golden written")


if __name__ == "__main__":
    torch.set_num_threads(8)
    main()
