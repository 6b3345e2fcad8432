#!/usr/bin/env python
"""Small invocation of every kernel for compute-sanitizer (racecheck / memcheck / synccheck are ~100x slower than a plain run):
    compute-sanitizer --tool racecheck python tools/sanitize_run.py
k-hop extraction + shared-memory kernel on a mix of task sizes (syn1: hub node 0 and tiny tasks), the streaming kernel (forced),
the gradient baseline, graph mode, densify, the off-edge regulariser sums of graph mode, neighbourhood rows, the unconstrained (dense) kernel, attention models, inputs wider than 128
features (explain_var.cu's wide path), models with 5 to 7 layers, graph-mode sharding's densify (dist_graphs), top-k delivery in global ids
(topk: gx_denoise_topk_edges with host and device buffers, and one Explainer.explain_nodes_topk call).  A few epochs each."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in ("gnn-model-explainer_b200", "oracle", "tests"):
    sys.path.insert(0, os.path.join(ROOT, p))
import util  # noqa: E402
import gnnx  # noqa: E402
from gnnx import _abi  # noqa: E402

EPOCHS = int(os.environ.get("SAN_EPOCHS", "4"))


def main():
    which = sys.argv[1:] or ["node", "stream", "graph", "misc", "var", "cluster", "dense", "att", "wide", "dist_graphs", "topk"]
    fx = util.load_fixture("syn1")
    if "node" in which:
        eng = util.make_engine(fx)
        nodes = [0, 3, 300, 301, 683, 699, 13, 550]
        plan = eng.plan_nodes(nodes, 3)
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_host(eng.make_hparams(num_epochs=EPOCHS), util.golden_m0(fx, plan), out)
        eng.explain_nodes_host(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=3), None, out)
        eng.grad_nodes_host(out)
        print("node ok", float(out.sum()))
        eng.close()
    if "stream" in which:
        fr = util.load_fixture("rand")
        for gang in (0, 3, -1):          # explain_gang.cu (automatic gang size, 3 CTAs per task) and explain_stream.cu
            eng = util.make_engine(fr)
            eng.debug_force_stream(True)
            eng.debug_gang(gang)
            plan = eng.plan_nodes(fr.nodes[:4], 3)
            out = np.zeros(plan.total_edges, np.float32)
            eng.explain_nodes_host(eng.make_hparams(num_epochs=EPOCHS), util.golden_m0(fr, plan), out)
            eng.grad_nodes_host(out)
            print("stream ok (gang %d)" % gang, float(out.sum()))
            eng.close()
    if "var" in which:
        g = np.load(util.GOLDEN + "/variants_golden.npz")
        import gnnx_oracle as O
        N = int(g["N"])
        rowptr, col = O.csr_from_edges(N, g["edges"])
        for tag, L, bn in (("bn", 3, True), ("L4", 4, False)):
            w = {k[len(tag) + 1:]: g[k] for k in g.files if k.startswith(tag + "_W") or k.startswith(tag + "_b")}
            eng = gnnx.Engine(0)
            eng.set_model(w, num_layers=L, bn=bn)
            eng.set_graph_csr(rowptr, col, g["feat"].astype(np.float32), g["label"].astype(np.int32), np.argmax(g[tag + "_pred"], 1).astype(np.int32))
            plan = eng.plan_nodes([0, 17], L)
            out = np.zeros(plan.total_edges, np.float32)
            eng.explain_nodes_host(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=2), None, out)
            print("var ok", tag, float(out.sum()))
            eng.close()
        rng = np.random.default_rng(5)   # a wide model (hidden 64 / output 48): two lane chunks per row
        sc = lambda *s_: (rng.normal(size=s_) * 0.4).astype(np.float32)
        d0 = g["feat"].shape[1]
        ww = dict(W1=sc(d0, 64), b1=sc(64), W2=sc(64, 64), b2=sc(64), W3=sc(64, 48), b3=sc(48), Wp=sc(3, 176), bp=sc(3))
        eng = gnnx.Engine(0)
        eng.set_model(ww, num_layers=3, bn=False)
        eng.set_graph_csr(rowptr, col, g["feat"].astype(np.float32), g["label"].astype(np.int32), np.zeros(N, np.int32))
        plan = eng.plan_nodes([0, 17], 3)
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_host(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=2), None, out)
        print("var ok wide", float(out.sum()))
        eng.close()
        eng = util.make_engine(fx)     # default model, optimiser other than Adam -> the variant kernel
        plan = eng.plan_nodes([300, 5], 3)
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_host(eng.make_hparams(num_epochs=EPOCHS, opt=1), util.golden_m0(fx, plan), out)
        print("var ok sgd", float(out.sum()))
        eng.close()
        gg = np.load(util.GOLDEN + "/graphs_golden.npz")   # graph mode: the default model with SGD -> the variant kernel
        eng = gnnx.Engine(0)
        eng.set_model({k: gg[k] for k in util.WKEYS})
        eng.set_graph_batch(gg["adj"], gg["feat"], gg["label"])
        eoff = eng.plan_graphs([0, 3, 5])
        out = np.zeros(int(eoff[-1]), np.float32)
        eng.explain_graphs_host(eng.make_hparams(num_epochs=EPOCHS, opt=1, init=_abi.GX_INIT_PHILOX, seed=3), None, out)
        print("var ok graph sgd", float(out.sum()))
        eng.close()
        # deep models (num_gc_layers 5 .. 7): L = 7 with --bn and widths 128 (conv weights and pred_model through L2), L = 5 attention,
        # node mode (hub and small tasks, 7 hops) and graph mode, the model forward with 128-float rows, the unconstrained kernel at L = 7
        for L, hid, bn, att in ((7, 128, True, False), (5, 20, False, True), (6, 64, False, False)):
            dims = [d0] + [hid] * L
            w = {}
            for l in range(1, L + 1):
                w["W%d" % l] = sc(dims[l - 1], dims[l]); w["b%d" % l] = sc(dims[l])
                if att:
                    w["Wa%d" % l] = sc(dims[l - 1], dims[l - 1])
            w["Wp"], w["bp"] = sc(3, hid * L), sc(3)
            attw = [w["Wa%d" % l] for l in range(1, L + 1)] if att else None
            eng = gnnx.Engine(0)
            eng.set_model(w, num_layers=L, bn=bn, att=attw)
            eng.set_graph_csr(rowptr, col, g["feat"].astype(np.float32), g["label"].astype(np.int32), np.zeros(N, np.int32))
            plan = eng.plan_nodes([0, 17], L)
            out = np.zeros(plan.total_edges, np.float32)
            eng.explain_nodes_host(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=2), None, out)
            pred = eng.model_forward()
            if not att:
                eng.explain_nodes_unconstrained(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=4), None, out)
            print("var ok deep node", L, hid, bn, att, float(out.sum()), float(pred.sum()))
            eng.close()
            wg = dict(w)
            wg["W1"] = sc(gg["feat"].shape[2], hid)
            if att:
                wg["Wa1"] = sc(gg["feat"].shape[2], gg["feat"].shape[2]); attw[0] = wg["Wa1"]
            eng = gnnx.Engine(0)
            eng.set_model(wg, num_layers=L, bn=bn, att=attw)
            eng.set_graph_batch(gg["adj"], gg["feat"], gg["label"] % 3)
            eoff = eng.plan_graphs([0, 3, 5])
            out = np.zeros(int(eoff[-1]), np.float32)
            eng.explain_graphs_host(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=3), None, out)
            print("var ok deep graph", L, hid, bn, att, float(out.sum()))
            eng.close()
        # hidden / output widths 129 .. 256 (explain_var.cu's row-block path): 256 / 256 with --bn, 160 / 136 on the wide input path
        # (d = 300), node mode (hub and small tasks) with the model forward, and graph mode
        for L, hid, emb, bn, d in ((3, 256, 256, True, d0), (4, 160, 136, False, 300)):
            dims = [d] + [hid] * (L - 1) + [emb]
            w = {}
            for l in range(1, L + 1):
                w["W%d" % l] = sc(dims[l - 1], dims[l]) / np.sqrt(dims[l - 1]); w["b%d" % l] = sc(dims[l])
            w["Wp"], w["bp"] = sc(3, hid * (L - 1) + emb), sc(3)
            feat = g["feat"].astype(np.float32) if d == d0 else rng.normal(size=(N, d)).astype(np.float32)
            eng = gnnx.Engine(0)
            eng.set_model(w, num_layers=L, bn=bn)
            eng.set_graph_csr(rowptr, col, feat, g["label"].astype(np.int32), np.zeros(N, np.int32))
            plan = eng.plan_nodes([0, 17], L)
            out = np.zeros(plan.total_edges, np.float32)
            eng.explain_nodes_host(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=2), None, out)
            pred = eng.model_forward()
            print("var ok wide layers node", L, hid, emb, bn, d, float(out.sum()), float(pred.sum()))
            eng.close()
            wg = dict(w)
            wg["W1"] = sc(gg["feat"].shape[2], hid)
            eng = gnnx.Engine(0)
            eng.set_model(wg, num_layers=L, bn=bn)
            eng.set_graph_batch(gg["adj"], gg["feat"], gg["label"] % 3)
            eoff = eng.plan_graphs([0, 3, 5])
            out = np.zeros(int(eoff[-1]), np.float32)
            eng.explain_graphs_host(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=3), None, out)
            print("var ok wide layers graph", L, hid, emb, bn, float(out.sum()))
            eng.close()
    if "cluster" in which:
        eng = util.make_engine(fx)
        eng.debug_cluster(4, 1)
        plan = eng.plan_nodes([0, 300, 13], 3)
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_host(eng.make_hparams(num_epochs=EPOCHS), util.golden_m0(fx, plan), out)
        print("cluster ok", float(out.sum()))
        eng.close()
    if "graph" in which:
        g = np.load(util.GOLDEN + "/graphs_golden.npz")
        eng = gnnx.Engine(0)
        eng.set_model({k: g[k] for k in util.WKEYS})
        eng.set_graph_batch(g["adj"], g["feat"], g["label"])
        gids = [0, 3, 5, 11]
        eoff = eng.plan_graphs(gids)
        m0 = np.concatenate([g["g%d_m0" % i] for i in gids]).astype(np.float32)
        out = np.zeros(int(eoff[-1]), np.float32)
        eng.explain_graphs_host(eng.make_hparams(num_epochs=EPOCHS), m0, out)
        print("graph ok", float(out.sum()))
        eng.close()
    if "dense" in which:   # explain_dense.cu: node mode with a trace, a --bn 4-layer model with SGD, graph mode
        import gnnx_oracle as O
        eng = util.make_engine(fx)
        plan = eng.plan_nodes([300, 5, 13], 3)
        n_t = [plan.n(t) for t in range(plan.count)]
        m0 = np.concatenate([O.draw_m0(n, seed=n).reshape(-1) for n in n_t])
        out = np.zeros(plan.total_edges, np.float32)
        md = np.zeros(sum(n * n for n in n_t), np.float32)
        tr = np.zeros((plan.count, EPOCHS, _abi.GX_TRACE_COLS), np.float32)
        tp = np.zeros((plan.count, EPOCHS, eng.num_classes), np.float32)
        eng.explain_nodes_unconstrained(eng.make_hparams(num_epochs=EPOCHS), m0, out, md, tr, tp)
        print("dense ok node", float(out.sum()), float(tr.sum()))
        eng.close()
        rng = np.random.default_rng(6)
        sc = lambda *s_: (rng.normal(size=s_) * 0.4).astype(np.float32)
        d0 = fx.feat.shape[1]
        C0 = fx.weights["Wp"].shape[0]
        w4 = dict(W1=sc(d0, 40), b1=sc(40), W2=sc(40, 40), b2=sc(40), W3=sc(40, 40), b3=sc(40), W4=sc(40, 24), b4=sc(24), Wp=sc(C0, 144), bp=sc(C0))
        eng = gnnx.Engine(0)
        eng.set_model(w4, num_layers=4, bn=True)
        eng.set_graph_csr(fx.rowptr, fx.col, fx.feat, fx.label, fx.pred_label)
        plan = eng.plan_nodes([300, 5], 4)
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_unconstrained(eng.make_hparams(num_epochs=EPOCHS, opt=1, init=_abi.GX_INIT_PHILOX, seed=4), None, out)
        print("dense ok bn L4 sgd", float(out.sum()))
        eng.close()
        g = np.load(util.GOLDEN + "/graphs_golden.npz")
        eng = gnnx.Engine(0)
        eng.set_model({k: g[k] for k in util.WKEYS})
        eng.set_graph_batch(g["adj"], g["feat"], g["label"])
        eoff = eng.plan_graphs([0, 3, 5])
        out = np.zeros(int(eoff[-1]), np.float32)
        eng.explain_graphs_unconstrained(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=5), None, out)
        print("dense ok graph", float(out.sum()))
        eng.close()
    if "att" in which:   # explain_var.cu's attention path: node mode (hub and small tasks; with hid = 128 the attention weights are read
        # through L2 while the conv weights stay in shared memory), graph mode, the model forward
        rng = np.random.default_rng(7)
        sc = lambda *s_: (rng.normal(size=s_) * 0.3).astype(np.float32)
        d0, C0 = fx.feat.shape[1], fx.weights["Wp"].shape[0]
        for hid, L, bn in ((20, 3, False), (128, 3, True)):
            dims = [d0] + [hid] * L
            w = {}
            for l in range(1, L + 1):
                w["W%d" % l] = sc(dims[l - 1], dims[l]); w["b%d" % l] = sc(dims[l]); w["Wa%d" % l] = sc(dims[l - 1], dims[l - 1])
            w["Wp"] = sc(C0, hid * L); w["bp"] = sc(C0)
            att = [w["Wa%d" % l] for l in range(1, L + 1)]
            eng = gnnx.Engine(0)
            eng.set_model(w, num_layers=L, bn=bn, att=att)
            eng.set_graph_csr(fx.rowptr, fx.col, fx.feat, fx.label, fx.pred_label)
            plan = eng.plan_nodes([0, 300, 5, 683], L)
            out = np.zeros(plan.total_edges, np.float32)
            eng.explain_nodes_host(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=8), None, out)
            pred = eng.model_forward() if hid <= 32 else np.zeros(1)
            print("att ok node", hid, L, bn, float(out.sum()), float(pred.sum()))
            eng.close()
        g = np.load(util.GOLDEN + "/graphs_golden.npz")
        dg, Cg = g["feat"].shape[2], g["Wp"].shape[0]
        w = dict(W1=sc(dg, 20), b1=sc(20), W2=sc(20, 20), b2=sc(20), W3=sc(20, 20), b3=sc(20), Wp=sc(Cg, 60), bp=sc(Cg))
        eng = gnnx.Engine(0)
        eng.set_model(w, num_layers=3, att=[sc(dg, dg), sc(20, 20), sc(20, 20)])
        eng.set_graph_batch(g["adj"], g["feat"], g["label"])
        eoff = eng.plan_graphs([0, 3, 5])
        out = np.zeros(int(eoff[-1]), np.float32)
        eng.explain_graphs_host(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=9), None, out)
        print("att ok graph", float(out.sum()))
        eng.close()
    if "wide" in which:   # explain_var.cu's wide path (d > 128): node mode with the hub and small tasks (rows beyond n2 gather dP), a
        # --bn 4-layer model with width 128, graph mode with one-hot features, and the model forward at d = 1500 (> 48 KB of shared memory)
        rng = np.random.default_rng(11)
        d0, C0 = 300, fx.weights["Wp"].shape[0]
        feat = rng.normal(size=(fx.N, d0)).astype(np.float32)
        for hid, L, bn in ((20, 3, False), (128, 4, True)):
            dims = [d0] + [hid] * L
            w = {}
            for l in range(1, L + 1):
                w["W%d" % l] = (rng.normal(size=(dims[l - 1], dims[l])) / np.sqrt(dims[l - 1])).astype(np.float32)
                w["b%d" % l] = (rng.normal(size=dims[l]) * 0.3).astype(np.float32)
            w["Wp"] = (rng.normal(size=(C0, hid * L)) * 0.3).astype(np.float32); w["bp"] = np.zeros(C0, np.float32)
            eng = gnnx.Engine(0)
            eng.set_model(w, num_layers=L, bn=bn)
            eng.set_graph_csr(fx.rowptr, fx.col, feat, fx.label, fx.pred_label)
            plan = eng.plan_nodes([0, 300, 5, 683], L)
            out = np.zeros(plan.total_edges, np.float32)
            fm = np.zeros((plan.count, d0), np.float32)
            eng.explain_nodes_host(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=8, opt=0 if bn else 1), None, out, fm)
            pred = eng.model_forward() if hid <= 32 else np.zeros(1)
            print("wide ok node", hid, L, bn, float(out.sum()), float(fm.sum()), float(pred.sum()))
            eng.close()
        g = np.load(util.GOLDEN + "/graphs_golden.npz")
        dg, Cg = 190, g["Wp"].shape[0]
        adj = g["adj"]
        featg = (np.eye(dg, dtype=np.float32)[rng.integers(0, dg, size=adj.shape[:2])] * (adj.sum(2, keepdims=True) > 0)).astype(np.float32)
        w = dict(W1=(rng.normal(size=(dg, 20)) / np.sqrt(dg)).astype(np.float32), b1=np.ones(20, np.float32) * 0.1,
                 W2=(rng.normal(size=(20, 20)) * 0.3).astype(np.float32), b2=np.zeros(20, np.float32),
                 W3=(rng.normal(size=(20, 20)) * 0.3).astype(np.float32), b3=np.zeros(20, np.float32),
                 Wp=(rng.normal(size=(Cg, 60)) * 0.3).astype(np.float32), bp=np.zeros(Cg, np.float32))
        eng = gnnx.Engine(0)
        eng.set_model(w, num_layers=3)
        eng.set_graph_batch(adj, featg, g["label"])
        eoff = eng.plan_graphs([0, 3, 5, 11])
        out = np.zeros(int(eoff[-1]), np.float32)
        eng.explain_graphs_host(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=9), None, out)
        print("wide ok graph", float(out.sum()))
        eng.close()
        w = dict(W1=(rng.normal(size=(1500, 20)) / np.sqrt(1500)).astype(np.float32), b1=np.zeros(20, np.float32),
                 W2=(rng.normal(size=(20, 20)) * 0.3).astype(np.float32), b2=np.zeros(20, np.float32),
                 Wp=(rng.normal(size=(C0, 40)) * 0.3).astype(np.float32), bp=np.zeros(C0, np.float32))
        eng = gnnx.Engine(0)
        eng.set_model(w, num_layers=2)
        eng.set_graph_csr(fx.rowptr, fx.col, rng.normal(size=(fx.N, 1500)).astype(np.float32), fx.label, fx.pred_label)
        print("wide ok forward", float(eng.model_forward().sum()))
        eng.close()
    if "misc" in which:
        eng = util.make_engine(fx)
        rows = eng.neighborhood_rows(np.arange(0, 700, 50), 3)
        plan = eng.plan_nodes([300, 5], 3)
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_host(eng.make_hparams(num_epochs=2), util.golden_m0(fx, plan), out)
        dense = eng.densify_host(out, int(sum(plan.n(t) ** 2 for t in range(plan.count))))
        print("misc ok", int(rows.sum()), float(dense.sum()))
        eng.close()
        # the off-edge regulariser sums of graph mode (trace.cu offedge_graph_kernel): padded graphs, some with padded rows
        g = np.load(util.GOLDEN + "/graphs_golden.npz")
        eng = gnnx.Engine(0)
        eng.set_model({k: g[k] for k in util.WKEYS})
        eng.set_graph_batch(g["adj"], g["feat"], g["label"])
        eng.plan_graphs([0, 3, 5, 11])
        n = int(g["max_nodes"])
        off = eng.offedge_regularisers_graphs(eng.make_hparams(num_epochs=EPOCHS),
                                              np.random.default_rng(0).normal(1.0, 0.2, 4 * n * n).astype(np.float32))
        print("misc ok offedge graphs", float(off.sum()))
        eng.close()
    if "dist_graphs" in which:   # gx_count_graphs and gx_densify_graphs (densify_graphs.cu) on a repeated id, with max_nodes 41 as well:
        # every other graph's dense block then starts at an odd double (the scalar head store)
        g = np.load(util.GOLDEN + "/graphs_golden.npz")
        for n in (40, 41):
            adj = np.zeros((12, n, n), np.uint8)
            adj[:, :40, :40] = g["adj"]
            eng = gnnx.Engine(0)
            eng.set_model({k: g[k] for k in util.WKEYS})
            eng.set_graph_batch(adj, np.pad(g["feat"], ((0, 0), (0, n - 40), (0, 0))), g["label"])
            gids = [5, 0, 11, 5, 3]
            eoff = eng.plan_graphs(gids)
            out = np.zeros(int(eoff[-1]), np.float32)
            eng.explain_graphs_host(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=3), None, out)
            _, e = eng.count_graphs(gids)
            dense = eng.densify_graphs_host(gids, out)
            print("dist_graphs ok", n, int(e.sum()), float(dense.sum()))
            eng.close()
    if "topk" in which:   # denoise.cu's edges mode: kernel masks, ties, a node without a positive value, a cap below the kept count;
        # then the chunk loop of explain_nodes_topk (chunks of 3, the hub node among them)
        import types
        import torch
        eng = util.make_engine(fx)
        plan = eng.plan_nodes([0, 3, 300, 683, 13], 3)
        out = np.zeros(plan.total_edges, np.float32)
        eng.explain_nodes_host(eng.make_hparams(num_epochs=EPOCHS, init=_abi.GX_INIT_PHILOX, seed=3), None, out)
        out[plan.edge_off[1]:plan.edge_off[2]] = np.round(out[plan.edge_off[1]:plan.edge_off[2]] * 4) / 4
        out[plan.edge_off[4]:plan.edge_off[5]] = 0.0
        thr, cnt, uv, vals = eng.denoise_topk_edges(out, 20)
        thr_d, cnt_d, uv_d, vals_d = eng.denoise_topk_edges(torch.from_numpy(out).cuda(), 3, cap=2)
        torch.cuda.synchronize()
        print("topk ok edges", int(cnt.sum()), int(uv.max()), int(cnt_d.sum()))
        eng.close()
        import gnnx_oracle as O
        args = types.SimpleNamespace(num_gc_layers=3, num_epochs=EPOCHS, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid",
                                     mask_bias=False, gpu=False, bias=True, method="base", dataset="syn1", bmname=None, hidden_dim=20,
                                     output_dim=20, name_suffix="", explainer_suffix="", logdir="/tmp", gnnx_init="device", gnnx_seed=2)
        model = gnnx.models.GcnEncoderNode(fx.feat.shape[1], 20, 20, fx.weights["Wp"].shape[0], 3, bn=False, args=args)
        model.load_state_dict({k: torch.tensor(v) for k, v in zip(
            ["conv_first.weight", "conv_first.bias", "conv_block.0.weight", "conv_block.0.bias", "conv_last.weight", "conv_last.bias",
             "pred_model.weight", "pred_model.bias"], [fx.weights[k] for k in util.WKEYS])})
        ex = gnnx.Explainer(model=model, adj=O.dense_from_csr(fx.rowptr, fx.col)[None], feat=fx.feat[None], label=fx.label[None],
                            pred=fx.pred[None], train_idx=[], args=args, writer=None, print_training=False, graph_idx=-1)
        thr, offsets, uv, vals = ex.explain_nodes_topk([0, 300, 5, 683, 13, 42, 7], chunk_size=3)
        print("topk ok explain_nodes_topk", int(offsets[-1]), float(vals.sum()))
        ex.engine.close()


if __name__ == "__main__":
    main()
