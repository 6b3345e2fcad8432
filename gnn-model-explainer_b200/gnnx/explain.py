"""Drop-in for the reference's explainer/explain.py:Explainer (node-classification path).

Same constructor, same method names/arguments, same return values (dense (n,n) float64 numpy
arrays, one per node, in input order) and the same .npy side effect
(explain.py:216-220).  The per-node optimisation is NOT executed in Python: the whole batch of
nodes goes through libgnnx (k-hop extraction kernel + one persistent CTA per node).

Differences that are deliberate and documented:
  * explain_nodes() batches all nodes into one launch; it returns the list of masks like the
    reference (explain.py:234-236,290-292) but does not run the reference's matplotlib/tensorboard
    post-processing (denoise_graph/align/log_graph, explain.py:238-288: viz, out of scope).
  * M0 policy (args.gnnx_init, default "torch"): "torch" draws FloatTensor(n,n).normal_(1, std)
    from torch's global CPU generator per node in call order, exactly the RNG consumption of
    ExplainModule.construct_edge_mask (explain.py:645-652) -> bit-identical M0 under the same
    torch.manual_seed; "device" draws N(1, 2/n) with Philox on the GPU (no n^2 host work).
  * args.gnnx_latency (default False): True lets small batches (one explain() call, a shard of a multi-GPU run) split their most
    expensive tasks over thread-block clusters; masks then agree with the default mode to
    round-off instead of bit for bit (gx_debug_set_cluster in include/gnnx.h).
  * a node outside its own k-hop set (isolated) raises instead of explaining a wrong row.
"""
import math
import os

import numpy as np
import torch

from . import _abi
from .engine import Engine
from . import graph_utils as _gu


def gen_prefix(args):
    """utils/io_utils.py:37-51 (file-name compatibility of the .npy side effect)."""
    name = args.bmname if getattr(args, "bmname", None) is not None else args.dataset
    name += "_" + args.method
    name += "_h" + str(args.hidden_dim) + "_o" + str(args.output_dim)
    if not args.bias:
        name += "_nobias"
    if len(args.name_suffix) > 0:
        name += "_" + args.name_suffix
    return name


def gen_explainer_prefix(args):
    """utils/io_utils.py:54-60."""
    name = gen_prefix(args) + "_explain"
    if len(args.explainer_suffix) > 0:
        name += "_" + args.explainer_suffix
    return name


def model_weights(model):
    """state_dict of a reference (or gnnx) GcnEncoderNode/GcnEncoderGraph -> weight dict.
    Keys as in the reference checkpoints (SURVEY 8a8): conv_first / conv_block.i / conv_last /
    pred_model; an attention model (--method att) also has <layer>.att_weight, returned as Wa1 .. WaL.  A model with an MLP
    prediction head (pred_hidden_dims, models.py:193-207: pred_model.0 / .2 / .. Linears around ReLUs) returns its hidden Linears as
    "head" = [(W, b), ..] (torch's (out, in) layout) and its last Linear as Wp / bp."""
    sd = {k: v.detach().cpu().float().numpy() for k, v in model.state_dict().items()}
    head = []
    if "pred_model.weight" not in sd:
        j = 0
        while ("pred_model.%d.weight" % j) in sd:
            head.append((sd["pred_model.%d.weight" % j], sd["pred_model.%d.bias" % j]))
            j += 2
        if len(head) < 2 or any(k.startswith("pred_model.") and not k.startswith(tuple("pred_model.%d." % i for i in range(0, j, 2)))
                                for k in sd):
            raise ValueError("pred_model is neither a Linear nor the Sequential(Linear, ReLU, .., Linear) of pred_hidden_dims")
    n_block = 0
    while ("conv_block.%d.weight" % n_block) in sd:
        n_block += 1
    names = ["conv_first"] + ["conv_block.%d" % i for i in range(n_block)] + ["conv_last"]
    w = {}
    for l, nm in enumerate(names, 1):
        w["W%d" % l] = sd[nm + ".weight"]
        w["b%d" % l] = sd.get(nm + ".bias")
        if (nm + ".self_weight") in sd:
            raise NotImplementedError("the add_self GraphConv variant is out of scope")
        if (nm + ".att_weight") in sd:
            w["Wa%d" % l] = sd[nm + ".att_weight"]
    if any(("Wa%d" % l) in w for l in range(1, len(names) + 1)) and not all(("Wa%d" % l) in w for l in range(1, len(names) + 1)):
        raise ValueError("att_weight on some conv layers only")
    if head:
        (w["Wp"], w["bp"]), w["head"] = head[-1], head[:-1]
    else:
        w["Wp"], w["bp"] = sd["pred_model.weight"], sd["pred_model.bias"]
    return w, len(names)


def torch_m0_walk(sizes):
    """The torch-compatible initial masks (args.gnnx_init="torch") of a list, drawn lazily in list order: per size n the float32 (n, n)
    array FloatTensor(n, n).normal_(1, std) of ExplainModule.construct_edge_mask (explain.py:645-652), a view of the drawn tensor.  n is
    the k-hop size in node mode and the padded max_nodes in graph mode.  The reference draws for every entry it explains, so every entry
    is drawn here too, used or not (another rank's entries, the gradient baseline): once the walk is exhausted torch's global CPU RNG is
    where the reference's loop over the same list leaves it.  The n^2 normals per entry are this policy's cost (~3 ns each on one core;
    args.gnnx_init="device" has no host work)."""
    for n in sizes:
        n = int(n)
        yield torch.FloatTensor(n, n).normal_(1.0, torch.nn.init.calculate_gain("relu") * math.sqrt(2.0 / (n + n))).numpy()


def _m0_at_edges(plan, draws):
    """M0 of a node plan at its directed-edge slots (float32[total_edges]): the next plan.count arrays of the iterator `draws`, one per
    task in plan order, each gathered at its task's slots."""
    m0 = np.empty(plan.total_edges, dtype=np.float32)
    flat = plan.flat_index()            # row * n + col of every edge slot, whole batch at once
    eo = plan.edge_off
    for t in range(plan.count):
        np.take(next(draws).reshape(-1), flat[eo[t]:eo[t + 1]], out=m0[eo[t]:eo[t + 1]])
    return m0


class Explainer:
    def __init__(self, model, adj, feat, label, pred, train_idx, args, writer=None,
                 print_training=True, graph_mode=False, graph_idx=False, device=None):
        self.model = model
        if hasattr(self.model, "eval"):
            self.model.eval()
        self.adj = adj
        self.feat = feat
        self.label = label
        self.pred = pred
        self.train_idx = train_idx
        self.n_hops = args.num_gc_layers
        self.graph_mode = graph_mode
        self.graph_idx = graph_idx
        self.args = args
        self.writer = writer
        self.print_training = print_training
        self._neighborhoods = None
        if getattr(args, "mask_act", "sigmoid") != "sigmoid":
            raise NotImplementedError("mask_act=%r is not built (default: sigmoid; the reference's ReLU variant returns NaN masks, "
                                      "tests/test_oracle.py)" % args.mask_act)
        # args.mask_bias: accepted.  The reference's bias matrix starts at 0 where ReLU6 has zero gradient, Adam never moves it and the
        # masks equal the default run bit for bit (explain.py:657-660,673-676; pinned by tests/test_oracle.py) -- no extra state needed.
        # utils/train_utils.py:7-23: adam / sgd / rmsprop / adagrad, schedulers none / step / cos
        if getattr(args, "opt", "adam") not in _abi.GX_OPT or getattr(args, "opt_scheduler", "none") not in _abi.GX_SCHED:
            raise ValueError("unknown optimiser / scheduler: %r / %r" % (getattr(args, "opt", None), getattr(args, "opt_scheduler", None)))
        bn = bool(getattr(model, "bn", False))
        if device is None:
            device = int(os.environ.get("LOCAL_RANK", "0")) if torch.cuda.is_available() else 0
        self.engine = Engine(device)
        weights, num_layers = model_weights(model)
        self._att = "Wa1" in weights
        self._wide = weights["W1"].shape[0] > 128   # inputs wider than 128: the variant kernel's wide path
        self._head = "head" in weights             # an MLP prediction head (pred_hidden_dims): the variant kernel
        self.engine.set_model(weights, num_layers=num_layers, bn=bn,
                              att=[weights["Wa%d" % l] for l in range(1, num_layers + 1)] if self._att else None,
                              head=weights.get("head"))
        if getattr(args, "gnnx_latency", False):
            self.engine.debug_cluster(0, 0)   # latency mode: thread-block clusters for the expensive tasks of batches that leave SMs idle
        self._max_width = max(weights["W%d" % l].shape[1] for l in range(1, num_layers + 1))
        self._wide_layers = self._max_width > 32
        # the models the tuned kernels do not run (outside the gradient baseline's coverage), gx_set_model's selection of the variant
        # kernel: --bn, num_gc_layers != 3, hidden or output widths above 32, attention, inputs wider than 128, an MLP head
        self._variant = bn or num_layers != 3 or self._wide_layers or self._att or self._wide or self._head
        # the variant kernel does not log the per-epoch trace print_training replays, nor does any optimiser other than Adam
        self._no_trace = self._variant or getattr(args, "opt", "adam") != "adam"
        # node mode also takes a scipy.sparse (N,N) adjacency, a batch of one graph (feat / label / pred keep their (1,N,..) shapes): a
        # graph of 10^5 nodes has 10^10 dense entries, its CSR comes straight from the sparse matrix
        self._sparse = _gu.is_sparse(adj)
        if graph_mode:
            # graph classification: the whole padded batch goes to the device once (explain.py:80-85)
            if self._sparse:
                raise ValueError("graph mode expects a dense adj of shape (G,n,n), not a sparse matrix")
            adj_np = np.asarray(adj)
            if adj_np.ndim != 3:
                raise ValueError("graph mode expects adj of shape (G,n,n)")
            self.engine.set_graph_batch(adj_np, np.asarray(feat), np.asarray(label))
            return
        if self._sparse:
            if len(adj.shape) != 2 or adj.shape[0] != adj.shape[1]:
                raise ValueError("a sparse adj must be one (N,N) graph")
        elif np.asarray(adj).ndim != 3:
            raise ValueError("node mode expects adj of shape (B,N,N)")
        # node tasks on a batch of graphs (explain.py:80-95 index adj / feat / label / pred with graph_idx): the engine holds one graph
        # at a time, graph 0 is uploaded now, another one when a call names it
        self._csr_cache = {}
        self._own_pred = {}
        self._current_graph = None
        self._select_graph(0)

    def _select_graph(self, graph_idx):
        g = 0 if graph_idx in (-1, None, False) else int(graph_idx)
        if g == self._current_graph:
            return g
        if not 0 <= g < self._num_graphs():
            raise IndexError("graph_idx %d out of range for adj of shape %s" % (g, self.adj.shape if self._sparse else np.asarray(self.adj).shape))
        if g not in self._csr_cache:
            self._csr_cache[g] = _gu.csr_from_sparse(self.adj) if self._sparse else _gu.csr_from_dense(np.asarray(self.adj)[g])
        self._rowptr, self._col = self._csr_cache[g]
        feat_np = np.asarray(self.feat, dtype=np.float32)[g]
        label_np = np.asarray(self.label)[g].astype(np.int32)
        if self.pred is None or g in self._own_pred:
            # no stored predictions (the reference reads cg["pred"] from the checkpoint, explainer_main.py:186-193): run the model's
            # forward on the device (gx_model_forward = GcnEncoderNode.forward on the whole graph) and keep the logits
            if g not in self._own_pred:
                self.engine.set_graph_csr(self._rowptr, self._col, feat_np, label_np, np.zeros(len(label_np), np.int32))
                self._own_pred[g] = self.engine.model_forward()
            pred_g = self._own_pred[g]
        else:
            pred_g = np.asarray(self.pred)[g]
        self._pred_label = np.argmax(pred_g, axis=1).astype(np.int32)          # explain.py:105
        self.engine.set_graph_csr(self._rowptr, self._col, feat_np, label_np, self._pred_label)
        self._current_graph = g
        return g

    def _num_graphs(self):
        return 1 if self._sparse else np.asarray(self.adj).shape[0]

    # the reference computes this dense (B,N,N) matrix eagerly in __init__ (explain.py:67); here
    # it is materialised on demand only (the engine never needs it).
    @property
    def neighborhoods(self):
        if self._neighborhoods is None:
            keep = self._current_graph
            mats = []
            for g in range(self._num_graphs()):
                self._select_graph(g)
                N = self.engine.num_nodes
                mats.append(self.engine.neighborhood_rows(np.arange(N, dtype=np.int32), self.n_hops).astype(int))
            self._select_graph(keep)
            self._neighborhoods = np.stack(mats)
        return self._neighborhoods

    def extract_neighborhood(self, node_idx, graph_idx=0):
        """explain.py:492-501: (node_idx_new, sub_adj, sub_feat, sub_label, neighbors)."""
        graph_idx = self._select_graph(graph_idx)
        plan = self.engine.plan_nodes([int(node_idx)], self.n_hops)
        nbrs = plan.neighbors_of(0).astype(np.int64)
        # the caller's own adjacency rows / columns, exactly like the reference (adj[g][nbrs][:, nbrs]): self loops, if any, stay in
        # sub_adj (the plan's edge list drops them, as the explainer's diag_mask does for the optimisation)
        if self._sparse:
            sub_adj = self.adj.tocsr()[nbrs][:, nbrs].toarray()
        else:
            sub_adj = np.asarray(self.adj)[graph_idx][nbrs][:, nbrs]
        sub_feat = np.asarray(self.feat)[graph_idx, nbrs]
        sub_label = np.asarray(self.label)[graph_idx][nbrs]
        return int(plan.node_idx_new[0]), sub_adj, sub_feat, sub_label, nbrs

    # ---------------------------------------------------------------- internals
    def _hparams(self):
        a = self.args
        init = getattr(a, "gnnx_init", "torch")
        if init not in ("torch", "device"):
            raise ValueError("args.gnnx_init must be 'torch' or 'device'")
        hp = self.engine.make_hparams(
            num_epochs=a.num_epochs, lr=a.lr,
            init=_abi.GX_INIT_M0 if init == "torch" else _abi.GX_INIT_PHILOX,
            seed=int(getattr(a, "gnnx_seed", 0)))
        hp.opt = _abi.GX_OPT[getattr(a, "opt", "adam")]
        hp.opt_scheduler = _abi.GX_SCHED[getattr(a, "opt_scheduler", "none")]
        if hp.opt_scheduler == _abi.GX_SCHED["step"]:
            hp.opt_decay_step = int(a.opt_decay_step); hp.opt_decay_rate = float(a.opt_decay_rate)
        elif hp.opt_scheduler == _abi.GX_SCHED["cos"]:
            hp.opt_restart = int(a.opt_restart)
        return hp, init

    @staticmethod
    def _draw_graph_m0_subset(n, num_graphs, positions, rows_cols):
        """Graph mode's M0 on one rank of a sharded run: the walk over the WHOLE graph list (num_graphs graphs padded to n), keeping
        M[rows, cols] of the graphs at `positions` (ascending; rows_cols[i] = (rows, cols) of positions[i]'s graph in slot order),
        concatenated -> float32.  torch's global RNG ends where one process's explain_graphs of the same list leaves it, whatever the
        rank owns."""
        kept = dict(zip((int(p) for p in positions), rows_cols))
        parts = [M[kept[p]] for p, M in enumerate(torch_m0_walk([n] * int(num_graphs))) if p in kept]
        return np.concatenate(parts) if parts else np.zeros(0, np.float32)

    def _explain_batch(self, node_indices, graph_idx=0, model="exp", unconstrained=False):
        if model not in ("exp", "grad"):
            raise NotImplementedError("model=%r (att) is not built" % model)
        self._select_graph(graph_idx)
        nodes = [int(i) for i in node_indices]
        plan = self.engine.plan_nodes(nodes, self.n_hops)
        edge_mask = np.empty(plan.total_edges, dtype=np.float32)
        draws = torch_m0_walk(np.diff(plan.node_off))     # lazy: draws nothing unless the torch init reads it below
        if model == "grad":        # explain.py:125-133: one backward to the adjacency, no mask parameters
            if self._head:
                raise NotImplementedError("model='grad' is not built for models with an MLP prediction head (pred_hidden_dims)")
            try:
                self.engine.grad_nodes_host(edge_mask)     # (unconstrained is ignored here, as in the reference)
            except _abi.GnnxError as e:
                if e.status == _abi.GX_ERR_UNSUPPORTED:    # a neighbourhood with self loops: refused before any RNG is consumed
                    raise NotImplementedError(str(e)) from None
                raise
            if self._hparams()[1] == "torch":      # the reference still constructs an ExplainModule per node, i.e. consumes n^2 normals:
                for _ in draws:                    # keep the RNG in step
                    pass
            return plan, edge_mask
        self._check_unconstrained(unconstrained)
        hp, init = self._hparams()
        if unconstrained:
            # explain.py:688-692: the dense mask drives the forward, so every one of the n^2 normals of M0 is a parameter
            m0 = np.concatenate([D.reshape(-1) for D in draws]) if init == "torch" else None
            if not self.print_training:
                self.engine.explain_nodes_unconstrained(hp, m0, edge_mask)
                return plan, edge_mask
            trace = np.zeros((plan.count, hp.num_epochs, _abi.GX_TRACE_COLS), np.float32)
            pred = np.zeros((plan.count, hp.num_epochs, self.engine.num_classes), np.float32)
            self.engine.explain_nodes_unconstrained(hp, m0, edge_mask, trace=trace, trace_pred=pred)
            self.last_trace = self._print_trace(hp, trace, pred, None, None)    # the kernel's loss covers all n^2 entries
            return plan, edge_mask
        if not self.print_training or self._no_trace:
            if self.print_training:
                self._print_no_trace()
            m0 = _m0_at_edges(plan, draws) if init == "torch" else None
            self.engine.explain_nodes_host(hp, m0, edge_mask)
            return plan, edge_mask
        # print_training (explain.py:148-159): the kernels log every epoch's loss terms / density / softmax row (gx_explain_io.trace); the
        # off-edge entries of the dense draws only matter for the printed loss
        dense = list(draws) if init == "torch" else None
        m0 = None if dense is None else _m0_at_edges(plan, iter(dense))
        trace = np.zeros((plan.count, hp.num_epochs, _abi.GX_TRACE_COLS), np.float32)
        pred = np.zeros((plan.count, hp.num_epochs, self.engine.num_classes), np.float32)
        self.engine.explain_nodes_ex(hp, m0, edge_mask, trace=trace, trace_pred=pred)
        off = self.engine.offedge_regularisers(hp, np.concatenate([D.reshape(-1) for D in dense])) if dense is not None else None
        self.last_trace = self._print_trace(hp, trace, pred, off, np.diff(plan.node_off).astype(np.float64) ** 2)
        return plan, edge_mask

    def _check_unconstrained(self, unconstrained):
        if not unconstrained:
            return
        if self._att:
            raise NotImplementedError("unconstrained=True is not built for attention models (--method att)")
        if self._wide:
            raise NotImplementedError("unconstrained=True is not built for inputs wider than 128 features")
        if self._max_width > 128:
            raise NotImplementedError("unconstrained=True is not built for hidden / output widths above 128 (this model: %d)" % self._max_width)

    def _print_no_trace(self):
        if self._head:
            print("(per-epoch trace is not built for models with an MLP prediction head (pred_hidden_dims))")
        elif self._att:
            print("(per-epoch trace is not built for attention models (--method att))")
        elif self._wide:
            print("(per-epoch trace is not built for inputs wider than 128 features)")
        else:
            print("(per-epoch trace is not built for --bn / num_gc_layers != 3 / optimisers other than Adam / hidden or output widths above 32)")

    def _print_trace(self, hp, trace, pred, off, nn):
        """Replays the reference's per-epoch print (explain.py:148-159), task after task.  With the torch-compatible init the loss is
        the reference's own number (edge part from the kernels + the regulariser sums over the n^2 - E_d mask entries that never reach
        the result, gx_offedge_regularisers / gx_offedge_regularisers_graphs; nn[t] = n^2 of task t's dense mask: the k-hop set in node
        mode, max_nodes in graph mode); with the device init those entries are never materialised and the printed loss covers the
        edge entries only."""
        loss = trace[:, :, _abi.TR_LOSS_EDGES].astype(np.float64)
        if off is not None:
            loss = loss + hp.coef_size * off[:, :, 0] + hp.coef_ent * off[:, :, 1] / np.asarray(nn, np.float64)[:, None]
        for t in range(trace.shape[0]):
            for epoch in range(hp.num_epochs):
                print("epoch: ", epoch, "; loss: ", float(loss[t, epoch]), "; mask density: ", float(trace[t, epoch, _abi.TR_DENSITY]),
                      "; pred: ", torch.from_numpy(pred[t, epoch]))
            print("finished training in ", 0.0)
        return dict(loss=loss, density=trace[:, :, _abi.TR_DENSITY].copy(), pred=pred, terms=trace)

    def _save(self, masked_adj, node_idx):
        fname = "masked_adj_" + gen_explainer_prefix(self.args) + (
            "node_idx_" + str(node_idx) + "graph_idx_" + str(self.graph_idx) + ".npy")
        os.makedirs(self.args.logdir, exist_ok=True)
        with open(os.path.join(self.args.logdir, fname), "wb") as outfile:
            np.save(outfile, np.asarray(masked_adj.copy()))
        return fname

    # ---------------------------------------------------------------- public API
    # a trace is built for at most this many epochs per call (gx_explain_io.trace); longer runs print a notice instead
    _MAX_TRACE_EPOCHS = 1536

    def _explain_graph_batch(self, graph_indices, unconstrained=False):
        self._check_unconstrained(unconstrained)
        gids = [int(g) for g in graph_indices]
        edge_off = self.engine.plan_graphs(gids)
        hp, init = self._hparams()
        # print_training (explain.py:148-159): the kernels log every epoch; the unconstrained kernel for every model, the tuned kernel
        # for the default model with Adam, up to _MAX_TRACE_EPOCHS epochs
        traced = self.print_training and (unconstrained or (not self._no_trace and hp.num_epochs <= self._MAX_TRACE_EPOCHS))
        if self.print_training and not traced:
            if self._no_trace:
                self._print_no_trace()
            else:
                print("(per-epoch trace is not built for more than %d epochs per call)" % self._MAX_TRACE_EPOCHS)
        n = self.engine.batch_n
        m0 = None
        dense = None      # the full (n, n) draws: the unconstrained kernel's M0, or the off-edge entries of the printed loss
        rc = [self.engine.graph_rows_cols(g) for g in gids]
        if init == "torch":
            draws = torch_m0_walk([n] * len(gids))      # n = the padded size
            if unconstrained or traced:
                dense = np.concatenate([M.reshape(-1) for M in draws])
                draws = dense.reshape(-1, n, n)
            m0 = dense if unconstrained else np.concatenate([M[rows_cols] for M, rows_cols in zip(draws, rc)])
        edge_mask = np.empty(int(edge_off[-1]), dtype=np.float32)
        trace = pred = None
        if traced:
            trace = np.zeros((len(gids), hp.num_epochs, _abi.GX_TRACE_COLS), np.float32)
            pred = np.zeros((len(gids), hp.num_epochs, self.engine.num_classes), np.float32)
        if unconstrained:
            self.engine.explain_graphs_unconstrained(hp, m0, edge_mask, trace=trace, trace_pred=pred)
        elif traced:
            self.engine.explain_nodes_ex(hp, m0, edge_mask, trace=trace, trace_pred=pred, graphs=True)
        else:
            self.engine.explain_graphs_host(hp, m0, edge_mask)
        if traced:
            off = None
            if not unconstrained and dense is not None:   # the unconstrained kernel's loss already covers all n^2 entries
                off = self.engine.offedge_regularisers_graphs(hp, dense)
            self.last_trace = self._print_trace(hp, trace, pred, off, np.full(len(gids), float(n) * n))
        return self._dense_graphs(rc, edge_off, edge_mask)

    def _dense_graphs(self, rc, edge_off, edge_mask):
        n = self.engine.batch_n
        out = []
        for t, (rows, cols) in enumerate(rc):
            D = np.zeros((n, n), dtype=np.float64)
            D[rows, cols] = edge_mask[edge_off[t]:edge_off[t + 1]]
            out.append(D)
        return out

    def _check_graph_grad(self):
        if self._variant:
            raise NotImplementedError("model='grad' in graph mode is built for the default model only (3 layers, hidden and output "
                                      "widths <= 32, no --bn, attention or MLP head, inputs <= 128 features)")

    def _graph_grad_labels(self, gids):
        """The loss label of model="grad" for every graph of `gids`: argmax(pred[0][g]) (explain.py:102), or -1 (the model's own
        prediction, arg-max of the logits of gx_grad_graphs' forward) when the Explainer has no stored predictions."""
        if self.pred is None:
            return np.full(len(gids), -1, np.int32)
        return np.argmax(np.asarray(self.pred)[0][np.asarray(gids, np.int64)], axis=-1).astype(np.int32)

    def _graph_grad_batch(self, graph_indices):
        """explain.py:97-133 in graph mode with model="grad" for a list of graphs, one launch (gx_grad_graphs): the gradient of
        -log softmax(logits)[label] with respect to the unmasked padded adjacency, sigmoid(|g| + |g|^T) * adj.  unconstrained is
        ignored, as in the reference."""
        self._check_graph_grad()          # before any RNG is consumed
        gids = [int(g) for g in graph_indices]
        edge_off = self.engine.plan_graphs(gids)
        labels = self._graph_grad_labels(gids)
        if self._hparams()[1] == "torch":
            # the reference still constructs an ExplainModule per graph, i.e. draws its n^2 normals (explain.py:645-652): keep the RNG in step
            for _ in torch_m0_walk([self.engine.batch_n] * len(gids)):
                pass
        edge_mask = np.empty(max(int(edge_off[-1]), 1), dtype=np.float32)
        try:
            self.engine.grad_graphs_host(labels, edge_mask)
        except _abi.GnnxError as e:
            if e.status == _abi.GX_ERR_UNSUPPORTED:
                raise NotImplementedError(str(e)) from None
            raise
        return self._dense_graphs([self.engine.graph_rows_cols(g) for g in gids], edge_off, edge_mask)

    def explain_graphs(self, graph_indices, save=True, model="exp"):
        """explain.py:356-402 -> list of (n,n) masked adjacencies (one batched launch; the reference's
        denoise_graph/log_graph drawing is out of scope).  model="grad": the gradient baseline of every graph instead (explain.py:125-133)."""
        if not self.graph_mode:
            raise ValueError("Explainer was not constructed with graph_mode=True")
        if model not in ("exp", "grad"):
            raise NotImplementedError("model=%r is not built in graph mode" % model)
        out = self._graph_grad_batch(graph_indices) if model == "grad" else self._explain_graph_batch(graph_indices)
        if save:
            for m in out:
                self._save(m, 0)      # the reference overwrites one file: node_idx_0 graph_idx_<self.graph_idx>
        return out

    def explain(self, node_idx, graph_idx=0, graph_mode=False, unconstrained=False, model="exp"):
        """explain.py:74-221 -> (n,n) float64 masked adjacency of the node's k-hop subgraph (node mode)
        or of the whole padded graph `graph_idx` (graph_mode=True)."""
        if graph_mode or self.graph_mode:
            if not self.graph_mode:
                raise ValueError("Explainer was not constructed with graph_mode=True")
            if model not in ("exp", "grad"):
                raise NotImplementedError("model=%r is not built in graph mode" % model)
            if model == "grad":
                masked_adj = self._graph_grad_batch([graph_idx])[0]
            else:
                masked_adj = self._explain_graph_batch([graph_idx], unconstrained)[0]
            fname = self._save(masked_adj, node_idx)
            if self.print_training:
                print("Saved adjacency matrix to ", fname)
            return masked_adj
        plan, edge_mask = self._explain_batch([node_idx], graph_idx, model, unconstrained)
        masked_adj = plan.dense_of(0, edge_mask, dtype=np.float64)
        fname = self._save(masked_adj, node_idx)
        if self.print_training:
            print("Saved adjacency matrix to ", fname)
        return masked_adj

    def explain_nodes(self, node_indices, args=None, graph_idx=0, save=True, copy=True):
        """explain.py:225-292 -> list of (n,n) float64 masked adjacencies in input order.  One batched launch; the dense arrays are
        built ON DEVICE (gx_densify) and come back in one transfer -- the list entries are views of that one buffer:
          copy=True  (default) independent results like the reference's: views of a pinned buffer that is not reused while any of them is alive;
          copy=False ONE pinned buffer owned by the Explainer, overwritten by the next call.
        save=True writes the reference's per-node .npy files (explain.py:216-220), which at ~0.4 MB per node dominates the call;
        args.gnnx_init="device" removes the n^2 host normals per node of the torch-compatible init."""
        self._select_graph(graph_idx)
        if self.print_training:
            plan, edge_mask = self._explain_batch(node_indices, graph_idx)
            out = [plan.dense_of(t, edge_mask, dtype=np.float64) for t in range(plan.count)]
        else:
            nodes = [int(i) for i in node_indices]
            eng = self.engine
            eng.follow_torch_stream()
            plan = eng.plan_nodes(nodes, self.n_hops)
            hp, init = self._hparams()
            dev = torch.device("cuda", eng.device)
            m0_dev = None
            if init == "torch":
                m0_dev = torch.from_numpy(_m0_at_edges(plan, torch_m0_walk(np.diff(plan.node_off)))).to(dev, non_blocking=False)
            mask_dev = eng.explain_nodes_device(hp, m0_dev)
            dense_dev = eng.densify_device(mask_dev)
            if copy:
                host = self._result_buffer(dense_dev.numel())       # pinned, never handed out twice while a result still refers to it
                torch.from_numpy(host)[:dense_dev.numel()].copy_(dense_dev)
            else:
                if getattr(self, "_pinned", None) is None or self._pinned.numel() < dense_dev.numel():
                    self._pinned = torch.empty(max(dense_dev.numel(), 1), dtype=torch.float64).pin_memory()
                self._pinned[:dense_dev.numel()].copy_(dense_dev)
                host = self._pinned.numpy()
            n_t = np.diff(plan.node_off).astype(np.int64)
            offs = np.concatenate([[0], np.cumsum(n_t * n_t)])
            out = [host[offs[t]:offs[t + 1]].reshape(n_t[t], n_t[t]) for t in range(plan.count)]
        if save:
            for t, node in enumerate(node_indices):
                self._save(out[t], int(node))
        return out

    def _result_buffer(self, numel):
        """Host memory for one call's dense results: a pinned buffer from a small pool.  The returned arrays are views of it
        (numpy keeps the buffer alive through .base), and a buffer is reused only when no earlier result refers to it any more
        (sys.getrefcount), so results stay independent like the reference's -- without a 0.3 GB pageable allocation + copy per call."""
        import sys
        pool = self.__dict__.setdefault("_pool", [])
        for i, (t, a) in enumerate(pool):
            if t.numel() >= numel and sys.getrefcount(a) <= 3:      # pool tuple + loop variable + getrefcount's argument
                return a
        pool[:] = [(t, a) for (t, a) in pool if sys.getrefcount(a) > 3][-2:]     # drop idle buffers that are too small
        t = torch.empty(max(int(numel), 1), dtype=torch.float64).pin_memory()
        a = t.numpy()
        pool.append((t, a))
        return a

    # ---------------------------------------------------------------- evaluation step right after the masks
    # planted-motif edges relative to the first motif node, in the sorted local numbering (explain.py:537-577)
    _MOTIF_EDGES = {
        "syn1": [(0, 1), (1, 2), (2, 3), (0, 3), (0, 4), (1, 4)],          # house
        "syn2": [(0, 1), (1, 2), (2, 3), (0, 3), (0, 4), (1, 4)],
        "syn4": [(0, 1), (1, 2), (2, 3), (3, 4), (4, 5), (0, 5)],          # 6-cycle
    }

    def make_pred_real(self, adj, start):
        """explain.py:535-579: (pred, real) over the upper-triangular positive entries of a masked adjacency;
        real = 1 on the planted motif's edges (fixed offsets from `start`)."""
        if self.args.dataset not in self._MOTIF_EDGES:
            raise NotImplementedError("make_pred_real knows syn1/syn2/syn4 only (like the reference)")
        adj = np.asarray(adj)
        upper = np.triu(adj) > 0
        pred = adj[upper]
        truth = np.zeros(adj.shape, dtype=bool)
        for (p_, q_) in self._MOTIF_EDGES[self.args.dataset]:
            if adj[start + p_][start + q_] > 0:        # IndexError past the subgraph, like the reference
                truth[start + p_, start + q_] = True
        real = truth[upper].astype(adj.dtype)
        return pred, real

    def explain_nodes_gnn_stats(self, node_indices, args=None, graph_idx=0, model="exp"):
        """explain.py:295-353: explain the nodes (one batched launch), score the edge masks against the planted
        motifs with ROC-AUC and write log/pr/auc_<dataset>_<model>.txt; returns the masks.  The PR-curve PNG
        and the tensorboard drawings of the reference are not produced (viz, out of scope)."""
        from sklearn.metrics import roc_auc_score
        plan, edge_mask = self._explain_batch(node_indices, graph_idx, model)
        masked_adjs = [plan.dense_of(t, edge_mask, dtype=np.float64) for t in range(plan.count)]
        pred_all, real_all = [], []
        for t in range(plan.count):
            pred, real = self.make_pred_real(masked_adjs[t], int(plan.node_idx_new[t]))
            pred_all.append(pred); real_all.append(real)
        real_cat, pred_cat = np.concatenate(real_all), np.concatenate(pred_all)
        self.auc = float(roc_auc_score(real_cat, pred_cat))
        os.makedirs(os.path.join("log", "pr"), exist_ok=True)
        # explain.py:308,329-335: the denoised graphs (threshold_num=20) and the precision/recall curve.  The reference draws both
        # (tensorboard / matplotlib); here the graphs are kept on the object and the curve is written as arrays (+ PNG if matplotlib exists)
        self.denoised, _ = self.denoise_nodes(plan, edge_mask, threshold_num=20, with_feat=True)
        from sklearn.metrics import precision_recall_curve
        precision, recall, thresholds = precision_recall_curve(real_cat, pred_cat)
        self.pr_curve = (precision, recall, thresholds)
        np.savez(os.path.join("log", "pr", "pr_" + self.args.dataset + "_" + model + ".npz"), precision=precision, recall=recall, thresholds=thresholds)
        try:
            import matplotlib
            matplotlib.use("agg")
            import matplotlib.pyplot as plt
            plt.plot(recall, precision)
            plt.savefig(os.path.join("log", "pr", "pr_" + self.args.dataset + "_" + model + ".png"))
            plt.close()
        except ImportError:
            pass
        with open(os.path.join("log", "pr", "auc_" + self.args.dataset + "_" + model + ".txt"), "w") as f:
            f.write("dataset: {}, model: {}, auc: {}\n".format(self.args.dataset, "exp", str(self.auc)))
        return masked_adjs

    def denoise_nodes(self, plan, edge_mask, threshold_num=20, max_component=True, with_feat=False):
        """io_utils.denoise_graph(masked_adj, node_idx_new, feat, threshold_num=20) (explain.py:308, utils/io_utils.py:193-245) for
        every node of a packed result: the 2*threshold_num-largest threshold and the surviving edges are computed on device
        (gx_denoise_topk); only those <= ~40 edges per node come back, the networkx object is assembled from them."""
        from . import io_utils
        thr, cnt, slots, vals = self.engine.denoise_topk(edge_mask, threshold_num)
        cap = slots.shape[1]
        if int(cnt.max(initial=0)) > cap:          # many values tie at the threshold: fetch again with room for all of them
            thr, cnt, slots, vals = self.engine.denoise_topk(edge_mask, threshold_num, cap=int(cnt.max()))
        flat = plan.flat_index()
        out = []
        for t in range(plan.count):
            n = plan.n(t)
            k = int(cnt[t])
            f = flat[plan.edge_off[t] + slots[t, :k]]
            feat = np.asarray(self.feat)[0, plan.neighbors_of(t)] if with_feat else None
            out.append(io_utils.graph_from_edges(n, int(plan.node_idx_new[t]), f // n, f % n, vals[t, :k], feat, None, max_component))
        return out, thr

    def explain_nodes_packed(self, node_indices, graph_idx=0):
        """Same computation, returning (plan, edge_mask) without densifying: edge_mask[edge_off[t]:
        edge_off[t+1]] are the masked_adj entries of node t at plan.csr_of(t) (row-major order)."""
        return self._explain_batch(node_indices, graph_idx)

    def explain_nodes_topk(self, node_indices, threshold_num=20, chunk_size=None, graph_idx=0):
        """explain_nodes followed by denoise_graph's thresholding (threshold_num=20: what explain_nodes_gnn_stats and the node loop
        of explain.py:244,308 keep of every mask), for lists whose masks do not fit on the host or the device at once (BASELINE
        configs[4]: ~0.4 GB of plan and optimiser state per node).  The list is explained `chunk_size` nodes at a time (default: the
        device's SM count, one task per SM) and every chunk's masks are thresholded on device (gx_denoise_topk_edges); only the kept
        counts come back to the host.  Returns, in input order:
          thr     float32 CUDA tensor [count]: the threshold of each node (+inf for a mask without a positive value)
          offsets int64 numpy array [count+1]: node t's edges are rows offsets[t]:offsets[t+1] of uv / vals
          uv      int32 CUDA tensor [total, 2]: the kept undirected edges in global node ids, u < v, ascending per node
          vals    float32 CUDA tensor [total]: their mask values
        A node's masks do not depend on the chunk it is explained in, so the result is the same bits for every chunk_size
        (args.gnnx_latency is switched off for the call).  With args.gnnx_init="torch" every node draws its n^2 normals in list order:
        M0 and torch's RNG afterwards are those of explain_nodes(node_indices).  No per-epoch trace, no .npy files."""
        if self.graph_mode:
            raise ValueError("explain_nodes_topk is node mode only (graph mode gathers its packed masks: gnnx.dist.explain_graphs_sharded)")
        self.engine.follow_torch_stream()
        self._select_graph(graph_idx)
        nodes = np.asarray(node_indices, np.int64).reshape(-1)
        thr, cnt, uv, vals = self._topk_chunks(nodes, np.arange(len(nodes)), None, threshold_num, chunk_size)
        return thr, np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64), uv, vals

    def _topk_chunks(self, nodes, positions, n_all, threshold_num, chunk_size, timings=None):
        """The chunk loop of explain_nodes_topk over the list entries `positions` (ascending) of `nodes`.  With the torch init it makes
        one forward walk over the list up to the last position, drawing every entry's n^2 normals and keeping those of the positions
        explained here (n_all[p] = k-hop size of entry p, gx_count_nodes; needed for the entries not explained here), then finishes
        the walk to the end of the list: torch's RNG ends where explain_nodes(nodes) leaves it.
        Returns (thr CUDA [k], counts int64 numpy [k], uv CUDA [total, 2], vals CUDA [total]) of those positions.
        timings (dict or None): accumulates the wall seconds of the phases (plan, m0, explain, topk; synchronising after each) and the
        explainer kernels' device seconds (explain_device)."""
        import time
        eng = self.engine
        dev = torch.device("cuda", eng.device)
        if chunk_size is None:
            chunk_size = torch.cuda.get_device_properties(dev).multi_processor_count
        chunk_size = int(chunk_size)
        if chunk_size < 1:
            raise ValueError("chunk_size must be >= 1")
        if int(threshold_num) < 1:
            raise ValueError("threshold_num must be >= 1")
        hp, init = self._hparams()
        clock = [time.perf_counter()]

        def tick(key):
            if timings is not None:
                torch.cuda.synchronize(dev)
                now = time.perf_counter()
                timings[key] = timings.get(key, 0.0) + now - clock[0]
                clock[0] = now

        thr_p, cnt_p, uv_p, val_p = [], [], [], []
        if init == "torch":
            # the walk reads an entry's size when it reaches the entry: a chunk's own plan fills in the sizes of its positions first
            sizes = np.zeros(len(nodes), np.int64) if n_all is None else np.array(n_all, np.int64)
            walk = enumerate(torch_m0_walk(sizes[p] for p in range(len(nodes))))
        latency = bool(getattr(self.args, "gnnx_latency", False))
        if latency:
            eng.debug_cluster(1, 0)
        try:
            for c0 in range(0, len(positions), chunk_size):
                pos = np.asarray(positions[c0:c0 + chunk_size], np.int64)
                clock[0] = time.perf_counter()
                plan = eng.plan_nodes(nodes[pos], self.n_hops, fetch=(init == "torch"))
                tick("plan")
                m0_dev = None
                if init == "torch":
                    sizes[pos] = np.diff(plan.node_off)
                    mine = set(pos.tolist())
                    m0_dev = torch.from_numpy(_m0_at_edges(plan, (M for p, M in walk if p in mine))).to(dev)
                    tick("m0")
                mask = eng.explain_nodes_device(hp, m0_dev)
                if timings is not None:
                    tick("explain")
                    timings["explain_device"] = timings.get("explain_device", 0.0) + eng.last_explain_ms() / 1e3
                thr, cnt, uv, vals = eng.denoise_topk_edges(mask, threshold_num)
                cnt_h = cnt.cpu().numpy().astype(np.int64)
                if int(cnt_h.max(initial=0)) > uv.shape[1]:      # values tie at the threshold: again with room for all of them
                    thr, cnt, uv, vals = eng.denoise_topk_edges(mask, threshold_num, cap=int(cnt_h.max()))
                keep = torch.arange(uv.shape[1], device=dev)[None, :] < cnt[:, None]
                thr_p.append(thr); cnt_p.append(cnt_h); uv_p.append(uv[keep]); val_p.append(vals[keep])
                tick("topk")
        finally:
            if latency:
                eng.debug_cluster(0, 0)
        if init == "torch":      # the rest of the list, so that torch's RNG ends as after one process's explain_nodes
            for _ in walk:
                pass
        if not thr_p:
            return (torch.zeros(0, dtype=torch.float32, device=dev), np.zeros(0, np.int64),
                    torch.zeros((0, 2), dtype=torch.int32, device=dev), torch.zeros(0, dtype=torch.float32, device=dev))
        return torch.cat(thr_p), np.concatenate(cnt_p), torch.cat(uv_p), torch.cat(val_p)

    def iter_explain_nodes_packed(self, node_indices, chunk_size, graph_idx=0, model="exp"):
        """Large graphs (BASELINE configs[4]: a k-hop neighbourhood is most of a 10^5-node graph, ~0.4 GB of plan and optimiser
        state per explained node): explain the list `chunk_size` nodes at a time and yield (nodes_of_chunk, plan, edge_mask)
        per chunk, so that neither the device workspace nor the host ever holds more than one chunk (one CTA per SM => 132 is a
        natural chunk on an H100).  The dense (n,n) arrays of explain_nodes would need 80 GB per node there."""
        nodes = [int(i) for i in node_indices]
        if chunk_size < 1:
            raise ValueError("chunk_size must be >= 1")
        for s0 in range(0, len(nodes), int(chunk_size)):
            part = nodes[s0:s0 + int(chunk_size)]
            plan, edge_mask = self._explain_batch(part, graph_idx, model)
            yield part, plan, edge_mask
