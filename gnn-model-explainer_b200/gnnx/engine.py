"""Engine: thin host wrapper around one libgnnx handle (one per GPU / host thread).

Numpy arrays are passed as HOST pointers; torch CUDA tensors as DEVICE pointers.  All arithmetic
happens inside the library's CUDA kernels; this module only marshals buffers."""
import ctypes as C

import numpy as np

from . import _abi


def _np_ptr(a):
    return C.c_void_p(a.ctypes.data) if a is not None else C.c_void_p(0)


def _f32c(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _i32c(a):
    return np.ascontiguousarray(a, dtype=np.int32)


class Plan:
    """Canonical (reference-ordered) description of a batch of k-hop subgraphs."""

    def __init__(self, nodes, node_off, edge_off, neighbors, node_idx_new, sub_rowptr, sub_col):
        self.nodes = nodes
        self.node_off = node_off
        self.edge_off = edge_off
        self.neighbors = neighbors
        self.node_idx_new = node_idx_new
        self.sub_rowptr = sub_rowptr
        self.sub_col = sub_col
        self.count = len(nodes)
        self.total_nodes = int(node_off[-1])
        self.total_edges = int(edge_off[-1])

    def n(self, t):
        return int(self.node_off[t + 1] - self.node_off[t])

    def neighbors_of(self, t):
        return self.neighbors[self.node_off[t]:self.node_off[t + 1]]

    def csr_of(self, t):
        """(rowptr[n+1], col[E_t]) of task t (task-local)."""
        n = self.n(t)
        rp = self.sub_rowptr[self.node_off[t] + t: self.node_off[t] + t + n + 1]
        return rp, self.sub_col[self.edge_off[t]:self.edge_off[t + 1]]

    def rows_cols_of(self, t):
        rp, col = self.csr_of(t)
        rows = np.repeat(np.arange(len(rp) - 1, dtype=np.int64), np.diff(rp))
        return rows, col.astype(np.int64)

    def flat_index(self):
        """row * n_t + col of every directed-edge slot of the batch (int64[total_edges]): where slot e lives in the row-major
        (n_t, n_t) dense array of its task."""
        count = self.count
        n_t = np.diff(self.node_off).astype(np.int64)
        deg = np.diff(self.sub_rowptr.astype(np.int64))
        if count > 1:
            deg = np.delete(deg, self.node_off[1:-1] + np.arange(1, count) - 1)   # differences across task boundaries
        row_local = np.arange(self.total_nodes, dtype=np.int64) - np.repeat(self.node_off[:-1], n_t)
        rows = np.repeat(row_local, deg)
        n_of_edge = np.repeat(n_t, np.diff(self.edge_off))
        return rows * n_of_edge + self.sub_col.astype(np.int64)

    def dense_of(self, t, edge_values, dtype=np.float64):
        """(n,n) dense array holding edge_values of task t at the sub-adjacency entries."""
        n = self.n(t)
        rows, cols = self.rows_cols_of(t)
        out = np.zeros((n, n), dtype=dtype)
        out[rows, cols] = edge_values[self.edge_off[t]:self.edge_off[t + 1]]
        return out


class Engine:
    def __init__(self, device=0):
        self._lib = _abi.lib()
        h = C.c_void_p()
        _abi.check(self._lib.gx_create(int(device), C.byref(h)))
        self._h = h
        self.device = int(device)
        self.input_dim = None
        self._plan = None

    def close(self):
        if getattr(self, "_h", None):
            self._lib.gx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---------------------------------------------------------------- setup
    def set_stream(self, cuda_stream_ptr):
        _abi.check(self._lib.gx_set_stream(self._h, C.c_void_p(int(cuda_stream_ptr))))

    def follow_torch_stream(self):
        """Binds the engine to torch's current stream on its device: the engine's work on device tensors is then ordered with the torch
        ops that fill or read them, and the caching allocator reuses them only after the engine is done.  The drop-in (Explainer,
        gnnx.dist) calls this at the start of every call that hands device tensors between torch and the engine."""
        import torch
        self.set_stream(torch.cuda.current_stream(self.device).cuda_stream)

    def sync(self):
        _abi.check(self._lib.gx_sync(self._h))

    def set_model(self, weights, num_layers=3, bn=False, att=None, head=None):
        """weights: dict W1,b1,W2,b2,W3,b3,Wp,bp (numpy; b* may be None).  Shapes are checked here: the C ABI takes bare
        pointers, so a checkpoint whose layers do not chain (or a concat=False model) must not reach it.
        att: an attention model's (in, in) conv_*.att_weight matrices, one per layer (gx_set_model_att); None for any other model.
        head: an MLP prediction head (pred_hidden_dims, models.py:193-207): [(W, b), ..] of its hidden Linears in order, torch's
        (out, in) layout; Wp / bp are then its last Linear (C, last hidden width) (gx_set_model_head).  None: pred_model is one Linear."""
        Ws = [_f32c(weights["W%d" % (l + 1)]) for l in range(num_layers)]
        bs = [None if weights.get("b%d" % (l + 1)) is None else _f32c(weights["b%d" % (l + 1)])
              for l in range(num_layers)]
        Wp, bp = _f32c(weights["Wp"]), _f32c(weights["bp"])
        if any(w.ndim != 2 for w in Ws) or Wp.ndim != 2 or bp.ndim != 1:
            raise ValueError("conv weights must be 2-D (in,out), pred_model.weight (C, sum of layer widths), pred_model.bias (C,)")
        hid = Ws[0].shape[1]
        for l in range(num_layers):
            want_in = Ws[0].shape[0] if l == 0 else Ws[l - 1].shape[1]
            if Ws[l].shape[0] != want_in:
                raise ValueError("layer %d weight is %s, expected %d input features" % (l + 1, Ws[l].shape, want_in))
            if 0 < l < num_layers - 1 and Ws[l].shape[1] != hid:
                raise ValueError("hidden layers must share one width (models.py:193-220): layer %d is %s" % (l + 1, Ws[l].shape))
            if bs[l] is not None and bs[l].shape != (Ws[l].shape[1],):
                raise ValueError("layer %d bias is %s, expected (%d,)" % (l + 1, bs[l].shape, Ws[l].shape[1]))
        pd = sum(w.shape[1] for w in Ws)
        hw, hb = [], []
        if head is not None:
            if not 1 <= len(head) <= _abi.GX_MAX_HEAD_LAYERS:
                raise NotImplementedError("an MLP prediction head of %d hidden layers is not built (1 .. %d)" % (len(head), _abi.GX_MAX_HEAD_LAYERS))
            width = pd
            for j, (w, b) in enumerate(head):
                w, b = _f32c(w), _f32c(b)
                if w.ndim != 2 or w.shape[1] != width or b.shape != (w.shape[0],):
                    raise ValueError("head layer %d is %s / %s, expected (out, %d) / (out,)" % (j, w.shape, b.shape, width))
                hw.append(w); hb.append(b)
                width = w.shape[0]
            pd = width      # the last Linear reads the last hidden layer
        if Wp.shape[1] != pd:
            if Wp.shape[1] == Ws[-1].shape[1]:
                raise NotImplementedError("concat=False models (pred_model over the last layer only, models.py:113-116) are not built")
            raise ValueError("pred_model.weight is %s, expected (C, %d) = concat of the layer outputs" % (Wp.shape, pd))
        if bp.shape != (Wp.shape[0],):
            raise ValueError("pred_model.bias is %s, expected (%d,)" % (bp.shape, Wp.shape[0]))
        wp = (C.c_void_p * num_layers)(*[w.ctypes.data for w in Ws])
        bp_arr = (C.c_void_p * num_layers)(*[(b.ctypes.data if b is not None else None) for b in bs])
        if head is not None:
            Was = [_f32c(a) for a in att] if att is not None else []
            if att is not None and [a.shape for a in Was] != [(w.shape[0], w.shape[0]) for w in Ws]:
                raise ValueError("att_weight shapes %s do not match the conv layers" % [a.shape for a in Was])
            dims = _abi.GxModelDims(Ws[0].shape[0], Ws[0].shape[1], Ws[-1].shape[1], Wp.shape[0], num_layers,
                                    (_abi.GX_MODEL_BN if bn else 0) | (_abi.GX_MODEL_ATT if att is not None else 0))
            ap = (C.c_void_p * num_layers)(*[a.ctypes.data for a in Was]) if att is not None else None
            widths = np.asarray([w.shape[0] for w in hw], np.int32)
            lw = hw + [Wp]
            lb = hb + [bp]
            hwp = (C.c_void_p * len(lw))(*[w.ctypes.data for w in lw])
            hbp = (C.c_void_p * len(lb))(*[b.ctypes.data for b in lb])
            _abi.check(self._lib.gx_set_model_head(self._h, C.byref(dims), wp, bp_arr, ap, len(hw), _np_ptr(widths), hwp, hbp))
        elif att is None:
            dims = _abi.GxModelDims(Ws[0].shape[0], Ws[0].shape[1], Ws[-1].shape[1], Wp.shape[0], num_layers,
                                    _abi.GX_MODEL_BN if bn else 0)
            _abi.check(self._lib.gx_set_model(self._h, C.byref(dims), wp, bp_arr, _np_ptr(Wp), _np_ptr(bp)))
        else:
            Was = [_f32c(a) for a in att]
            if len(Was) != num_layers:
                raise ValueError("att: %d attention matrices for %d layers" % (len(Was), num_layers))
            for l, a in enumerate(Was):
                if a.shape != (Ws[l].shape[0], Ws[l].shape[0]):
                    raise ValueError("layer %d att_weight is %s, expected (%d, %d)" % (l + 1, a.shape, Ws[l].shape[0], Ws[l].shape[0]))
            dims = _abi.GxModelDims(Ws[0].shape[0], Ws[0].shape[1], Ws[-1].shape[1], Wp.shape[0], num_layers,
                                    (_abi.GX_MODEL_BN if bn else 0) | _abi.GX_MODEL_ATT)
            ap = (C.c_void_p * num_layers)(*[a.ctypes.data for a in Was])
            _abi.check(self._lib.gx_set_model_att(self._h, C.byref(dims), wp, bp_arr, ap, _np_ptr(Wp), _np_ptr(bp)))
        self.input_dim = int(Ws[0].shape[0])
        self.num_classes = int(Wp.shape[0])

    def set_graph_csr(self, rowptr, col, feat, label, pred_label):
        rowptr, col = _i32c(rowptr), _i32c(col)
        feat = _f32c(feat)
        N = len(rowptr) - 1
        assert feat.shape[0] == N
        label = None if label is None else _i32c(label)
        pred_label = _i32c(pred_label)
        _abi.check(self._lib.gx_set_graph_csr(self._h, N, _np_ptr(rowptr), _np_ptr(col), _np_ptr(feat),
                                              feat.shape[1], _np_ptr(label), _np_ptr(pred_label)))
        self.num_nodes = N

    def set_graph_csr_structure(self, rowptr, col):
        """Structure-only upload (for neighbourhood queries): dummy 1-d features / labels."""
        N = len(rowptr) - 1
        self.set_graph_csr(rowptr, col, np.zeros((N, 1), np.float32), None, np.zeros(N, np.int32))

    # ---------------------------------------------------------------- k-hop
    def neighborhood_rows(self, nodes, n_hops):
        nodes = _i32c(nodes)
        out = np.zeros((len(nodes), self.num_nodes), dtype=np.uint8)
        if len(nodes):
            _abi.check(self._lib.gx_neighborhood_rows(self._h, _np_ptr(nodes), len(nodes), int(n_hops), _np_ptr(out)))
        return out

    def plan_nodes(self, nodes, n_hops, fetch=True):
        nodes = _i32c(nodes)
        tn, te = C.c_int64(), C.c_int64()
        _abi.check(self._lib.gx_plan_nodes(self._h, _np_ptr(nodes), len(nodes), int(n_hops), C.byref(tn), C.byref(te)))
        self._plan_sizes = (len(nodes), tn.value, te.value)
        self._plan = None
        if not fetch:
            return None
        return self.fetch_plan(nodes)

    def fetch_plan(self, nodes):
        count, tn, te = self._plan_sizes
        node_off = np.empty(count + 1, np.int64)
        edge_off = np.empty(count + 1, np.int64)
        nbrs = np.empty(tn, np.int32)
        idx_new = np.empty(count, np.int32)
        srp = np.empty(tn + count, np.int32)
        scol = np.empty(te, np.int32)
        _abi.check(self._lib.gx_plan_fetch(self._h, _np_ptr(node_off), _np_ptr(edge_off), _np_ptr(nbrs),
                                           _np_ptr(idx_new), _np_ptr(srp), _np_ptr(scol)))
        self._plan = Plan(np.asarray(nodes), node_off, edge_off, nbrs, idx_new, srp, scol)
        return self._plan

    # ---------------------------------------------------------------- graph-classification mode
    def set_graph_batch(self, adj, feat, label):
        """adj (G,n,n) 0/1 symmetric, feat (G,n,d), label (G,): the padded batch of Explainer(graph_mode=True)."""
        adj = np.asarray(adj)
        G, n, _ = adj.shape
        gi, ri, ci = np.nonzero(adj)
        if gi.size and not np.all(adj[gi, ri, ci] == 1):
            raise NotImplementedError("weighted adjacency is not built (reference datasets are 0/1)")
        rowptr = np.zeros(G * n + 1, dtype=np.int64)
        np.add.at(rowptr, gi * n + ri + 1, 1)
        rowptr = np.cumsum(rowptr).astype(np.int32)
        col = _i32c(ci)
        feat = _f32c(np.asarray(feat).reshape(G * n, -1))
        label = _i32c(np.asarray(label).reshape(G))
        _abi.check(self._lib.gx_set_graph_batch_csr(self._h, G, n, _np_ptr(rowptr), _np_ptr(col), _np_ptr(feat),
                                                    feat.shape[1], _np_ptr(label)))
        self.batch_rowptr, self.batch_col, self.batch_G, self.batch_n = rowptr, col, G, n

    def plan_graphs(self, graph_ids):
        gids = _i32c(graph_ids)
        edge_off = np.empty(len(gids) + 1, np.int64)
        te = C.c_int64()
        _abi.check(self._lib.gx_plan_graphs(self._h, _np_ptr(gids), len(gids), _np_ptr(edge_off), C.byref(te)))
        self._graph_count = len(gids)
        self._graph_total = te.value
        return edge_off

    def graph_rows_cols(self, g):
        """(rows, cols) of graph g's adjacency entries in slot (row-major) order."""
        n = self.batch_n
        rp = self.batch_rowptr[g * n: (g + 1) * n + 1]
        rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(rp))
        return rows, self.batch_col[rp[0]:rp[-1]].astype(np.int64)

    def explain_graphs_host(self, hp, m0_edges, edge_mask_out, feat_mask_out=None):
        _abi.check(self._lib.gx_explain_graphs(self._h, C.byref(hp), _abi.GX_HOST, _np_ptr(m0_edges),
                                               _np_ptr(edge_mask_out), _np_ptr(feat_mask_out)))

    def explain_graphs_device(self, hp, m0=None, out=None):
        """The planned graphs with DEVICE buffers (gx_explain_graphs, GX_DEVICE): m0 (optional torch.float32 CUDA tensor, GX_INIT_M0)
        -> edge masks as a torch.float32 CUDA tensor [total_edges]; asynchronous on the engine's stream."""
        import torch
        te = self._graph_total
        if out is None:
            out = torch.empty(max(te, 1), dtype=torch.float32, device=torch.device("cuda", self.device))
        _abi.check(self._lib.gx_explain_graphs(self._h, C.byref(hp), _abi.GX_DEVICE, C.c_void_p(m0.data_ptr() if m0 is not None else None),
                                               C.c_void_p(out.data_ptr()), None))
        return out[:te]

    def count_graphs(self, graph_ids):
        """(n[count], e_d[count]) of every listed graph of the uploaded batch without building a plan (gx_count_graphs): its rows with
        an edge and its directed edges."""
        gids = _i32c(graph_ids)
        n = np.zeros(len(gids), np.int32); e = np.zeros(len(gids), np.int32)
        _abi.check(self._lib.gx_count_graphs(self._h, _np_ptr(gids), len(gids), _np_ptr(n), _np_ptr(e)))
        return n, e

    def densify_graphs_device(self, graph_ids, values, out=None):
        """gx_densify_graphs on device: the packed float32 masks of the listed graphs in list order (CUDA tensor) -> float64 CUDA tensor
        (len(graph_ids), max_nodes, max_nodes), zero outside each graph's edges."""
        import torch
        gids = _i32c(graph_ids)
        n = self.batch_n
        if out is None:
            out = torch.empty((len(gids), n, n), dtype=torch.float64, device=values.device)
        _abi.check(self._lib.gx_densify_graphs(self._h, _abi.GX_DEVICE, _np_ptr(gids), len(gids),
                                               C.c_void_p(values.data_ptr() if values.numel() else None), C.c_void_p(out.data_ptr())))
        return out

    def densify_graphs_host(self, graph_ids, values):
        """The same with host buffers: numpy float32 values -> numpy float64 (len(graph_ids), max_nodes, max_nodes)."""
        gids, values = _i32c(graph_ids), _f32c(values)
        out = np.empty((len(gids), self.batch_n, self.batch_n), np.float64)
        _abi.check(self._lib.gx_densify_graphs(self._h, _abi.GX_HOST, _np_ptr(gids), len(gids), _np_ptr(values), _np_ptr(out)))
        return out

    # ---------------------------------------------------------------- hot path
    def make_hparams(self, num_epochs=100, lr=0.1, init=_abi.GX_INIT_M0, seed=0, **over):
        hp = _abi.GxHparams()
        self._lib.gx_default_hparams(C.byref(hp))
        hp.num_epochs = int(num_epochs)
        hp.lr = float(lr)
        hp.init = int(init)
        hp.seed = int(seed)
        for k, v in over.items():
            setattr(hp, k, v)
        return hp

    def explain_nodes_host(self, hp, m0_edges, edge_mask_out, feat_mask_out=None):
        """Host buffers (numpy).  m0_edges may be None with GX_INIT_PHILOX."""
        _abi.check(self._lib.gx_explain_nodes(self._h, C.byref(hp), _abi.GX_HOST, _np_ptr(m0_edges),
                                              _np_ptr(edge_mask_out), _np_ptr(feat_mask_out)))

    def explain_nodes_ex(self, hp, m0_edges, edge_mask_out, feat_mask_out=None, trace=None, trace_pred=None,
                         state_in=None, state_out=None, graphs=False):
        """gx_explain_nodes_ex / gx_explain_graphs_ex with host (numpy) buffers.  trace: float32 (count, num_epochs, 8) out;
        trace_pred: float32 (count, num_epochs, C) out; state_in / state_out: dicts with M? (state_in: m0_edges carries M),
        'm', 'v' (total_edges,) and 'feat' (count, 3, d) float32 arrays (state_out also 'M')."""
        io = _abi.GxExplainIo()
        ptr = lambda a: a.ctypes.data if a is not None else None
        io.m0_edges = ptr(m0_edges); io.edge_mask = ptr(edge_mask_out); io.feat_mask = ptr(feat_mask_out)
        io.trace = ptr(trace); io.trace_pred = ptr(trace_pred)
        if state_in is not None:
            io.adam_m_in = ptr(state_in["m"]); io.adam_v_in = ptr(state_in["v"]); io.feat_state_in = ptr(state_in.get("feat"))
        if state_out is not None:
            io.mask_param_out = ptr(state_out.get("M")); io.adam_m_out = ptr(state_out.get("m")); io.adam_v_out = ptr(state_out.get("v"))
            io.feat_state_out = ptr(state_out.get("feat"))
        fn = self._lib.gx_explain_graphs_ex if graphs else self._lib.gx_explain_nodes_ex
        _abi.check(fn(self._h, C.byref(hp), _abi.GX_HOST, C.byref(io)))

    def explain_nodes_unconstrained(self, hp, m0_dense, edge_mask_out, mask_dense_out=None, trace=None, trace_pred=None):
        """Explainer.explain(..., unconstrained=True) for every planned node (gx_explain_nodes_unconstrained), host (numpy) buffers:
        m0_dense float32 [sum_t n_t^2] (None with GX_INIT_PHILOX); edge_mask_out float32 [total_edges]; mask_dense_out float32
        [sum_t n_t^2]; trace float32 (count, num_epochs, 8); trace_pred float32 (count, num_epochs, C)."""
        self._unconstrained(self._lib.gx_explain_nodes_unconstrained, hp, m0_dense, edge_mask_out, mask_dense_out, trace, trace_pred)

    def explain_graphs_unconstrained(self, hp, m0_dense, edge_mask_out, mask_dense_out=None, trace=None, trace_pred=None):
        """The same for every planned graph (gx_explain_graphs_unconstrained): n_t = max_nodes, edge_mask_out at the graphs' CSR slots."""
        self._unconstrained(self._lib.gx_explain_graphs_unconstrained, hp, m0_dense, edge_mask_out, mask_dense_out, trace, trace_pred)

    def _unconstrained(self, fn, hp, m0_dense, edge_mask_out, mask_dense_out, trace, trace_pred):
        m0 = None if m0_dense is None else _f32c(m0_dense)
        _abi.check(fn(self._h, C.byref(hp), _abi.GX_HOST, _np_ptr(m0), _np_ptr(edge_mask_out), _np_ptr(mask_dense_out),
                      _np_ptr(trace), _np_ptr(trace_pred)))

    def offedge_regularisers(self, hp, m0_dense):
        """(count, num_epochs, 2) float64: per epoch (sum sigmoid(M), sum H(sigmoid(M))) over the mask entries outside the
        sub-adjacency -- the part of the reference's printed loss that never influences the result (gx_offedge_regularisers)."""
        count = self._plan_sizes[0]
        out = np.zeros((count, hp.num_epochs, 2), np.float64)
        m0_dense = _f32c(m0_dense)
        _abi.check(self._lib.gx_offedge_regularisers(self._h, C.byref(hp), _abi.GX_HOST, _np_ptr(m0_dense), _np_ptr(out)))
        return out

    def offedge_regularisers_graphs(self, hp, m0_dense):
        """The same for the planned graphs (gx_offedge_regularisers_graphs): m0_dense = the (max_nodes, max_nodes) M0 of every
        planned graph in plan order; the sums run over all entries but the graph's directed edges (padded rows, non-edges, diagonal)."""
        out = np.zeros((self._graph_count, hp.num_epochs, 2), np.float64)
        m0_dense = _f32c(m0_dense)
        if m0_dense.size != self._graph_count * self.batch_n * self.batch_n:
            raise ValueError("m0_dense has %d entries, expected %d graphs x %d^2" % (m0_dense.size, self._graph_count, self.batch_n))
        _abi.check(self._lib.gx_offedge_regularisers_graphs(self._h, C.byref(hp), _abi.GX_HOST, _np_ptr(m0_dense), _np_ptr(out)))
        return out

    def grad_nodes_host(self, edge_mask_out):
        """Gradient baseline (explain(model="grad")) of every planned node into a host buffer."""
        _abi.check(self._lib.gx_grad_nodes(self._h, _abi.GX_HOST, _np_ptr(edge_mask_out)))

    def _graph_labels(self, pred_label):
        lbl = _i32c(pred_label).reshape(-1)
        if lbl.size != self._graph_count:
            raise ValueError("pred_label has %d entries for %d planned graphs" % (lbl.size, self._graph_count))
        return lbl

    def grad_graphs_host(self, pred_label, edge_mask_out):
        """Gradient baseline (explain(..., graph_mode=True, model="grad")) of every planned graph into a host buffer (gx_grad_graphs).
        pred_label: the loss label of every planned graph in plan order, -1 = the model's own prediction."""
        lbl = self._graph_labels(pred_label)
        _abi.check(self._lib.gx_grad_graphs(self._h, _abi.GX_HOST, _np_ptr(lbl), _np_ptr(edge_mask_out)))

    def grad_graphs_device(self, pred_label, out=None):
        """The same into DEVICE memory: -> torch.float32 CUDA tensor [total_edges]; asynchronous on the engine's stream (pred_label is
        a host array)."""
        import torch
        lbl = self._graph_labels(pred_label)
        te = self._graph_total
        if out is None:
            out = torch.empty(max(te, 1), dtype=torch.float32, device=torch.device("cuda", self.device))
        _abi.check(self._lib.gx_grad_graphs(self._h, _abi.GX_DEVICE, _np_ptr(lbl), C.c_void_p(out.data_ptr())))
        return out[:te]

    def explain_nodes_ptr(self, hp, space, m0_ptr, out_ptr, feat_ptr=0):
        _abi.check(self._lib.gx_explain_nodes(self._h, C.byref(hp), int(space), C.c_void_p(int(m0_ptr) or None),
                                              C.c_void_p(int(out_ptr)), C.c_void_p(int(feat_ptr) or None)))

    # ---------------------------------------------------------------- device-resident variants (torch CUDA tensors)
    def explain_nodes_device(self, hp, m0=None, out=None):
        """The planned batch with DEVICE buffers: m0 (optional torch.float32 CUDA tensor, GX_INIT_M0) -> edge masks as a
        torch.float32 CUDA tensor [total_edges]; asynchronous on the engine's stream."""
        import torch
        te = self._plan_sizes[2]
        if out is None:
            out = torch.empty(max(te, 1), dtype=torch.float32, device=torch.device("cuda", self.device))
        self.explain_nodes_ptr(hp, _abi.GX_DEVICE, m0.data_ptr() if m0 is not None else 0, out.data_ptr())
        return out[:te]

    def densify_device(self, edge_mask, out=None):
        """gx_densify on device: packed float32 edge masks (CUDA tensor) -> float64 CUDA tensor [sum_t n_t^2] holding the dense
        (n_t, n_t) arrays Explainer.explain returns, task after task."""
        import torch
        total = int(self._dense_total())
        if out is None:
            out = torch.empty(max(total, 1), dtype=torch.float64, device=edge_mask.device)
        _abi.check(self._lib.gx_densify(self._h, _abi.GX_DEVICE, C.c_void_p(edge_mask.data_ptr()), C.c_void_p(out.data_ptr())))
        return out[:total]

    def _dense_total(self):
        """sum_t n_t^2 of the library's current node plan (gx_plan_fetch's node offsets: a host-side copy, no device work)."""
        node_off = np.empty(self._plan_sizes[0] + 1, np.int64)
        _abi.check(self._lib.gx_plan_fetch(self._h, _np_ptr(node_off), None, None, None, None, None))
        return int(np.sum(np.diff(node_off) ** 2))

    # ---------------------------------------------------------------- multi-GPU (one all-gather of the masks)
    def count_nodes(self, nodes, n_hops):
        """(n[count], e_d[count]) of every node's k-hop subgraph without building a plan (gx_count_nodes)."""
        nodes = _i32c(nodes)
        n = np.zeros(len(nodes), np.int32); e = np.zeros(len(nodes), np.int32)
        if len(nodes):
            _abi.check(self._lib.gx_count_nodes(self._h, _np_ptr(nodes), len(nodes), int(n_hops), _np_ptr(n), _np_ptr(e)))
        return n, e

    @staticmethod
    def comm_unique_id():
        buf = C.create_string_buffer(128)
        _abi.check(_abi.lib().gx_comm_unique_id(buf))
        return buf.raw

    def comm_init(self, world, rank, unique_id):
        _abi.check(self._lib.gx_comm_init(self._h, int(world), int(rank), C.c_char_p(bytes(unique_id))))
        self.comm_world, self.comm_rank = int(world), int(rank)

    def comm_destroy(self):
        self._lib.gx_comm_destroy(self._h)
        self.comm_world = None

    def allgather_masks(self, local, slot_floats, gathered=None):
        """ONE ncclAllGather (gx_allgather_masks) of this rank's packed mask values (CUDA float32 tensor) -> [world, slot_floats]."""
        import torch
        if gathered is None:
            gathered = torch.empty((self.comm_world, int(slot_floats)), dtype=torch.float32, device=local.device)
        _abi.check(self._lib.gx_allgather_masks(self._h, C.c_void_p(local.data_ptr() if local.numel() else None), int(local.numel()),
                                                int(slot_floats), C.c_void_p(gathered.data_ptr())))
        return gathered

    def unshard_masks(self, gathered, src_off, dst_off, sizes, out):
        src_off = np.ascontiguousarray(src_off, np.int64); dst_off = np.ascontiguousarray(dst_off, np.int64); sizes = _i32c(sizes)
        _abi.check(self._lib.gx_unshard_masks(self._h, C.c_void_p(gathered.data_ptr()), len(sizes), _np_ptr(src_off), _np_ptr(dst_off),
                                              _np_ptr(sizes), C.c_void_p(out.data_ptr())))
        return out

    def denoise_topk(self, edge_mask, threshold_num=20, cap=None):
        """io_utils.denoise_graph's thresholding (utils/io_utils.py:193-231) of every planned node on device: returns
        (threshold[count], count[count], slots[count,cap], vals[count,cap]); slots are task-local edge slots (ascending), -1 padded."""
        count = self._plan_sizes[0]
        cap = int(cap or 2 * threshold_num + 16)
        thr = np.zeros(count, np.float32); cnt = np.zeros(count, np.int32)
        slots = np.zeros((count, cap), np.int32); vals = np.zeros((count, cap), np.float32)
        _abi.check(self._lib.gx_denoise_topk(self._h, _abi.GX_HOST, _np_ptr(_f32c(edge_mask)), int(threshold_num), cap,
                                             _np_ptr(thr), _np_ptr(cnt), _np_ptr(slots), _np_ptr(vals)))
        return thr, cnt, slots, vals

    def denoise_topk_edges(self, edge_mask, threshold_num=20, cap=None):
        """denoise_topk's thresholding of every planned node, delivered as undirected edges in global node ids (gx_denoise_topk_edges):
        returns (threshold[count], count[count], uv[count,cap,2], vals[count,cap]); node t's kept edges are uv[t, :count[t]] (u < v,
        ascending), -1 padded.  A numpy edge_mask gives numpy arrays; a CUDA tensor gives CUDA tensors on the same device, asynchronous
        on the engine's stream.  count[t] > cap when values tie at the threshold: only the first cap edges are written."""
        count = self._plan_sizes[0]
        cap = int(cap or threshold_num + 16)
        if hasattr(edge_mask, "is_cuda") and edge_mask.is_cuda:
            import torch
            dev = edge_mask.device
            em = edge_mask.contiguous()
            thr = torch.empty(count, dtype=torch.float32, device=dev)
            cnt = torch.empty(count, dtype=torch.int32, device=dev)
            uv = torch.empty((count, cap, 2), dtype=torch.int32, device=dev)
            vals = torch.empty((count, cap), dtype=torch.float32, device=dev)
            ptr = lambda t: C.c_void_p(t.data_ptr() if t.numel() else None)
            _abi.check(self._lib.gx_denoise_topk_edges(self._h, _abi.GX_DEVICE, C.c_void_p(em.data_ptr()), int(threshold_num), cap,
                                                       ptr(thr), ptr(cnt), ptr(uv), ptr(vals)))
            return thr, cnt, uv, vals
        thr = np.zeros(count, np.float32); cnt = np.zeros(count, np.int32)
        uv = np.zeros((count, cap, 2), np.int32); vals = np.zeros((count, cap), np.float32)
        _abi.check(self._lib.gx_denoise_topk_edges(self._h, _abi.GX_HOST, _np_ptr(_f32c(edge_mask)), int(threshold_num), cap,
                                                   _np_ptr(thr), _np_ptr(cnt), _np_ptr(uv), _np_ptr(vals)))
        return thr, cnt, uv, vals

    def densify_host(self, edge_mask, total_dense):
        out = np.empty(total_dense, np.float64)
        _abi.check(self._lib.gx_densify(self._h, _abi.GX_HOST, _np_ptr(_f32c(edge_mask)), _np_ptr(out)))
        return out

    def debug_force_stream(self, on=True):
        """Test knob: plan every task into the streaming kernel (explain_stream.cu) regardless of its size."""
        _abi.check(self._lib.gx_debug_force_stream(self._h, int(bool(on))))

    def model_forward(self):
        """Logits (N, C) of the uploaded model on the uploaded graph: GcnEncoderNode.forward(x, adj)[0][0] (gx_model_forward)."""
        out = np.zeros((self.num_nodes, self.num_classes), np.float32)
        _abi.check(self._lib.gx_model_forward(self._h, _abi.GX_HOST, _np_ptr(out)))
        return out

    def debug_gang(self, ctas_per_task=0):
        """Test knob: CTAs per task of the streaming kernel (0 automatic, -1 first-generation kernel)."""
        _abi.check(self._lib.gx_debug_set_gang(self._h, int(ctas_per_task)))

    def debug_cluster(self, size=0, min_cost=0):
        """Cluster class of the shared-memory kernel: size 1 = never (default), 0 = latency mode (automatic for batches that leave SMs idle),
        2 / 4 = every task above min_cost (gx_debug_set_cluster)."""
        _abi.check(self._lib.gx_debug_set_cluster(self._h, int(size), int(min_cost)))

    def debug_ieee_edge(self, on=True):
        """Test knob: IEEE exp/div/sqrt in the edge phase instead of the hardware approximations."""
        _abi.check(self._lib.gx_debug_ieee_edge(self._h, int(bool(on))))

    def plan_class_counts(self, with_smem=False):
        """(tasks per launch class [7], cluster size) of the current node plan (gx_plan_class_counts); with_smem: also the largest per-CTA
        shared-memory footprint of each class."""
        counts = np.zeros(7, np.int32)
        smem = np.zeros(7, np.int32)
        cs = np.zeros(1, np.int32)
        _abi.check(self._lib.gx_plan_class_counts(self._h, _np_ptr(counts), _np_ptr(smem), _np_ptr(cs)))
        return (counts, int(cs[0]), smem) if with_smem else (counts, int(cs[0]))

    def last_class_ms(self):
        """(begin_ms[7], end_ms[7]) of the launch classes of the last explain call, relative to its first event (gx_last_class_ms)."""
        b = np.zeros(7, np.float32)
        e = np.zeros(7, np.float32)
        _abi.check(self._lib.gx_last_class_ms(self._h, _np_ptr(b), _np_ptr(e)))
        return b, e

    def launch_count(self):
        return int(self._lib.gx_launch_count(self._h))

    def last_explain_ms(self):
        ms = C.c_float()
        _abi.check(self._lib.gx_last_explain_ms(self._h, C.byref(ms)))
        return float(ms.value)
