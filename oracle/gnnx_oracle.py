"""gnnx_oracle.py -- CPU restatement of the reference hot path.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may
import this module; the product package (gnn-model-explainer_b200/gnnx) never does and fails
loudly when its CUDA library is missing.

Pinning status: the reference (RexYing/gnn-model-explainer @ bc984829) ships NO tests, golden
vectors or fixtures for this path (SURVEY.md section 4 / 8c), so parity is pinned by executing
the reference itself: tests/golden/*.npz were produced by oracle/gen_golden.py running the
UNMODIFIED reference in the authoring container, and tests/test_oracle.py checks every function
below against them.

Two restatements of the mask optimisation are kept on purpose:
  * explain_dense_torch  -- line-by-line port (dense n x n tensors, torch autograd, torch.optim), i.e. the reference's own
                            cost structure, for every model variant (--bn, any number of layers, attention, MLP heads),
                            unconstrained=True and any dtype; this is the CPU baseline ("port") that bench.py times, and
                            the one port every test compares against.
  * explain_closed_form  -- hand-derived forward/backward in numpy (fp64 or fp32) with parameters
                            that matter only on the directed edges; this is the specification the
                            CUDA kernel implements (SURVEY.md section 8a "validated edge-list spec").
"""
import math
import types

import numpy as np

# ----------------------------------------------------------------------------------------------
# Hyper-parameters: defaults of explainer_main.py:143-167 and ExplainModule.coeffs (explain.py:624-631)
# ----------------------------------------------------------------------------------------------


def default_hparams(**over):
    d = dict(num_epochs=100, lr=0.1, beta1=0.9, beta2=0.999, eps=1e-8,
             size=0.005, feat_size=1.0, ent=1.0, lap=1.0,
             opt="adam", opt_scheduler="none", opt_decay_step=0, opt_decay_rate=1.0, opt_restart=0)   # utils/parser_utils.py:10-19
    d.update(over)
    return types.SimpleNamespace(**d)


# ----------------------------------------------------------------------------------------------
# a1: graph_utils.neighborhoods (utils/graph_utils.py:147-158)
# ----------------------------------------------------------------------------------------------


def neighborhoods_dense(adj, n_hops):
    """adj (B,N,N) 0/1 -> (B,N,N) int: (A + A^2 + ... + A^k) > 0.  Line-by-line restatement
    (float32 matmuls exactly like the reference, utils/graph_utils.py:149-158)."""
    adj = np.asarray(adj, dtype=np.float32)
    hop = power = adj
    for _ in range(n_hops - 1):
        power = power @ adj
        hop = ((hop + power) > 0).astype(np.float32)
    return hop.astype(int)


def csr_from_edges(N, edges):
    """Undirected edge list (m,2) -> symmetric CSR (rowptr int32[N+1], col int32[2m]) with
    ascending columns in every row (the row-major order of np.nonzero on the dense matrix)."""
    e = np.asarray(edges, dtype=np.int64).reshape(-1, 2)
    src = np.concatenate([e[:, 0], e[:, 1]])
    dst = np.concatenate([e[:, 1], e[:, 0]])
    order = np.lexsort((dst, src))
    src, dst = src[order], dst[order]
    rowptr = np.zeros(N + 1, dtype=np.int64)
    np.add.at(rowptr, src + 1, 1)
    rowptr = np.cumsum(rowptr)
    return rowptr.astype(np.int32), dst.astype(np.int32)


def csr_from_dense(adj):
    adj = np.asarray(adj)
    N = adj.shape[0]
    ei, ej = np.nonzero(adj)
    rowptr = np.zeros(N + 1, dtype=np.int64)
    np.add.at(rowptr, ei + 1, 1)
    return np.cumsum(rowptr).astype(np.int32), ej.astype(np.int32)


def dense_from_csr(rowptr, col, N=None):
    N = len(rowptr) - 1 if N is None else N
    A = np.zeros((N, N), dtype=np.float64)
    for i in range(N):
        A[i, col[rowptr[i]:rowptr[i + 1]]] = 1.0
    return A


def khop_walk_set(rowptr, col, node, k):
    """Set {j : exists a walk of length 1..k from node to j}, ascending, as the reference's dense
    matrix powers define it (utils/graph_utils.py:152-157): integer frontier expansion where the
    start node is NOT pre-marked (it is a member only if a closed walk of length <= k exists)."""
    N = len(rowptr) - 1
    seen = np.zeros(N, dtype=bool)
    frontier = np.array([node], dtype=np.int64)
    for _ in range(k):
        nxt = []
        for u in frontier:
            for v in col[rowptr[u]:rowptr[u + 1]]:
                if not seen[v]:
                    seen[v] = True
                    nxt.append(v)
        frontier = np.array(nxt, dtype=np.int64)
        if len(frontier) == 0:
            break
    return np.nonzero(seen)[0].astype(np.int32)


# ----------------------------------------------------------------------------------------------
# a2: Explainer.extract_neighborhood (explainer/explain.py:492-501)
# ----------------------------------------------------------------------------------------------


def extract_neighborhood(rowptr, col, feat, label, node, k):
    """-> (node_idx_new, sub_rowptr, sub_col, sub_feat, sub_label, neighbors).  The induced
    sub-adjacency is returned as canonical CSR (rows/cols = rank among the ascending neighbours),
    which is the row-major nonzero order of the reference's dense sub_adj."""
    nbrs = khop_walk_set(rowptr, col, node, k)
    node_idx_new = int(np.searchsorted(nbrs, node))       # == sum(row[:node_idx]) (explain.py:496)
    N = len(rowptr) - 1
    loc = -np.ones(N, dtype=np.int64)
    loc[nbrs] = np.arange(len(nbrs))
    sub_rowptr = [0]
    sub_col = []
    for g in nbrs:
        c = loc[col[rowptr[g]:rowptr[g + 1]]]
        c = c[c >= 0]
        sub_col.append(c)
        sub_rowptr.append(sub_rowptr[-1] + len(c))
    sub_col = np.concatenate(sub_col) if sub_col else np.zeros(0, np.int64)
    return (node_idx_new, np.asarray(sub_rowptr, np.int32), sub_col.astype(np.int32),
            np.asarray(feat)[nbrs], np.asarray(label)[nbrs], nbrs)


def draw_m0(n, seed=None):
    """ExplainModule.construct_edge_mask (explain.py:645-652): FloatTensor(n,n).normal_(1, std),
    std = gain('relu') * sqrt(2/(n+n)).  Consumes exactly n*n normals of torch's global CPU RNG."""
    import torch
    if seed is not None:
        torch.manual_seed(seed)
    std = torch.nn.init.calculate_gain("relu") * math.sqrt(2.0 / (n + n))
    return torch.FloatTensor(n, n).normal_(1.0, std).numpy()


# ----------------------------------------------------------------------------------------------
# The kernels' device init (GX_INIT_PHILOX, csrc/explain_common.cuh): Philox4x32-10 (Salmon et al. 2011,
# the Random123 philox4x32 with 10 rounds) and one Box-Muller normal per (seed, key, slot)
# ----------------------------------------------------------------------------------------------
_MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: 4 uint32 words (scalars or equal-length arrays), key: 2 uint32 words -> the 4 output words (uint32 arrays)."""
    c = [np.asarray(x, dtype=np.uint64) & _MASK32 for x in ctr]
    k0, k1 = (np.asarray(x, dtype=np.uint64) & _MASK32 for x in key)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & _MASK32
        hi1, lo1 = p1 >> np.uint64(32), p1 & _MASK32
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0 = (k0 + np.uint64(0x9E3779B9)) & _MASK32
        k1 = (k1 + np.uint64(0xBB67AE85)) & _MASK32
    return [x.astype(np.uint32) for x in c]


def philox_normal(seed, key, slot):
    """N(0,1) the kernels draw for (seed, key, slot), in float64: counter (slot, key, 0x67, 0x6e78), key (seed lo, seed hi),
    Box-Muller on the top 24 bits of the first two output words."""
    slot = np.asarray(slot, dtype=np.uint64)
    seed = int(seed)
    r = philox4x32_10((slot, np.full_like(slot, key), np.full_like(slot, 0x67), np.full_like(slot, 0x6E78)),
                      (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))
    u1 = ((r[0] >> np.uint32(8)).astype(np.float64) + 0.5) / 16777216.0
    u2 = ((r[1] >> np.uint32(8)).astype(np.float64) + 0.5) / 16777216.0
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def philox_m0(seed, key, num_slots, n):
    """The M0 entries GX_INIT_PHILOX draws for one task, float64 [num_slots], slot = position in the task's edge arrays:
    1 + sqrt(2/n) * philox_normal(seed, key, slot), i.e. N(1, gain('relu')^2 * 2/(n+n)) as construct_edge_mask draws.
    Node mode: key = the explained node's id, n = its neighbourhood size, slots in canonical (row-major) order.
    Graph mode: key = the graph id, n = max_nodes (the padded size), slots in the order of the graph's CSR."""
    return 1.0 + math.sqrt(2.0 / n) * philox_normal(seed, key, np.arange(num_slots))


# ----------------------------------------------------------------------------------------------
# a3..a12, line-by-line port: dense tensors + autograd + torch.optim.Adam
# ----------------------------------------------------------------------------------------------


_POOL = [None]


def max_pool(outs):
    """The graph readout's per-layer max over rows (models.py:283,293,304): torch.max, whose backward routes each column's gradient to
    its first maximal row.  Every graph-mode port pools here; set_pool(fn) makes fn(outs) pool instead (tests/pool_oracle.py forces and
    records those arg-max choices)."""
    import torch
    if _POOL[0] is not None:
        return _POOL[0](outs)
    return [torch.max(o, dim=1)[0] for o in outs]


def set_pool(fn):
    """Installs fn (None: torch.max) as max_pool's readout; returns the previous one."""
    prev, _POOL[0] = _POOL[0], fn
    return prev


def _gcn_forward_torch(x, adj, W, graph_mode, bn=False):
    """models.py:58-80 (GraphConv.forward), :230-267 (gcn_forward), :363-376 (node readout),
    :269-316 (graph readout), :193-207 (pred_model).  x (1,n,d), adj (1,n,n).  Any number of layers (len(W["conv_w"]) =
    args.num_gc_layers).  bn=True: models.py:222-228,242-243,252-253 -- a FRESH BatchNorm1d(n) in train mode
    after the ReLU of every layer but the last, i.e. each node's row is standardised over its features
    (biased variance, eps 1e-5, no affine).  W["att_w"] (--method att): every layer scales the adjacency it is given by the
    unnormalised scores P P^T, P = H_{l-1} Wa_l (models.py:62-68).  W["head"] (pred_hidden_dims): Linear, ReLU, .. before the last
    Linear (W["pred_w"], W["pred_b"])."""
    import torch
    import torch.nn.functional as F
    outs = []
    h = x
    L = len(W["conv_w"])
    for l in range(L):
        a = adj
        if W.get("att_w") is not None:
            x_att = torch.matmul(h, W["att_w"][l])     # models.py:63
            a = adj * (x_att @ x_att.permute(0, 2, 1))  # models.py:66-68
        y = torch.matmul(a, h)                         # models.py:70
        y = torch.matmul(y, W["conv_w"][l])            # models.py:71
        if W["conv_b"][l] is not None:
            y = y + W["conv_b"][l]                     # models.py:76
        y = F.normalize(y, p=2, dim=2)                 # models.py:78
        if l < L - 1:
            y = torch.relu(y)                          # models.py:241,251 (not on the last layer)
            if bn:
                y = F.batch_norm(y, None, None, None, None, True, 0.1, 1e-5)   # BatchNorm1d(n)(x) on (1,n,h): channels = nodes
        outs.append(y)
        h = y
    if graph_mode:
        emb = torch.cat(max_pool(outs), dim=1)                     # models.py:283,293,304,309
    else:
        emb = torch.cat(outs, dim=2)                               # models.py:260
    for w, b in W.get("head", ()):
        emb = torch.relu(F.linear(emb, w, b))                      # models.py:193-207
    return F.linear(emb, W["pred_w"], W["pred_b"])                 # (1,C) graph mode, (1,n,C) node mode (models.py:375)


def head_layers(weights):
    """The hidden head Linears [(W, b), ..]: weights["head"], or the fixture's Wh1 / bh1, Wh2 / bh2, .."""
    if "head" in weights:
        return list(weights["head"])
    out, j = [], 1
    while ("Wh%d" % j) in weights:
        out.append((weights["Wh%d" % j], weights["bh%d" % j]))
        j += 1
    return out


def weights_to_torch(weights, requires_grad=True, dtype=None):
    """weights: dict with W1,b1,..,WL,bL,Wp,bp (numpy) -> the structure _gcn_forward_torch uses, in dtype (None: torch.float).
    Wa1..WaL (attention) become "att_w"; the head's hidden Linears (head_layers, torch's (out, in) layout) become "head", and Wp / bp
    are then the last Linear.  requires_grad=True mirrors the reference, whose frozen model is a registered sub-module of
    ExplainModule (explain.py:598) so autograd also computes the (unused) weight gradients."""
    import torch
    t = lambda a: torch.tensor(np.asarray(a), dtype=dtype or torch.float, requires_grad=requires_grad)
    conv_w, conv_b = [], []
    l = 1
    while ("W%d" % l) in weights:
        conv_w.append(t(weights["W%d" % l]))
        b = weights.get("b%d" % l)
        conv_b.append(None if b is None else t(b))
        l += 1
    W = dict(conv_w=conv_w, conv_b=conv_b, pred_w=t(weights["Wp"]), pred_b=t(weights["bp"]))
    if "Wa1" in weights:
        W["att_w"] = [t(weights["Wa%d" % l]) for l in range(1, len(conv_w) + 1)]
    head = head_layers(weights)
    if head:
        W["head"] = [(t(w), t(b)) for w, b in head]
    return W


def model_pred(adj, feat, weights, bn=False, graph_mode=False):
    """GcnEncoderNode / GcnEncoderGraph.forward on the raw adjacency (self loops included): the `pred` of the checkpoint, float32."""
    import torch
    with torch.no_grad():
        return _gcn_forward_torch(torch.tensor(np.asarray(feat, np.float32)[None]), torch.tensor(np.asarray(adj, np.float32)[None]),
                                  weights_to_torch(weights, requires_grad=False), graph_mode, bn)[0].numpy()


def build_optimizer(hp, params):
    """utils/train_utils.py:7-23 (build_optimizer; explain.py:622) -> (optimizer, scheduler or None)."""
    import torch
    if hp.opt == "adam":
        opt = torch.optim.Adam(params, lr=hp.lr, betas=(hp.beta1, hp.beta2), eps=hp.eps)
    elif hp.opt == "sgd":
        opt = torch.optim.SGD(params, lr=hp.lr, momentum=0.95)
    elif hp.opt == "rmsprop":
        opt = torch.optim.RMSprop(params, lr=hp.lr)
    elif hp.opt == "adagrad":
        opt = torch.optim.Adagrad(params, lr=hp.lr)
    else:
        raise ValueError(hp.opt)
    sched = None
    if hp.opt_scheduler == "step":
        sched = torch.optim.lr_scheduler.StepLR(opt, step_size=hp.opt_decay_step, gamma=hp.opt_decay_rate)
    elif hp.opt_scheduler == "cos":
        sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=hp.opt_restart)
    return opt, sched


def _sym(mask):
    import torch
    sym = torch.sigmoid(mask)                                                   # explain.py:671-676
    return (sym + sym.t()) / 2


def _epoch_loss(mask, feat_mask, adj, x, diag_mask, W, gt_label, pred_label_t, node_idx_new, hp, graph_mode=False, bn=False,
                unconstrained=False):
    """ExplainModule.{_masked_adj,forward,loss} (explain.py:665-808) at mask parameters `mask` (n,n) and `feat_mask` (d,):
    adj (1,n,n), x (1,n,d), diag_mask (n,n), pred_label_t (n,) the Laplacian term's labels (node mode).
    The operations run in the reference's order: autograd sums a tensor's gradient contributions in the order of their creation, so
    the order is part of the bits.  In particular sigmoid(feat_mask) and sigmoid(mask) are evaluated afresh for the regularisers.
    unconstrained=True: the forward's adjacency is the dense sym(sigmoid(M)) (.) (1 - I) and the features are not masked
    (explain.py:688-692).  Returns (loss, masked_adj, res, terms) with res the softmax the prediction loss reads and terms the
    loss terms plus m = sigmoid(mask), mask_ent (n,n) and fm = sigmoid(feat_mask)."""
    import torch
    sym = _sym(mask)
    if unconstrained:
        masked_adj = torch.unsqueeze(sym, 0) * diag_mask                        # explain.py:688-692
        ypred = _gcn_forward_torch(x, masked_adj, W, graph_mode, bn)            # explain.py:709, raw features
    else:
        masked_adj = adj * sym * diag_mask                                      # explain.py:678,694
        ypred = _gcn_forward_torch(x * torch.sigmoid(feat_mask), masked_adj, W, graph_mode, bn)   # explain.py:695-709
    if graph_mode:
        res = torch.softmax(ypred[0], dim=0)                                    # explain.py:711
    else:
        res = torch.softmax(ypred[-1, node_idx_new, :], dim=0)                  # explain.py:713-714
    pred_loss = -torch.log(res[int(gt_label)])                                  # explain.py:750-753
    m = torch.sigmoid(mask)                                                     # explain.py:756-757
    size_loss = hp.size * torch.sum(m)                                          # explain.py:760
    fm = torch.sigmoid(feat_mask)
    feat_size_loss = hp.feat_size * torch.mean(fm)                              # explain.py:764-766
    mask_ent = -m * torch.log(m) - (1 - m) * torch.log(1 - m)                   # explain.py:769
    mask_ent_loss = hp.ent * torch.mean(mask_ent)                               # explain.py:770
    if graph_mode:
        lap_loss = 0                                                            # explain.py:787-788
    else:
        D = torch.diag(torch.sum(masked_adj[0], 0))                             # explain.py:780
        Lm = D - masked_adj[-1]                                                 # explain.py:781-782
        lap_loss = hp.lap * (pred_label_t @ Lm @ pred_label_t) / adj.numel()    # explain.py:789-793
    loss = pred_loss + size_loss + lap_loss + mask_ent_loss + feat_size_loss    # explain.py:808
    terms = dict(pred_loss=pred_loss, size=size_loss, feat_size=feat_size_loss, ent=mask_ent_loss, lap=lap_loss, m=m, mask_ent=mask_ent,
                 fm=fm)
    return loss, masked_adj, res, terms


def explain_dense_torch(sub_adj, sub_feat, gt_label, pred_label, node_idx_new, weights, M0, hp=None, graph_mode=False, trace=None,
                        bn=False, return_feat=False, dtype=None, unconstrained=False, full=False):
    """Port of Explainer.explain's optimisation (explain.py:97-146,209-211) with
    ExplainModule.{_masked_adj,forward,loss,mask_density} (explain.py:665-808) inlined, in dtype (None: torch.float), for every model
    _gcn_forward_torch runs (weights as weights_to_torch reads them, or already converted).

    sub_adj (n,n) 0/1; sub_feat (n,d); gt_label = label[0][node_idx] (node) or the graph label;
    pred_label (n,) int = argmax(pred[nbrs]) (node mode; unused in graph mode); M0 (n,n) float32.
    unconstrained=True: Explainer.explain(..., unconstrained=True), every entry of M0 a parameter (_epoch_loss).
    Returns the (n,n) float64 array the reference returns (masked_adj[0] * sub_adj), with full=True the whole masked_adj[0];
    return_feat=True also returns sigmoid(feat_mask) as the last epoch's forward used it (after num_epochs - 1 updates), float64 (d,).
    trace: list receiving per epoch what print_training prints (loss, density, pred; explain.py:148-159) and the terms it is made
    of; size_edges / ent_edges restrict the size and entropy terms to the entries of the sub-adjacency (the only mask entries that
    can reach the constrained result), size_off / ent_off are the complement.  density is mask_density, which keeps the
    constrained _masked_adj in both modes (explain.py:680-683)."""
    import torch
    hp = hp or default_hparams()
    dtype = dtype or torch.float
    W = weights if isinstance(weights, dict) and "conv_w" in weights else weights_to_torch(weights, dtype=dtype)
    n = sub_adj.shape[0]
    adj = torch.tensor(np.asarray(sub_adj)[None], dtype=dtype)                             # explain.py:97
    x = torch.tensor(np.asarray(sub_feat)[None], requires_grad=True, dtype=dtype)          # :98
    mask = torch.nn.Parameter(torch.tensor(np.asarray(M0), dtype=dtype))                   # explain.py:646-652
    feat_mask = torch.nn.Parameter(torch.zeros(x.size(-1), dtype=dtype))                   # explain.py:633-643
    diag_mask = torch.ones(n, n, dtype=dtype) - torch.eye(n, dtype=dtype)                  # explain.py:617
    opt, sched = build_optimizer(hp, [mask, feat_mask])
    pred_label_t = None if graph_mode else torch.tensor(np.asarray(pred_label), dtype=dtype)
    # explainer.zero_grad() (explain.py:138) clears the frozen model's weight gradients too: it is a sub-module
    leaves = ([mask, feat_mask, x] + W["conv_w"] + [b for b in W["conv_b"] if b is not None] + W.get("att_w", [])
              + [p for layer in W.get("head", ()) for p in layer] + [W["pred_w"], W["pred_b"]])
    masked_adj = terms = None
    for epoch in range(hp.num_epochs):                                                     # explain.py:137
        for p in leaves:
            p.grad = None
        loss, masked_adj, res, terms = _epoch_loss(mask, feat_mask, adj, x, diag_mask, W, gt_label, pred_label_t, node_idx_new, hp,
                                                   graph_mode, bn, unconstrained)
        loss.backward()                                                                    # explain.py:142
        opt.step()                                                                         # explain.py:144
        if sched is not None:
            sched.step()                                                                   # explain.py:145-146
        if trace is not None:
            with torch.no_grad():
                density = torch.sum(adj * _sym(mask) * diag_mask) / torch.sum(adj)         # explain.py:148,680-683
                on = adj[0] > 0
                m, ent = terms["m"], terms["mask_ent"]
                trace.append(dict(loss=float(loss), density=float(density), pred=res.detach().numpy().copy(),
                                  pred_loss=float(terms["pred_loss"]), lap=float(terms["lap"]), feat_size=float(terms["feat_size"]),
                                  size=float(terms["size"]), ent=float(terms["ent"]),
                                  size_edges=float(hp.size * torch.sum(m[on])), size_off=float(hp.size * torch.sum(m[~on])),
                                  ent_edges=float(hp.ent * torch.sum(ent[on]) / adj.numel()),
                                  ent_off=float(hp.ent * torch.sum(ent[~on]) / adj.numel())))
    out = masked_adj[0].detach().numpy().astype(np.float64)
    if not full:
        out = out * np.asarray(sub_adj, dtype=np.float64)                                  # explain.py:209-211
    if return_feat:
        return out, terms["fm"].detach().numpy().astype(np.float64)
    return out


# ----------------------------------------------------------------------------------------------
# closed form (the kernel's specification), numpy
# ----------------------------------------------------------------------------------------------


def grad_baseline_dense_torch(sub_adj, sub_feat, pred_label_node, node_idx_new, weights, dtype=np.float32):
    """The reference's gradient baseline, Explainer.explain(model="grad") (explain.py:125-133) with
    ExplainModule.adj_feat_grad (explain.py:717-738), restated: one forward of the frozen model on the UNMASKED
    sub-adjacency and features (diagonal included: the reference uses the raw sub_adj), loss = -log softmax(logits[node])
    [predicted label of the node], one backward w.r.t. the dense adjacency; result sigmoid(|dA| + |dA|^T) * A.
    dtype=np.float64: the same autograd computation in double precision (inputs and weights cast)."""
    import torch
    tdt = torch.float64 if dtype == np.float64 else torch.float
    A = torch.tensor(np.asarray(sub_adj, dtype)[None], dtype=tdt, requires_grad=True)
    x = torch.tensor(np.asarray(sub_feat, dtype)[None], dtype=tdt, requires_grad=True)
    ypred = _gcn_forward_torch(x, A, weights_to_torch(weights, dtype=tdt), False)
    logit = torch.softmax(ypred[0, node_idx_new, :], dim=0)[int(pred_label_node)]
    loss = -torch.log(logit)
    loss.backward()
    g = torch.abs(A.grad)[0]
    m = torch.sigmoid(g + g.t())
    return m.detach().numpy() * np.asarray(sub_adj, dtype)


def grad_closed_form(sub_adj, sub_feat, pred_label_node, node_idx_new, weights, dtype=np.float64, return_grad=False):
    """Hand-derived form of grad_baseline_dense_torch, numpy, any number of layers (no --bn).  The forward runs on sub_adj AS
    GIVEN -- the reference's raw sub-adjacency, so a self loop (diagonal entry) takes part in the forward and the backward and
    gets its own result entry sigmoid(2 |dL/dA_ii|).  dL/dA = sum_l dZ_l H_{l-1}^T with dZ_l the gradient at A H_{l-1}.
    Returns the (n, n) result sigmoid(|dA| + |dA|^T) * A; return_grad=True also returns dA."""
    f = dtype
    A = np.asarray(sub_adj, dtype=f)
    X = np.asarray(sub_feat, dtype=f)
    n = A.shape[0]
    Ws, bs = [], []
    l = 1
    while ("W%d" % l) in weights:
        Ws.append(np.asarray(weights["W%d" % l], dtype=f))
        b = weights.get("b%d" % l)
        bs.append(np.zeros(Ws[-1].shape[1], f) if b is None else np.asarray(b, dtype=f))
        l += 1
    L = len(Ws)
    dims = [w.shape[1] for w in Ws]
    offs = np.concatenate([[0], np.cumsum(dims)])
    Wp = np.asarray(weights["Wp"], dtype=f)
    bp = np.asarray(weights["bp"], dtype=f)
    r = int(node_idx_new)
    H, Yh, q = [X], [], []
    for l in range(L):
        Y = (A @ H[-1]) @ Ws[l] + bs[l]                                             # models.py:70-76
        ql = np.maximum(np.sqrt((Y * Y).sum(1, keepdims=True)), f(1e-12))           # F.normalize eps
        Yh.append(Y / ql); q.append(ql)
        H.append(np.maximum(Yh[-1], 0) if l < L - 1 else Yh[-1])
    emb = np.concatenate([H[l + 1][r] for l in range(L)])
    logits = Wp @ emb + bp
    p = np.exp(logits - logits.max()); p = p / p.sum()
    g = p.copy(); g[int(pred_label_node)] -= 1                                      # d(-log p[pred_label])/dlogits
    dEmb = Wp.T @ g
    dA = np.zeros((n, n), f)
    dH = np.zeros((n, dims[L - 1]), f)
    for l in range(L - 1, -1, -1):
        dYh = dH.copy()
        dYh[r] += dEmb[offs[l]:offs[l + 1]]
        if l < L - 1:
            dYh = dYh * (Yh[l] > 0)
        dY = (dYh - Yh[l] * (Yh[l] * dYh).sum(1, keepdims=True)) / q[l]             # backward of x / max(|x|, eps)
        dZ = dY @ Ws[l].T
        dA += dZ @ H[l].T
        dH = A.T @ dZ
    G = np.abs(dA)
    out = _sigmoid(G + G.T) * A
    return (out, dA) if return_grad else out


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def explain_closed_form(sub_adj, sub_feat, gt_label, pred_label, node_idx_new, weights, M0,
                        hp=None, graph_mode=False, dtype=np.float64, return_state=False, bn=False, init_state=None):
    """Hand-derived forward/backward (SURVEY.md section 8a), any number of layers; bn=True adds the per-node
    standardisation of models.py:222-228 after every hidden layer's ReLU (forward and its backward).  Dense numpy arrays are used for
    brevity, but only the edge entries of M carry information: off-edge entries never influence
    the returned array.  Derivation notes next to each line cite what autograd differentiates."""
    hp = hp or default_hparams()
    f = dtype
    A = np.asarray(sub_adj, dtype=f)
    A = A * (1 - np.eye(A.shape[0], dtype=f))             # diag_mask (explain.py:617,678)
    X = np.asarray(sub_feat, dtype=f)
    n, d = X.shape
    Ws, bs = [], []
    l = 1
    while ("W%d" % l) in weights:
        Ws.append(np.asarray(weights["W%d" % l], dtype=f))
        b = weights.get("b%d" % l)
        bs.append(np.zeros(Ws[-1].shape[1], f) if b is None else np.asarray(b, dtype=f))
        l += 1
    L = len(Ws)
    dims = [w.shape[1] for w in Ws]
    offs = np.concatenate([[0], np.cumsum(dims)])
    Wp = np.asarray(weights["Wp"], dtype=f)
    bp = np.asarray(weights["bp"], dtype=f)
    C = Wp.shape[0]
    r = int(node_idx_new)
    M = np.asarray(M0, dtype=f).copy()
    mM = np.zeros_like(M); vM = np.zeros_like(M)
    F = np.zeros(d, f); mF = np.zeros(d, f); vF = np.zeros(d, f)
    step0 = 0
    if init_state is not None:     # resume / teacher forcing: (m, v) dense like M0, feat = (3,d) [F, exp_avg, exp_avg_sq], step = Adam steps taken
        mM = np.asarray(init_state["m"], dtype=f).copy(); vM = np.asarray(init_state["v"], dtype=f).copy()
        F, mF, vF = (np.asarray(init_state["feat"][k], dtype=f).copy() for k in range(3))
        step0 = int(init_state["step"])
    if not graph_mode:
        y = np.asarray(pred_label, dtype=f)
        lapA = (y[None, :] ** 2 - y[:, None] * y[None, :]) / f(n * n) * f(hp.lap)   # d/dA_ij of y^T(D-A)y/n^2
    else:
        lapA = np.zeros((n, n), f)
    a = None
    for t in range(1, hp.num_epochs + 1):
        S = _sigmoid(M)
        a = A * (S + S.T) / 2                                                       # explain.py:665-678
        if t == hp.num_epochs and not return_state:
            break
        sF = _sigmoid(F)
        H = [X * sF]
        Yh, q = [], []
        bn_state = []
        for l in range(L):
            Y = (a @ H[-1]) @ Ws[l] + bs[l]                                         # models.py:70-76
            ql = np.maximum(np.sqrt((Y * Y).sum(1, keepdims=True)), f(1e-12))       # F.normalize eps
            Yl = Y / ql
            Yh.append(Yl); q.append(ql)
            if l < L - 1:
                Hl = np.maximum(Yl, 0)
                if bn:                                                                 # BatchNorm1d(n), train mode, no affine
                    mu = Hl.mean(1, keepdims=True)
                    istd = 1 / np.sqrt(((Hl - mu) ** 2).mean(1, keepdims=True) + f(1e-5))
                    Hl = (Hl - mu) * istd
                    bn_state.append((Hl, istd))
                H.append(Hl)
            else:
                H.append(Yl)
        dE = [np.zeros((n, dims[l]), f) for l in range(L)]
        if graph_mode:
            pooled = [H[l + 1].max(0) for l in range(L)]
            arg = [H[l + 1].argmax(0) for l in range(L)]          # first max index, like torch.max
            emb = np.concatenate(pooled)
        else:
            emb = np.concatenate([H[l + 1][r] for l in range(L)])
        logits = Wp @ emb + bp
        p = np.exp(logits - logits.max()); p = p / p.sum()
        g = p.copy(); g[int(gt_label)] -= 1                                          # d(-log p[gt])/dlogits
        dEmb = Wp.T @ g
        for l in range(L):
            sl = dEmb[offs[l]:offs[l + 1]]
            if graph_mode:
                dE[l][arg[l], np.arange(dims[l])] += sl
            else:
                dE[l][r] += sl
        dA = lapA.copy()
        dH = np.zeros((n, dims[L - 1]), f)
        for l in range(L - 1, -1, -1):
            dYh = dE[l] + dH
            if l < L - 1:
                if bn:                                                                 # backward of the row standardisation
                    Hb, istd = bn_state[l]
                    dYh = (dYh - dYh.mean(1, keepdims=True) - Hb * (dYh * Hb).mean(1, keepdims=True)) * istd
                dYh = dYh * (Yh[l] > 0)
            dY = (dYh - Yh[l] * (Yh[l] * dYh).sum(1, keepdims=True)) / q[l]          # backward of x/max(|x|,eps)
            dZ = dY @ Ws[l].T
            dA += dZ @ H[l].T
            dH = a.T @ dZ
        gF = sF * (1 - sF) * ((X * dH).sum(0) + f(hp.feat_size) / f(d))              # explain.py:766 mean -> 1/d
        # masked_adj = A * (S + S^T)/2 ; size = c*sum(S) ; ent = mean(H(S)) over ALL n^2 entries
        gM = S * (1 - S) * ((A * dA + (A * dA).T) / 2 + f(hp.size) - f(hp.ent) * M / f(n * n))
        b1t = 1 - hp.beta1 ** (step0 + t); b2t = 1 - hp.beta2 ** (step0 + t)
        step = f(hp.lr / b1t); b2s = f(math.sqrt(b2t))
        for P, G, m_, v_ in ((M, gM, mM, vM), (F, gF, mF, vF)):
            m_ += (G - m_) * f(1 - hp.beta1)                                         # exp_avg.lerp_
            v_ *= f(hp.beta2); v_ += f(1 - hp.beta2) * G * G
            P -= step * m_ / (np.sqrt(v_) / b2s + f(hp.eps))
    out = a.astype(np.float64) * np.asarray(sub_adj, dtype=np.float64)
    if return_state:
        # M, F and the Adam moments after num_epochs updates; init_state=dict(m=mM, v=vM, feat=(F, mF, vF), step=...) resumes from them
        return out, dict(M=M, F=F, gM=gM, gF=gF, p=p, mM=mM, vM=vM, mF=mF, vF=vF)
    return out


def rel_l2(a, b):
    a = np.asarray(a, dtype=np.float64).ravel(); b = np.asarray(b, dtype=np.float64).ravel()
    den = np.linalg.norm(b)
    return float(np.linalg.norm(a - b) / den) if den > 0 else float(np.linalg.norm(a - b))
