"""kernel_spec.py -- TEST INFRASTRUCTURE ONLY (never imported by the product path).

Executable specification of what the CUDA explainer kernels compute, in the form they compute it: parameters on
the directed EDGES only, every layer evaluated only on the rows its receptive field needs, edges split into inner
pairs (optimised with the GCN gradient) and outer pairs (regulariser-only scalar recurrences).  Numpy, any number of
GCN layers, optional --bn.  Its job is to show -- against oracle.explain_closed_form, the dense unpruned restatement
that is pinned to the reference -- that the restructuring is EXACT for every model variant, before a kernel is written
for it (round-1 kernels: 3 layers, no bn; SURVEY 8 f3 lists the others).

Row sets (node mode, L layers, d_i = hop distance of node i from the explained node r):
    layer l (1..L) is needed on R_l = {i : d_i <= L - l}           (layer L: the node's own row only)
    every gather of layer l reads H_{l-1}[j] with d_j <= d_i + 1 <= L - l + 1, i.e. j in R_{l-1}   (R_0 = everything)
    an undirected edge {i,j} receives GCN gradient iff min(d_i, d_j) <= L - 1 (some endpoint is a layer-1 row)
Reference: explainer/explain.py:665-808 (mask, forward, loss), models.py:58-80,222-267 (GraphConv, bn, gcn_forward).
"""
import math

import numpy as np


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def hop_distances(rowptr, col, r, k):
    """BFS distances (0 for r) up to k hops on a local CSR; -1 beyond."""
    n = len(rowptr) - 1
    d = np.full(n, -1, np.int64)
    d[r] = 0
    frontier = [r]
    for lvl in range(1, k + 1):
        nxt = []
        for u in frontier:
            for v in col[rowptr[u]:rowptr[u + 1]]:
                if d[v] < 0:
                    d[v] = lvl
                    nxt.append(int(v))
        frontier = nxt
    return d


def explain_pruned_edges(rowptr, col, X, gt_label, pred_label, r, weights, M0_edges, num_epochs=100, lr=0.1, beta1=0.9,
                         beta2=0.999, eps=1e-8, c_size=0.005, c_feat=1.0, c_ent=1.0, c_lap=1.0, bn=False, dtype=np.float64, return_F=False):
    """rowptr/col: symmetric local CSR of the k-hop sub-adjacency (k = number of layers), no self loops; X (n,d);
    r = node_idx_new; M0_edges[e] = M0[i,j] at CSR slot e.  Returns the mask value of every CSR slot (the entries
    of the reference's masked_adj at the nonzeros of sub_adj, row-major) and a dict of counters; return_F=True also
    returns the feature-mask parameter F after the last update (num_epochs - 1 updates: sigmoid(F) is the feature mask
    the kernels return next to the edge mask)."""
    f = dtype
    n, d = X.shape
    X = np.asarray(X, f)
    Ws, bs = [], []
    l = 1
    while ("W%d" % l) in weights:
        Ws.append(np.asarray(weights["W%d" % l], f))
        b = weights.get("b%d" % l)
        bs.append(np.zeros(Ws[-1].shape[1], f) if b is None else np.asarray(b, f))
        l += 1
    L = len(Ws)
    dims = [w.shape[1] for w in Ws]
    offs = np.concatenate([[0], np.cumsum(dims)])
    Wp = np.asarray(weights["Wp"], f); bp = np.asarray(weights["bp"], f)
    ei = np.repeat(np.arange(n), np.diff(rowptr)); ej = np.asarray(col, np.int64)
    E = len(ej)
    slot = {(int(a), int(b)): e for e, (a, b) in enumerate(zip(ei, ej))}
    rev = np.array([slot[(int(b), int(a))] for a, b in zip(ei, ej)])
    dist = hop_distances(rowptr, col, r, L)
    assert (dist >= 0).all(), "the sub-graph must be the L-hop neighbourhood of r"
    rows = [dist <= L - l for l in range(0, L + 1)]           # rows[l] = R_l as a mask (rows[0] = all)
    erow = [rows[l][ei] for l in range(0, L + 1)]             # edges whose source row is in R_l
    inner = np.minimum(dist[ei], dist[ej]) <= L - 1           # directed slots of inner pairs
    y = np.asarray(pred_label, f)
    lap = (y[ej] ** 2 - y[ei] * y[ej]) / f(n * n) * f(c_lap)  # d/dA_ij of y^T (D - A) y / n^2
    M = np.asarray(M0_edges, f).copy()
    mM = np.zeros(E, f); vM = np.zeros(E, f)
    F = np.zeros(d, f); mF = np.zeros(d, f); vF = np.zeros(d, f)
    a = None
    stats = dict(n=n, E=E, rows_per_layer=[int(rows[l].sum()) for l in range(1, L + 1)], inner_slots=int(inner.sum()),
                 gathered_edges_per_epoch=int(sum(erow[l].sum() for l in range(1, L + 1))))

    def spmm(rowmask, emask, vals, H):                         # Z[i] = sum_{e: ei=i} vals[e] H[ej[e]]   for i in rowmask
        Z = np.zeros((n, H.shape[1]), f)
        np.add.at(Z, ei[emask], vals[emask, None] * H[ej[emask]])
        return Z

    for t in range(1, num_epochs + 1):
        S = _sigmoid(M)
        a = (S + S[rev]) / 2                                   # explain.py:665-678 on the edges
        if t == num_epochs:
            break
        sF = _sigmoid(F)
        H = [X * sF]
        Yh, q, bnst = [], [], []
        for l in range(1, L + 1):
            Rm = rows[l]
            Z = spmm(Rm, erow[l], a, H[-1])
            Y = Z @ Ws[l - 1] + bs[l - 1]
            ql = np.maximum(np.sqrt((Y * Y).sum(1, keepdims=True)), f(1e-12))
            Yl = np.where(Rm[:, None], Y / ql, 0)              # rows outside R_l are never read
            Yh.append(Yl); q.append(ql)
            if l < L:
                Hl = np.maximum(Yl, 0)
                if bn:
                    mu = Hl.mean(1, keepdims=True)
                    istd = 1 / np.sqrt(((Hl - mu) ** 2).mean(1, keepdims=True) + f(1e-5))
                    Hl = np.where(Rm[:, None], (Hl - mu) * istd, 0)
                    bnst.append((Hl, istd))
                H.append(Hl)
            else:
                H.append(Yl)
        emb = np.concatenate([H[l][r] for l in range(1, L + 1)])
        logits = Wp @ emb + bp
        p = np.exp(logits - logits.max()); p /= p.sum()
        g = p.copy(); g[int(gt_label)] -= 1
        dEmb = Wp.T @ g
        dA = np.where(inner, lap, 0)                            # outer slots keep only the regularisers (below)
        dH = np.zeros((n, dims[L - 1]), f)
        for l in range(L, 0, -1):
            Rm = rows[l]
            dYh = dH.copy()
            dYh[r] += dEmb[offs[l - 1]:offs[l]]
            if l < L:
                if bn:
                    Hb, istd = bnst[l - 1]
                    dYh = (dYh - dYh.mean(1, keepdims=True) - Hb * (dYh * Hb).mean(1, keepdims=True)) * istd
                dYh = dYh * (Yh[l - 1] > 0)
            dY = np.where(Rm[:, None], (dYh - Yh[l - 1] * (Yh[l - 1] * dYh).sum(1, keepdims=True)) / q[l - 1], 0)
            dZ = dY @ Ws[l - 1].T
            em = erow[l]
            dA[em] += (dZ[ei[em]] * H[l - 1][ej[em]]).sum(1)   # SDDMM on the edges of the layer's rows
            # dH_{l-1}[j] = sum_{i in R_l} a_ij dZ[i]  (transpose aggregation over the same edges)
            dH = np.zeros((n, H[l - 1].shape[1]), f)
            np.add.at(dH, ej[em], a[em, None] * dZ[ei[em]])
        gF = sF * (1 - sF) * ((X * dH).sum(0) + f(c_feat) / f(d))
        lap_outer = np.where(inner, 0, lap)                     # outer pairs: Laplacian + size + entropy only
        gM = S * (1 - S) * ((dA + dA[rev]) / 2 + (lap_outer + lap_outer[rev]) / 2 + f(c_size) - f(c_ent) * M / f(n * n))
        b1t = 1 - beta1 ** t; b2t = 1 - beta2 ** t
        step = f(lr / b1t); b2s = f(math.sqrt(b2t))
        for P_, G_, m_, v_ in ((M, gM, mM, vM), (F, gF, mF, vF)):
            m_ += (G_ - m_) * f(1 - beta1)
            v_ *= f(beta2); v_ += f(1 - beta2) * G_ * G_
            P_ -= step * m_ / (np.sqrt(v_) / b2s + f(eps))
    return (a, stats, F) if return_F else (a, stats)


def explain_pruned_edges_sparse(rowptr, col, X, gt_label, pred_label, r, weights, M0_edges, num_epochs=5, lr=0.1, beta1=0.9, beta2=0.999,
                                eps=1e-8, c_size=0.005, c_feat=1.0, c_ent=1.0, c_lap=1.0, dtype=np.float64, chunk=1 << 18,
                                return_F=False):
    """explain_pruned_edges for LARGE subgraphs (BASELINE configs[4]: n ~ 10^5, E_d ~ 6.4e6, d = 128): the same pruned edge-list
    mathematics with scipy.sparse SpMM and chunked SDDMM instead of np.add.at over (E, width) temporaries.  3-layer / no-bn model
    (what the streaming kernel implements).  tests/test_oracle.py pins it to explain_pruned_edges (and through it to the dense closed
    form and the reference) on small graphs; bench.py --workload c5 uses it to check the streaming kernel at full scale.
    return_F=True: returns (a, F) with F the feature-mask parameter after the last update, as explain_pruned_edges does."""
    import scipy.sparse as sp
    f = dtype
    n, d = X.shape
    X = np.asarray(X, f)
    Ws = [np.asarray(weights["W%d" % l], f) for l in (1, 2, 3)]
    bs = [np.zeros(Ws[l].shape[1], f) if weights.get("b%d" % (l + 1)) is None else np.asarray(weights["b%d" % (l + 1)], f) for l in range(3)]
    L = 3
    dims = [w.shape[1] for w in Ws]
    offs = np.concatenate([[0], np.cumsum(dims)])
    Wp = np.asarray(weights["Wp"], f); bp = np.asarray(weights["bp"], f)
    rowptr = np.asarray(rowptr, np.int64); ej = np.asarray(col, np.int64)
    ei = np.repeat(np.arange(n, dtype=np.int64), np.diff(rowptr))
    E = len(ej)
    # reverse slot of every directed edge: sort the keys (j, i) -- they enumerate the same set as (i, j) in row-major order
    order = np.lexsort((ei, ej))                      # slots sorted by (ej, ei): position p holds the slot whose (ej,ei) is the p-th (i,j)
    rev = np.empty(E, np.int64); rev[order] = np.arange(E)
    assert np.array_equal(ei[rev], ej) and np.array_equal(ej[rev], ei), "sub-adjacency is not symmetric"
    dist = hop_distances(rowptr, ej, r, L)
    assert (dist >= 0).all()
    rows = [dist <= L - l for l in range(0, L + 1)]
    erow = [rows[l][ei] for l in range(0, L + 1)]
    inner = np.minimum(dist[ei], dist[ej]) <= L - 1
    y = np.asarray(pred_label, f)
    lap = (y[ej] ** 2 - y[ei] * y[ej]) / f(n * n) * f(c_lap)
    M = np.asarray(M0_edges, f).copy()
    mM = np.zeros(E, f); vM = np.zeros(E, f)
    F = np.zeros(d, f); mF = np.zeros(d, f); vF = np.zeros(d, f)

    def masked_csr(vals, emask):
        return sp.csr_matrix((np.where(emask, vals, 0), ej, rowptr), shape=(n, n))

    def sddmm(em, Zl, Hl):
        out = np.zeros(E, f)
        idx = np.nonzero(em)[0]
        for s0 in range(0, len(idx), chunk):
            k = idx[s0:s0 + chunk]
            out[k] = np.einsum("ij,ij->i", Zl[ei[k]], Hl[ej[k]])
        return out

    a = None
    for t in range(1, num_epochs + 1):
        S = _sigmoid(M)
        a = (S + S[rev]) / 2
        if t == num_epochs:
            break
        sF = _sigmoid(F)
        H = [X * sF]
        Yh, q = [], []
        for l in range(1, L + 1):
            Rm = rows[l]
            Z = masked_csr(a, erow[l]) @ H[-1]
            Y = Z @ Ws[l - 1] + bs[l - 1]
            ql = np.maximum(np.sqrt((Y * Y).sum(1, keepdims=True)), f(1e-12))
            Yl = np.where(Rm[:, None], Y / ql, 0)
            Yh.append(Yl); q.append(ql)
            H.append(np.maximum(Yl, 0) if l < L else Yl)
        emb = np.concatenate([H[l][r] for l in range(1, L + 1)])
        logits = Wp @ emb + bp
        p = np.exp(logits - logits.max()); p /= p.sum()
        g = p.copy(); g[int(gt_label)] -= 1
        dEmb = Wp.T @ g
        dA = np.where(inner, lap, 0)
        dH = np.zeros((n, dims[L - 1]), f)
        for l in range(L, 0, -1):
            Rm = rows[l]
            dYh = dH.copy()
            dYh[r] += dEmb[offs[l - 1]:offs[l]]
            if l < L:
                dYh = dYh * (Yh[l - 1] > 0)
            dY = np.where(Rm[:, None], (dYh - Yh[l - 1] * (Yh[l - 1] * dYh).sum(1, keepdims=True)) / q[l - 1], 0)
            dZ = dY @ Ws[l - 1].T
            em = erow[l]
            dA += sddmm(em, dZ, H[l - 1])
            dH = masked_csr(a, em).T @ dZ
        gF = sF * (1 - sF) * ((X * dH).sum(0) + f(c_feat) / f(d))
        lap_outer = np.where(inner, 0, lap)
        gM = S * (1 - S) * ((dA + dA[rev]) / 2 + (lap_outer + lap_outer[rev]) / 2 + f(c_size) - f(c_ent) * M / f(n * n))
        b1t = 1 - beta1 ** t; b2t = 1 - beta2 ** t
        step = f(lr / b1t); b2s = f(math.sqrt(b2t))
        for P_, G_, m_, v_ in ((M, gM, mM, vM), (F, gF, mF, vF)):
            m_ += (G_ - m_) * f(1 - beta1)
            v_ *= f(beta2); v_ += f(1 - beta2) * G_ * G_
            P_ -= step * m_ / (np.sqrt(v_) / b2s + f(eps))
    return (a, F) if return_F else a


def grad_edges_sparse(rowptr, col, X, pred_label_node, r, weights, loops=None, dtype=np.float64, chunk=1 << 18):
    """The gradient baseline (explain.py:125-133,717-738; oracle.grad_closed_form) for subgraphs too large for a dense form:
    scipy.sparse forward / backward on the full sub-adjacency, dL/dA evaluated only at the CSR slots.  rowptr/col: the local CSR
    without the diagonal; loops: optional bool (n,) -- the members with a self loop, whose diagonal entry joins the forward and the
    backward as in the reference's raw sub_adj.  Any number of layers (no --bn).  Returns (slot values, diagonal values) with the
    diagonal values sigmoid(2 |dL/dA_ii|) where loops is set and 0 elsewhere; slot values sigmoid(|dL/dA_ij| + |dL/dA_ji|)."""
    import scipy.sparse as sp
    f = dtype
    n = len(rowptr) - 1
    X = np.asarray(X, f)
    Ws, bs = [], []
    l = 1
    while ("W%d" % l) in weights:
        Ws.append(np.asarray(weights["W%d" % l], f))
        b = weights.get("b%d" % l)
        bs.append(np.zeros(Ws[-1].shape[1], f) if b is None else np.asarray(b, f))
        l += 1
    L = len(Ws)
    dims = [w.shape[1] for w in Ws]
    offs = np.concatenate([[0], np.cumsum(dims)])
    Wp = np.asarray(weights["Wp"], f); bp = np.asarray(weights["bp"], f)
    rowptr = np.asarray(rowptr, np.int64); ej = np.asarray(col, np.int64)
    ei = np.repeat(np.arange(n, dtype=np.int64), np.diff(rowptr))
    E = len(ej)
    order = np.lexsort((ei, ej))
    rev = np.empty(E, np.int64); rev[order] = np.arange(E)
    assert np.array_equal(ei[rev], ej) and np.array_equal(ej[rev], ei), "sub-adjacency is not symmetric"
    assert not (ei == ej).any(), "pass self loops through `loops`"
    dvec = np.zeros(n, f) if loops is None else np.asarray(loops, bool).astype(f)
    A = sp.csr_matrix((np.ones(E, f), ej, rowptr), shape=(n, n)) + sp.diags(dvec)
    H, Yh, q = [X], [], []
    for l in range(L):
        Y = (A @ H[-1]) @ Ws[l] + bs[l]
        ql = np.maximum(np.sqrt((Y * Y).sum(1, keepdims=True)), f(1e-12))
        Yh.append(Y / ql); q.append(ql)
        H.append(np.maximum(Yh[-1], 0) if l < L - 1 else Yh[-1])
    emb = np.concatenate([H[l + 1][r] for l in range(L)])
    logits = Wp @ emb + bp
    p = np.exp(logits - logits.max()); p /= p.sum()
    g = p.copy(); g[int(pred_label_node)] -= 1
    dEmb = Wp.T @ g
    gA = np.zeros(E, f)
    gD = np.zeros(n, f)
    dH = np.zeros((n, dims[L - 1]), f)
    for l in range(L - 1, -1, -1):
        dYh = dH.copy()
        dYh[r] += dEmb[offs[l]:offs[l + 1]]
        if l < L - 1:
            dYh = dYh * (Yh[l] > 0)
        dY = (dYh - Yh[l] * (Yh[l] * dYh).sum(1, keepdims=True)) / q[l]
        dZ = dY @ Ws[l].T
        for s0 in range(0, E, chunk):                          # SDDMM: dL/dA_ij = <dZ_i, H_j> at the slots
            gA[s0:s0 + chunk] += np.einsum("ij,ij->i", dZ[ei[s0:s0 + chunk]], H[l][ej[s0:s0 + chunk]])
        gD += np.einsum("ij,ij->i", dZ, H[l])
        dH = A.T @ dZ
    G = np.abs(gA)
    return _sigmoid(G + G[rev]), np.where(dvec > 0, _sigmoid(2 * np.abs(gD)), 0.0)
