"""dense_oracle.py -- the hand-derived restatement of Explainer.explain(..., unconstrained=True).  TEST INFRASTRUCTURE ONLY.

With unconstrained=True (ExplainModule.forward, explain.py:688-692) the forward's adjacency is the DENSE mask
sym(sigmoid(M)) * (1 - I), not multiplied by the sub-adjacency, and the features are not masked.  The line-by-line torch port of
that path is gnnx_oracle.explain_dense_torch(..., unconstrained=True), bit-exact to the unmodified reference
(tests/golden/unconstrained_golden.npz, tools/gen_unconstrained_golden.py); here:
  * explain_closed_form  -- hand-derived forward / backward in numpy (fp64 or fp32): the specification csrc/explain_dense.cu implements.
It returns the (n, n) float64 array the reference returns, masked_adj[0] * sub_adj (explain.py:209-211), or with full=True the whole
masked_adj[0] ExplainModule.forward built (the kernel's mask_dense output).
"""
import math

import numpy as np

import gnnx_oracle as O


def entry_classes(A):
    """The off-diagonal entries of an (n, n) dense mask by class, {name: (rows, cols)}: "edge" the sub-adjacency slots, "nonedge" the
    other pairs of rows that have an edge, "pad" the pairs with a row that has none (graph mode's padding and isolated rows).  Empty
    classes are left out."""
    A = np.asarray(A)
    n = len(A)
    live = (A != 0).any(1)
    off = ~np.eye(n, dtype=bool)
    both = live[:, None] & live[None, :]
    cls = {"edge": off & (A != 0), "nonedge": off & (A == 0) & both, "pad": off & ~both}
    return {k: np.nonzero(v) for k, v in cls.items() if v.any()}


def _lr_at(hp, t):
    """Learning rate of update t (1-based) under the scheduler, stepped once per epoch after the optimiser (explain.py:144-146)."""
    e = t - 1
    if hp.opt_scheduler == "step":
        return hp.lr * hp.opt_decay_rate ** (e // hp.opt_decay_step)
    if hp.opt_scheduler == "cos":
        return hp.lr * 0.5 * (1.0 + math.cos(math.pi * e / hp.opt_restart))
    return hp.lr


def _opt_update(hp, t, f, P, G, m_, v_):
    """One in-place update of utils/train_utils.py:7-23's optimisers (torch defaults; SGD momentum 0.95) at update t."""
    lr = _lr_at(hp, t)
    if hp.opt == "adam":
        b1t = 1 - hp.beta1 ** t; b2t = 1 - hp.beta2 ** t
        m_ += (G - m_) * f(1 - hp.beta1)
        v_ *= f(hp.beta2); v_ += f(1 - hp.beta2) * G * G
        P -= f(lr / b1t) * m_ / (np.sqrt(v_) / f(math.sqrt(b2t)) + f(hp.eps))
    elif hp.opt == "sgd":
        m_ *= f(0.95); m_ += G
        P -= f(lr) * m_
    elif hp.opt == "rmsprop":
        v_ *= f(0.99); v_ += f(0.01) * G * G
        P -= f(lr) * G / (np.sqrt(v_) + f(1e-8))
    elif hp.opt == "adagrad":
        v_ += G * G
        P -= f(lr) * G / (np.sqrt(v_) + f(1e-10))
    else:
        raise ValueError(hp.opt)


def explain_closed_form(sub_adj, sub_feat, gt_label, pred_label, node_idx_new, weights, M0, hp=None, graph_mode=False, dtype=np.float64,
                        return_state=False, bn=False, full=False, trace=None):
    """Hand-derived forward / backward of the unconstrained optimisation, any number of layers, --bn, an MLP prediction head
    (weights["head"] = [(W, b), ..], torch's (out, in) layout, models.py:193-207), every optimiser and scheduler.
    The forward's adjacency is a = (1 - I) (.) (S + S^T)/2 with S = sigmoid(M) over all n^2 entries, the features are unmasked (so F is
    moved by feat_size alone), the Laplacian term covers every pair (node mode).  return_state=True also returns M, F and the
    one-step gradients gM, gF of the last update (with num_epochs=1: the gradients at M0, F = 0).  full=True returns the whole a
    instead of a (.) sub_adj.  trace: list receiving per epoch dict(a=the epoch's dense mask, size=sum sigmoid(M), ent=sum H(sigmoid(M))
    over all n^2 entries, feat=sum sigmoid(F)), the sums of the loss terms the kernel's trace reports (before that epoch's update), and
    gM, the gradient of that epoch's update (absent from the last epoch unless return_state)."""
    hp = hp or O.default_hparams()
    f = dtype
    X = np.asarray(sub_feat, dtype=f)
    n, d = X.shape
    A = 1 - np.eye(n, dtype=f)                                                     # diag_mask (explain.py:617,692)
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
    head = [(np.asarray(w, dtype=f), np.asarray(b, dtype=f)) for w, b in weights.get("head", [])]
    r = int(node_idx_new)
    M = np.asarray(M0, dtype=f).copy()
    mM = np.zeros_like(M); vM = np.zeros_like(M)
    F = np.zeros(d, f); mF = np.zeros(d, f); vF = np.zeros(d, f)
    if not graph_mode:
        y = np.asarray(pred_label, dtype=f)
        lapA = (y[None, :] ** 2 - y[:, None] * y[None, :]) / f(n * n) * f(hp.lap)   # d/dA_ij of y^T(D-A)y/n^2
    else:
        lapA = np.zeros((n, n), f)
    a = gM = gF = None
    for t in range(1, hp.num_epochs + 1):
        S = O._sigmoid(M)
        a = A * (S + S.T) / 2                                                       # explain.py:688-692
        sF = O._sigmoid(F)
        if trace is not None:
            trace.append(dict(a=a, size=float(S.sum()), ent=float((-S * np.log(S) - (1 - S) * np.log(1 - S)).sum()), feat=float(sF.sum())))
        if t == hp.num_epochs and not return_state:
            break
        H = [X]
        Yh, q, bn_state = [], [], []
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
        hs = [emb]
        for w, b in head:                                                           # models.py:193-207: Linear, ReLU, .., Linear
            hs.append(np.maximum(w @ hs[-1] + b, 0))
        logits = Wp @ hs[-1] + bp
        p = np.exp(logits - logits.max()); p = p / p.sum()
        g = p.copy(); g[int(gt_label)] -= 1                                          # d(-log p[gt])/dlogits
        dEmb = Wp.T @ g
        for k in range(len(head) - 1, -1, -1):
            dEmb = head[k][0].T @ (dEmb * (hs[k + 1] > 0))
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
        gF = sF * (1 - sF) * (f(hp.feat_size) / f(d))                                # the forward never sees F
        # size = c*sum(S), ent = mean(H(S)) over ALL n^2 entries; the diagonal gets the regularisers only (A_ii = 0)
        gM = S * (1 - S) * ((A * dA + (A * dA).T) / 2 + f(hp.size) - f(hp.ent) * M / f(n * n))
        if trace is not None:
            trace[-1]["gM"] = gM
        for P, G, m_, v_ in ((M, gM, mM, vM), (F, gF, mF, vF)):
            _opt_update(hp, t, f, P, G, m_, v_)
    out = a.astype(np.float64) if full else a.astype(np.float64) * np.asarray(sub_adj, dtype=np.float64)
    if return_state:
        return out, dict(M=M, F=F, gM=gM, gF=gF)
    return out
