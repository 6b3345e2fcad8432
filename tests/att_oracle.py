"""att_oracle.py -- the hand-derived backward of Explainer.explain on an attention model (train.py / explainer_main.py --method att).
TEST INFRASTRUCTURE ONLY.

An attention GraphConv (models.py:62-68) scales the adjacency it is given by the unnormalised scores s = P P^T, P = H_{l-1} Wa_l,
before the usual aggregation; every layer gets the explainer's masked adjacency (models.py:240,250,256,278-297).  The torch port
(gnnx_oracle.explain_dense_torch) runs these models when the weights carry Wa1 .. WaL; here:
  * mask_grads_closed_form -- the hand-derived backward of one epoch (numpy, fp64): dL/dM and dL/dfeat_mask from the equations in
                            DESIGN.md ("Attention models"), checked against autograd (tests/mask_grad_oracle.py).
weights: the gnnx_oracle weight dict plus Wa1 .. WaL, the (in, in) att_weight matrices.
"""
import numpy as np

import gnnx_oracle as O


def _sig(z):
    return 1.0 / (1.0 + np.exp(-z))


def mask_grads_closed_form(sub_adj, sub_feat, gt_label, pred_label, node_idx_new, weights, M, F, hp=None, graph_mode=False, bn=False):
    """The same gradients from the hand-derived backward (fp64 numpy), per layer l with D_l = dL/dZ_l, Z_l = (A_m (.) s_l) H_{l-1}:
         dL/dH_{l-1} = (A_m (.) s_l)^T D_l + dL/dP_l Wa_l^T,   t_l = D_l H_{l-1}^T,
         dL/dP_l = (A_m (.) t_l + (A_m (.) t_l)^T) P_l,      dL/dA_m += s_l (.) t_l,
       then dL/dA_m -> dL/dM through the symmetrised sigmoid and the diagonal mask, plus the regularisers."""
    hp = hp or O.default_hparams()
    A = np.asarray(sub_adj, np.float64)
    X = np.asarray(sub_feat, np.float64)
    n = A.shape[0]
    L = sum(1 for k in weights if k.startswith("W") and k[1:].isdigit())
    Wc = [np.asarray(weights["W%d" % (l + 1)], np.float64) for l in range(L)]
    bc = [None if weights.get("b%d" % (l + 1)) is None else np.asarray(weights["b%d" % (l + 1)], np.float64) for l in range(L)]
    Wa = [np.asarray(weights["Wa%d" % (l + 1)], np.float64) for l in range(L)]
    Wp, bp = np.asarray(weights["Wp"], np.float64), np.asarray(weights["bp"], np.float64)
    M = np.asarray(M, np.float64)
    Sg = _sig(M)
    Am = A * (Sg + Sg.T) / 2 * (1 - np.eye(n))
    sF = _sig(np.asarray(F, np.float64))
    H = [X * sF]
    cache = []
    for l in range(L):
        P = H[-1] @ Wa[l]
        s = P @ P.T
        Z = (Am * s) @ H[-1]
        Y = Z @ Wc[l] + (bc[l] if bc[l] is not None else 0)
        q = np.maximum(np.linalg.norm(Y, axis=1, keepdims=True), 1e-12)
        Yh = Y / q
        h, istd = Yh, None
        if l < L - 1:
            h = np.maximum(Yh, 0)
            if bn:
                mu = h.mean(axis=1, keepdims=True)
                var = ((h - mu) ** 2).mean(axis=1, keepdims=True)
                istd = 1 / np.sqrt(var + 1e-5)
                h = (h - mu) * istd
        cache.append((P, s, Yh, q, istd, h))
        H.append(h)
    if graph_mode:
        arg = [np.argmax(h, axis=0) for h in H[1:]]
        emb = np.concatenate([h[a, np.arange(h.shape[1])] for h, a in zip(H[1:], arg)])
    else:
        emb = np.concatenate([h[node_idx_new] for h in H[1:]])
    logits = Wp @ emb + bp
    p = np.exp(logits - logits.max())
    p /= p.sum()
    dlog = p.copy()
    dlog[int(gt_label)] -= 1
    dEmb = Wp.T @ dlog
    dH = [np.zeros_like(h) for h in H]
    off = 0
    for l in range(L):
        w = H[l + 1].shape[1]
        if graph_mode:
            dH[l + 1][arg[l], np.arange(w)] += dEmb[off:off + w]
        else:
            dH[l + 1][node_idx_new] += dEmb[off:off + w]
        off += w
    dAm = np.zeros((n, n))
    for l in range(L - 1, -1, -1):
        P, s, Yh, q, istd, h = cache[l]
        g = dH[l + 1]
        if l < L - 1:
            if bn:
                g = (g - g.mean(axis=1, keepdims=True) - h * (g * h).mean(axis=1, keepdims=True)) * istd
            g = g * (Yh > 0)
        dY = (g - Yh * (g * Yh).sum(axis=1, keepdims=True)) / q
        Dl = dY @ Wc[l].T
        Hp = H[l]
        t = Dl @ Hp.T
        dAm += s * t
        dP = (Am * t + (Am * t).T) @ P
        dH[l] = dH[l] + (Am * s).T @ Dl + dP @ Wa[l].T
    dF_pred = (dH[0] * X).sum(axis=0) * sF * (1 - sF)
    dF = dF_pred + hp.feat_size / X.shape[1] * sF * (1 - sF)
    if not graph_mode:
        y = np.asarray(pred_label, np.float64)
        dAm += hp.lap / A.size * (y[None, :] - y[:, None]) ** 2 / 2   # y^T (D - A_m) y = sum_ij A_m,ij (y_i - y_j)^2 / 2
    dS = (dAm + dAm.T) / 2 * A * (1 - np.eye(n))
    dM = Sg * (1 - Sg) * (dS + hp.size - hp.ent / A.size * M)
    return dM, dF
