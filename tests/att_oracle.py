"""att_oracle.py -- CPU restatements of Explainer.explain on an attention model (train.py / explainer_main.py --method att).
TEST INFRASTRUCTURE ONLY.

An attention GraphConv (models.py:62-68) scales the adjacency it is given by the unnormalised scores s = P P^T, P = H_{l-1} Wa_l,
before the usual aggregation; every layer gets the explainer's masked adjacency (models.py:240,250,256,278-297).  Two restatements,
built on the helpers of oracle/gnnx_oracle.py:
  * explain_att_torch    -- line-by-line port (dense tensors, torch autograd, torch.optim); dtype=torch.float64 gives the fp64
                            specification the kernel's single update is checked against.
  * mask_grads_closed_form -- the hand-derived backward of one epoch (numpy, fp64): dL/dM and dL/dfeat_mask from the equations in
                            DESIGN.md ("Attention models"), checked against autograd.
weights: the gnnx_oracle weight dict plus Wa1 .. WaL, the (in, in) att_weight matrices.
"""
import numpy as np

import gnnx_oracle as O
from dense_oracle import _optimizer


def att_weights_to_torch(weights, dtype=None, requires_grad=True):
    import torch
    dtype = dtype or torch.float
    t = lambda a: torch.tensor(np.asarray(a), dtype=dtype, requires_grad=requires_grad)
    W = O.weights_to_torch(weights, requires_grad)
    W = {k: ([t(x.detach().numpy()) if x is not None else None for x in v] if isinstance(v, list) else t(v.detach().numpy()))
         for k, v in W.items()}
    W["att_w"] = [t(weights["Wa%d" % (l + 1)]) for l in range(len(W["conv_w"]))]
    return W


def gcn_forward_att_torch(x, adj, W, graph_mode, bn=False):
    """gnnx_oracle._gcn_forward_torch with the attention of models.py:62-68 in every layer."""
    import torch
    import torch.nn.functional as F
    outs = []
    h = x
    L = len(W["conv_w"])
    for l in range(L):
        x_att = torch.matmul(h, W["att_w"][l])                 # models.py:63
        att = x_att @ x_att.permute(0, 2, 1)                   # models.py:66
        a = adj * att                                          # models.py:68
        y = torch.matmul(a, h)
        y = torch.matmul(y, W["conv_w"][l])
        if W["conv_b"][l] is not None:
            y = y + W["conv_b"][l]
        y = F.normalize(y, p=2, dim=2)
        if l < L - 1:
            y = torch.relu(y)
            if bn:
                y = F.batch_norm(y, None, None, None, None, True, 0.1, 1e-5)
        outs.append(y)
        h = y
    if graph_mode:
        emb = torch.cat(O.max_pool(outs), dim=1)
        return F.linear(emb, W["pred_w"], W["pred_b"])
    return F.linear(torch.cat(outs, dim=2), W["pred_w"], W["pred_b"])


def model_pred_att(adj, feat, weights, bn=False, graph_mode=False):
    """GcnEncoderNode / GcnEncoderGraph.forward on the raw adjacency (self loops included): the `pred` of the checkpoint."""
    import torch
    W = att_weights_to_torch(weights, requires_grad=False)
    with torch.no_grad():
        return gcn_forward_att_torch(torch.tensor(np.asarray(feat, np.float32)[None]), torch.tensor(np.asarray(adj, np.float32)[None]),
                                     W, graph_mode, bn)[0].numpy()


def _loss(W, adj, x, mask, feat_mask, diag_mask, gt_label, pred_label_t, node_idx_new, hp, graph_mode, bn):
    """explain.py:665-808 with the attention forward: (loss, masked_adj, sigmoid(feat_mask))."""
    import torch
    sym = torch.sigmoid(mask)
    sym = (sym + sym.t()) / 2
    masked_adj = adj * sym * diag_mask
    fm = torch.sigmoid(feat_mask)
    ypred = gcn_forward_att_torch(x * fm, masked_adj, W, graph_mode, bn)
    res = torch.softmax(ypred[0] if graph_mode else ypred[-1, node_idx_new, :], dim=0)
    pred_loss = -torch.log(res[int(gt_label)])
    m = torch.sigmoid(mask)
    size_loss = hp.size * torch.sum(m)
    feat_size_loss = hp.feat_size * torch.mean(fm)
    mask_ent = -m * torch.log(m) - (1 - m) * torch.log(1 - m)
    mask_ent_loss = hp.ent * torch.mean(mask_ent)
    if graph_mode:
        lap_loss = 0
    else:
        D = torch.diag(torch.sum(masked_adj[0], 0))
        lap_loss = hp.lap * (pred_label_t @ (D - masked_adj[-1]) @ pred_label_t) / adj.numel()
    return pred_loss + size_loss + lap_loss + mask_ent_loss + feat_size_loss, masked_adj, fm


def explain_att_torch(sub_adj, sub_feat, gt_label, pred_label, node_idx_new, weights, M0, hp=None, graph_mode=False, bn=False,
                      dtype=None, return_feat=False):
    """Port of Explainer.explain's optimisation (explain.py:97-146,209-211) on an attention model.  Arguments as
    gnnx_oracle.explain_dense_torch.  Returns the (n,n) float64 masked adjacency (and sigmoid(feat_mask) as the last forward used it)."""
    import torch
    hp = hp or O.default_hparams()
    dtype = dtype or torch.float
    W = att_weights_to_torch(weights, dtype)
    n = sub_adj.shape[0]
    adj = torch.tensor(np.asarray(sub_adj)[None], dtype=dtype)
    x = torch.tensor(np.asarray(sub_feat)[None], dtype=dtype, requires_grad=True)
    mask = torch.nn.Parameter(torch.tensor(np.asarray(M0), dtype=dtype))
    feat_mask = torch.nn.Parameter(torch.zeros(x.size(-1), dtype=dtype))
    diag_mask = torch.ones(n, n, dtype=dtype) - torch.eye(n, dtype=dtype)
    opt, sched = _optimizer(hp, [mask, feat_mask])
    pred_label_t = None if graph_mode else torch.tensor(np.asarray(pred_label), dtype=dtype)
    masked_adj = fm = None
    for _ in range(hp.num_epochs):
        opt.zero_grad()
        loss, masked_adj, fm = _loss(W, adj, x, mask, feat_mask, diag_mask, gt_label, pred_label_t, node_idx_new, hp, graph_mode, bn)
        fm = fm.detach()
        loss.backward()
        opt.step()
        if sched is not None:
            sched.step()
    out = masked_adj[0].detach().numpy().astype(np.float64) * np.asarray(sub_adj, dtype=np.float64)
    return (out, fm.numpy().astype(np.float64)) if return_feat else out


def mask_grads_autograd(sub_adj, sub_feat, gt_label, pred_label, node_idx_new, weights, M, F, hp=None, graph_mode=False, bn=False):
    """dL/dM and dL/dfeat_mask of one epoch by torch autograd in fp64 (the reference for mask_grads_closed_form)."""
    import torch
    hp = hp or O.default_hparams()
    dt = torch.float64
    W = att_weights_to_torch(weights, dt, requires_grad=False)
    n = sub_adj.shape[0]
    adj = torch.tensor(np.asarray(sub_adj)[None], dtype=dt)
    x = torch.tensor(np.asarray(sub_feat)[None], dtype=dt)
    mask = torch.tensor(np.asarray(M), dtype=dt, requires_grad=True)
    feat_mask = torch.tensor(np.asarray(F), dtype=dt, requires_grad=True)
    diag_mask = torch.ones(n, n, dtype=dt) - torch.eye(n, dtype=dt)
    pl = None if graph_mode else torch.tensor(np.asarray(pred_label), dtype=dt)
    loss, _, _ = _loss(W, adj, x, mask, feat_mask, diag_mask, gt_label, pl, node_idx_new, hp, graph_mode, bn)
    loss.backward()
    return mask.grad.numpy(), feat_mask.grad.numpy()


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
