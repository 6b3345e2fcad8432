"""head_oracle.py -- CPU restatement of Explainer.explain on a model with an MLP prediction head (GcnEncoderNode / GcnEncoderGraph with
pred_hidden_dims, models.py:193-207).  TEST INFRASTRUCTURE ONLY.

pred_model = Sequential(Linear(PD, h1), ReLU, .., Linear(hk, C)) over the concatenated embedding (node mode: the explained node's row;
graph mode: the per-layer max-pool).  One line-by-line port (dense tensors, torch autograd, torch.optim) with a dtype argument, covering
node and graph mode, --bn, any number of layers, attention (--method att) and unconstrained=True; dtype=torch.float64 is the one-update
specification the kernel is checked against.  With an empty head it is gnnx_oracle.explain_dense_torch.
weights: the gnnx_oracle weight dict (W1 .. WL, b1 .., Wp, bp) plus, optionally, Wa1 .. WaL (attention) and "head" = [(W, b), ..] (or
Wh1 / bh1, Wh2 / bh2, .. as in tests/golden/head_golden.npz), the hidden Linears in torch's (out, in) layout; Wp / bp are then the last
Linear.
"""
import numpy as np
import torch
import torch.nn.functional as F

import gnnx_oracle as O
from dense_oracle import _optimizer


def head_layers(weights):
    """The hidden head Linears [(W, b), ..]: weights["head"], or the fixture's Wh1 / bh1, Wh2 / bh2, .."""
    if "head" in weights:
        return list(weights["head"])
    out, j = [], 1
    while ("Wh%d" % j) in weights:
        out.append((weights["Wh%d" % j], weights["bh%d" % j]))
        j += 1
    return out


def to_torch(weights, dtype=torch.float):
    """weights -> tensors (requires_grad, as the reference's frozen model registered under ExplainModule, explain.py:598)."""
    t = lambda a: torch.tensor(np.asarray(a), dtype=dtype, requires_grad=True)
    L = 1
    while ("W%d" % L) in weights:
        L += 1
    L -= 1
    W = dict(conv_w=[t(weights["W%d" % l]) for l in range(1, L + 1)],
             conv_b=[None if weights.get("b%d" % l) is None else t(weights["b%d" % l]) for l in range(1, L + 1)],
             att_w=[t(weights["Wa%d" % l]) for l in range(1, L + 1)] if "Wa1" in weights else None,
             head=[(t(w), t(b)) for w, b in head_layers(weights)],
             pred_w=t(weights["Wp"]), pred_b=t(weights["bp"]))
    return W


def pred_model(emb, W):
    """models.py:193-207: Linear, ReLU, .., Linear."""
    h = emb
    for w, b in W["head"]:
        h = torch.relu(F.linear(h, w, b))
    return F.linear(h, W["pred_w"], W["pred_b"])


def gcn_forward(x, adj, W, graph_mode, bn=False):
    """models.py:58-80 (with the attention of :62-68 when W["att_w"]), :230-267, :269-316, :363-376; the head on the readout."""
    outs = []
    h = x
    L = len(W["conv_w"])
    for l in range(L):
        a = adj
        if W["att_w"] is not None:
            x_att = torch.matmul(h, W["att_w"][l])
            a = adj * (x_att @ x_att.permute(0, 2, 1))
        y = torch.matmul(torch.matmul(a, h), W["conv_w"][l])
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
        return pred_model(torch.cat(O.max_pool(outs), dim=1), W)
    return pred_model(torch.cat(outs, dim=2), W)


def model_pred(adj, feat, weights, bn=False, graph_mode=False):
    """The model's forward on the raw adjacency (self loops included): the `pred` of the checkpoint, float32."""
    W = to_torch(weights)
    with torch.no_grad():
        return gcn_forward(torch.tensor(np.asarray(feat, np.float32)[None]), torch.tensor(np.asarray(adj, np.float32)[None]), W, graph_mode,
                           bn)[0].numpy()


def explain_torch(sub_adj, sub_feat, gt_label, pred_label, node_idx_new, weights, M0, hp=None, graph_mode=False, bn=False,
                  dtype=torch.float, unconstrained=False, return_feat=False, full=False):
    """Port of Explainer.explain's optimisation (explain.py:97-146,209-211; ExplainModule.forward :688-714, loss :740-808) in `dtype`.
    Arguments as gnnx_oracle.explain_dense_torch.  unconstrained: the dense mask sym(sigmoid(M)) (.) (1 - I) drives the forward and the
    features are not masked (explain.py:688-692).  Returns the (n, n) float64 masked adjacency times sub_adj (and, with return_feat,
    sigmoid(feat_mask) as the last epoch's forward used it).  full=True returns the whole masked adjacency, not times sub_adj."""
    hp = hp or O.default_hparams()
    W = to_torch(weights, dtype)
    n = sub_adj.shape[0]
    adj = torch.tensor(np.asarray(sub_adj)[None], dtype=dtype)
    x = torch.tensor(np.asarray(sub_feat)[None], dtype=dtype, requires_grad=True)
    mask = torch.nn.Parameter(torch.tensor(np.asarray(M0), dtype=dtype))
    feat_mask = torch.nn.Parameter(torch.zeros(x.size(-1), dtype=dtype))
    diag_mask = torch.ones(n, n, dtype=dtype) - torch.eye(n, dtype=dtype)
    opt, sched = _optimizer(hp, [mask, feat_mask])
    pl = None if graph_mode else torch.tensor(np.asarray(pred_label), dtype=dtype)
    masked = fm_used = None
    for _ in range(hp.num_epochs):
        opt.zero_grad()
        # the operations in the reference's order (explain.py:688-808): autograd sums a tensor's gradient contributions in the order
        # of their creation, so the order is part of the bits
        sym = torch.sigmoid(mask)
        sym = (sym + sym.t()) / 2
        if unconstrained:
            masked = torch.unsqueeze(sym, 0) * diag_mask
            ypred = gcn_forward(x, masked, W, graph_mode, bn)
        else:
            masked = adj * sym * diag_mask
            ypred = gcn_forward(x * torch.sigmoid(feat_mask), masked, W, graph_mode, bn)
        res = torch.softmax(ypred[0] if graph_mode else ypred[-1, node_idx_new, :], dim=0)
        pred_loss = -torch.log(res[int(gt_label)])
        m = torch.sigmoid(mask)
        size_loss = hp.size * torch.sum(m)
        fm = torch.sigmoid(feat_mask)
        fm_used = fm.detach()
        feat_size_loss = hp.feat_size * torch.mean(fm)
        ent = -m * torch.log(m) - (1 - m) * torch.log(1 - m)
        ent_loss = hp.ent * torch.mean(ent)
        if graph_mode:
            lap_loss = 0
        else:
            D = torch.diag(torch.sum(masked[0], 0))
            lap_loss = hp.lap * (pl @ (D - masked[-1]) @ pl) / adj.numel()
        loss = pred_loss + size_loss + lap_loss + ent_loss + feat_size_loss
        loss.backward()
        opt.step()
        if sched is not None:
            sched.step()
    out = masked[0].detach().numpy().astype(np.float64)
    if not full:
        out = out * np.asarray(sub_adj, np.float64)
    return (out, fm_used.numpy().astype(np.float64)) if return_feat else out
