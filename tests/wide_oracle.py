"""Inputs wider than 128 features (explain_var.cu's wide path): the reference's optimisation as a torch port with a dtype argument
(the fp64 run bounds how far two faithful fp32 restatements land apart), and the layer-1 contraction order the kernel uses,
restated in numpy fp64:

    P = X (sigmoid(F) (.) W1),   y1 = A_m P + b1,
    dP = A_m^T dY1,   G = X^T dP,   dL/dsigmoid(F)_f = sum_c W1_fc G_fc + c_feat / d,
    layer 1's share of dL/dA_ij = <dY1_i, P_j>."""
import numpy as np
import torch

import gnnx_oracle as O


def explain_torch(sub_adj, sub_feat, gt_label, pred_label, node_idx_new, weights, M0, hp=None, graph_mode=False, bn=False,
                  dtype=torch.float, return_feat=False):
    """gnnx_oracle.explain_dense_torch (explain.py:97-146,665-808) in `dtype`.  Returns the (n, n) float64 mask and, with return_feat,
    sigmoid(feat_mask) as the last epoch's forward used it."""
    hp = hp or O.default_hparams()
    t = lambda a: torch.tensor(np.asarray(a), dtype=dtype)
    L = 1
    while ("W%d" % L) in weights:
        L += 1
    W = dict(conv_w=[t(weights["W%d" % l]) for l in range(1, L)],
             conv_b=[None if weights.get("b%d" % l) is None else t(weights["b%d" % l]) for l in range(1, L)],
             pred_w=t(weights["Wp"]), pred_b=t(weights["bp"]))
    n = sub_adj.shape[0]
    adj = t(np.asarray(sub_adj)[None])
    x = t(np.asarray(sub_feat)[None])
    mask = torch.nn.Parameter(t(M0))
    feat_mask = torch.nn.Parameter(torch.zeros(x.size(-1), dtype=dtype))
    diag_mask = torch.ones(n, n, dtype=dtype) - torch.eye(n, dtype=dtype)
    opts = dict(adam=lambda p: torch.optim.Adam(p, lr=hp.lr, betas=(hp.beta1, hp.beta2), eps=hp.eps),
                sgd=lambda p: torch.optim.SGD(p, lr=hp.lr, momentum=0.95), rmsprop=lambda p: torch.optim.RMSprop(p, lr=hp.lr),
                adagrad=lambda p: torch.optim.Adagrad(p, lr=hp.lr))
    opt = opts[hp.opt]([mask, feat_mask])
    sched = None
    if hp.opt_scheduler == "step":
        sched = torch.optim.lr_scheduler.StepLR(opt, step_size=hp.opt_decay_step, gamma=hp.opt_decay_rate)
    elif hp.opt_scheduler == "cos":
        sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=hp.opt_restart)
    pl = None if graph_mode else t(pred_label)
    masked = fm_used = None
    for _ in range(hp.num_epochs):
        opt.zero_grad()
        S = torch.sigmoid(mask)
        masked = adj * (S + S.t()) / 2 * diag_mask
        fm = torch.sigmoid(feat_mask)
        fm_used = fm.detach()
        ypred = O._gcn_forward_torch(x * fm, masked, W, graph_mode, bn)
        res = torch.softmax(ypred[0] if graph_mode else ypred[-1, node_idx_new, :], dim=0)
        m = torch.sigmoid(mask)
        ent = -m * torch.log(m) - (1 - m) * torch.log(1 - m)
        loss = -torch.log(res[int(gt_label)]) + hp.size * torch.sum(m) + hp.ent * torch.mean(ent) + hp.feat_size * torch.mean(fm)
        if not graph_mode:
            D = torch.diag(torch.sum(masked[0], 0))
            loss = loss + hp.lap * (pl @ (D - masked[-1]) @ pl) / adj.numel()
        loss.backward()
        opt.step()
        if sched is not None:
            sched.step()
    out = masked[0].detach().numpy().astype(np.float64) * np.asarray(sub_adj, np.float64)
    return (out, fm_used.numpy().astype(np.float64)) if return_feat else out


def layer1_wide_grads(a, X, F, W1, dY1, c_feat):
    """The wide path's layer-1 backward in fp64: (dL/dsigmoid(F), layer 1's dL/da as an (n, n) matrix), from the layer-1
    pre-activation gradient dY1 (rows that are not layer-1 rows are zero)."""
    sF = 1 / (1 + np.exp(-F))
    P = X @ (sF[:, None] * W1)
    dP = a.T @ dY1
    G = X.T @ dP
    return (W1 * G).sum(1) + c_feat / X.shape[1], dY1 @ P.T


def layer1_wide_forward(a, X, F, W1, b1):
    sF = 1 / (1 + np.exp(-F))
    return a @ (X @ (sF[:, None] * W1)) + b1
