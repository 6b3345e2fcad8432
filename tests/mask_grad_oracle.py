"""mask_grad_oracle.py -- dL/dM and dL/dfeat_mask of the reference's loss (explain.py:665-808) at one point (M, F), by torch autograd.
TEST INFRASTRUCTURE ONLY.

One function for every model and mode the kernels build: the plain GCN (gnnx_oracle._gcn_forward_torch, graph readout through
gnnx_oracle.max_pool), attention (att_oracle.gcn_forward_att_torch), MLP prediction heads (head_oracle.gcn_forward), --bn, any number of
layers, node and graph mode, and unconstrained=True (the dense mask sym(sigmoid(M)) (.) (1 - I) without the adjacency factor, features
unmasked).  Dense (n, n) arrays: meant for n up to about 2000.

Besides the gradients it reports how far the point is from the two places where an fp32 kernel may legitimately take another branch than
the fp64 reference: the smallest |ReLU input| relative to its row's L2 norm (a ReLU kink), and, in graph mode, the max-pool columns whose
best and next-best rows are within 2 fp32 ulps (pool_oracle.near_ties).  A point close to either is resampled, not compared."""
import types

import numpy as np
import torch
import torch.nn.functional as TF
from torch.overrides import TorchFunctionMode

import att_oracle as AO
import gnnx_oracle as O
import head_oracle as HO
import pool_oracle as PO


class _ReluMargin(TorchFunctionMode):
    """Records min |x| / ||x_row|| over every ReLU input of the forward (rows of zero norm carry no gradient and are skipped)."""

    def __init__(self):
        super().__init__()
        self.margin = np.inf

    def __torch_function__(self, func, types_, args=(), kwargs=None):
        if func in (torch.relu, TF.relu):
            x = args[0].detach()
            scale = x.norm(dim=-1, keepdim=True)
            rel = (x.abs() / scale.clamp_min(1e-300))[(scale > 0).expand_as(x)]
            if rel.numel():
                self.margin = min(self.margin, float(rel.min()))
        return func(*args, **(kwargs or {}))


def _plain_weights(weights, dtype):
    t = lambda a: torch.tensor(np.asarray(a), dtype=dtype)
    L = 1
    while ("W%d" % L) in weights:
        L += 1
    return dict(conv_w=[t(weights["W%d" % l]) for l in range(1, L)],
                conv_b=[None if weights.get("b%d" % l) is None else t(weights["b%d" % l]) for l in range(1, L)],
                pred_w=t(weights["Wp"]), pred_b=t(weights["bp"]))


def mask_grads(A, X, gt, pl, idx, weights, M, F, hp, *, graph_mode=False, bn=False, att=False, head=False, unconstrained=False,
               dtype=torch.float64):
    """dL/dM (n, n) and dL/dF (d,) of one epoch's loss at mask parameters M (n, n) and feature-mask parameters F (d,), in `dtype`.
    A (n, n) 0/1 sub-adjacency; X (n, d); gt the explained label; pl (n,) the Laplacian term's labels (node mode); idx the explained
    node's row (node mode); weights as gnnx_oracle (plus Wa1 .. WaL with att, "head" / Wh1 .. with head); hp: gnnx_oracle.default_hparams.
    Returns a namespace: gM, gF (float64 numpy), kink (smallest relative ReLU input), ties (graph mode: near-tied pooled columns)."""
    n = A.shape[0]
    t = lambda a: torch.tensor(np.asarray(a), dtype=dtype)
    if head:
        W, forward = HO.to_torch(weights, dtype), HO.gcn_forward
    elif att:
        W, forward = AO.att_weights_to_torch(weights, dtype, requires_grad=False), AO.gcn_forward_att_torch
    else:
        W, forward = _plain_weights(weights, dtype), O._gcn_forward_torch
    adj = t(np.asarray(A)[None])
    x = t(np.asarray(X)[None])
    mask = t(M).requires_grad_(True)
    fmask = t(F).requires_grad_(True)
    diag = torch.ones(n, n, dtype=dtype) - torch.eye(n, dtype=dtype)
    sym = torch.sigmoid(mask)
    sym = (sym + sym.t()) / 2
    fm = torch.sigmoid(fmask)
    if unconstrained:                                              # explain.py:688-692
        masked, xin = torch.unsqueeze(sym, 0) * diag, x
    else:                                                          # explain.py:665-678, 695-707
        masked, xin = adj * sym * diag, x * fm
    relu = _ReluMargin()
    pool = PO._Pool(None, True, 2) if graph_mode else None        # records the readout's arg-max margins of this (first) forward
    prev = O.set_pool(pool) if graph_mode else None
    try:
        with relu:
            ypred = forward(xin, masked, W, graph_mode, bn)
    finally:
        if graph_mode:
            O.set_pool(prev)
    res = torch.softmax(ypred[0] if graph_mode else ypred[-1, idx, :], dim=0)
    m = torch.sigmoid(mask)
    ent = -m * torch.log(m) - (1 - m) * torch.log(1 - m)
    loss = -torch.log(res[int(gt)]) + hp.size * torch.sum(m) + hp.ent * torch.mean(ent) + hp.feat_size * torch.mean(fm)
    if not graph_mode:
        y = t(pl)
        D = torch.diag(torch.sum(masked[0], 0))
        loss = loss + hp.lap * (y @ (D - masked[0]) @ y) / adj.numel()
    loss.backward()
    return types.SimpleNamespace(gM=mask.grad.numpy().astype(np.float64), gF=fmask.grad.numpy().astype(np.float64), kink=relu.margin,
                                 ties=PO.near_ties(pool.rec) if graph_mode else [])
