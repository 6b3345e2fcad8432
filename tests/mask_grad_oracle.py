"""mask_grad_oracle.py -- dL/dM and dL/dfeat_mask of the reference's loss (explain.py:665-808) at one point (M, F), by torch autograd.
TEST INFRASTRUCTURE ONLY.

One function for every model and mode the kernels build, through the loss of the explainer port (gnnx_oracle._epoch_loss): the plain
GCN, attention and MLP prediction heads (as the weights carry them), --bn, any number of layers, node and graph mode (graph readout
through gnnx_oracle.max_pool), and unconstrained=True (the dense mask sym(sigmoid(M)) (.) (1 - I) without the adjacency factor, features
unmasked).  Dense (n, n) arrays: meant for n up to about 2000.

Besides the gradients it reports how far the point is from the two places where an fp32 kernel may legitimately take another branch than
the fp64 reference: the smallest |ReLU input| relative to its row's L2 norm (a ReLU kink), and, in graph mode, the max-pool columns whose
best and next-best rows are within 2 fp32 ulps (pool_oracle.near_ties).  A point close to either is resampled, not compared."""
import types

import numpy as np
import torch
import torch.nn.functional as TF
from torch.overrides import TorchFunctionMode

import gnnx_oracle as O
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


def mask_grads(A, X, gt, pl, idx, weights, M, F, hp, *, graph_mode=False, bn=False, unconstrained=False, dtype=torch.float64):
    """dL/dM (n, n) and dL/dF (d,) of one epoch's loss (gnnx_oracle._epoch_loss) at mask parameters M (n, n) and feature-mask parameters
    F (d,), in `dtype`.  A (n, n) 0/1 sub-adjacency; X (n, d); gt the explained label; pl (n,) the Laplacian term's labels (node mode);
    idx the explained node's row (node mode); weights as gnnx_oracle.weights_to_torch reads them; hp: gnnx_oracle.default_hparams.
    Returns a namespace: gM, gF (float64 numpy), kink (smallest relative ReLU input), ties (graph mode: near-tied pooled columns)."""
    n = A.shape[0]
    t = lambda a: torch.tensor(np.asarray(a), dtype=dtype)
    W = O.weights_to_torch(weights, requires_grad=False, dtype=dtype)
    mask = t(M).requires_grad_(True)
    fmask = t(F).requires_grad_(True)
    diag = torch.ones(n, n, dtype=dtype) - torch.eye(n, dtype=dtype)
    relu = _ReluMargin()
    pool = PO._Pool(None, True, 2) if graph_mode else None        # records the readout's arg-max margins of this (first) forward
    prev = O.set_pool(pool) if graph_mode else None
    try:
        with relu:
            loss, _, _, _ = O._epoch_loss(mask, fmask, t(np.asarray(A)[None]), t(np.asarray(X)[None]), diag, W, gt,
                                          None if graph_mode else t(pl), idx, hp, graph_mode, bn, unconstrained)
    finally:
        if graph_mode:
            O.set_pool(prev)
    loss.backward()
    return types.SimpleNamespace(gM=mask.grad.numpy().astype(np.float64), gF=fmask.grad.numpy().astype(np.float64), kink=relu.margin,
                                 ties=PO.near_ties(pool.rec) if graph_mode else [])
