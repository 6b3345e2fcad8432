"""Inputs wider than 128 features (explain_var.cu's wide path): the layer-1 contraction order the kernel uses, restated in numpy fp64
(the optimisation itself is gnnx_oracle.explain_dense_torch):

    P = X (sigmoid(F) (.) W1),   y1 = A_m P + b1,
    dP = A_m^T dY1,   G = X^T dP,   dL/dsigmoid(F)_f = sum_c W1_fc G_fc + c_feat / d,
    layer 1's share of dL/dA_ij = <dY1_i, P_j>."""
import numpy as np


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
