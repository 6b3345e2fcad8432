"""CPU specification of the gradient baseline in graph-classification mode: Explainer.explain(0, graph_idx=g, graph_mode=True,
model="grad") (explain.py:102,125-133) with ExplainModule.adj_feat_grad's graph branch (explain.py:717-738) -- one forward of the frozen
GcnEncoderGraph on the unmasked padded graph, loss = -log softmax(logits)[label], one backward to the dense adjacency, result
sigmoid(|dL/dA| + |dL/dA|^T) * adj (batch entry 0).

  grad_graph_torch        line-by-line port through gnnx_oracle's graph-mode forward: float32 reproduces the reference's arithmetic,
                          float64 is the autograd specification
  grad_graph_closed_form  the same derivative by hand, numpy float64: the max-pool routes each readout column's gradient to its first
                          maximal row (np.argmax, as torch.max)

label = -1 means the model's own prediction: the arg-max of the logits of the same forward (first maximum)."""
import numpy as np
import torch

import gnnx_oracle as O


def grad_graph_torch(adj, feat, label, weights, dtype=np.float32, return_label=False):
    """adj (n, n) 0/1 padded graph, feat (n, d) -> (n, n) float64 mask (zero off the edges)."""
    tdt = torch.float64 if dtype == np.float64 else torch.float
    A = torch.tensor(np.asarray(adj, dtype)[None], dtype=tdt, requires_grad=True)          # explain.py:97 (requires_grad: :720)
    x = torch.tensor(np.asarray(feat, dtype)[None], dtype=tdt, requires_grad=True)         # :98
    ypred = O._gcn_forward_torch(x, A, O.weights_to_torch(weights, dtype=tdt), True)       # :729
    label = int(label)
    if label < 0:
        label = int(np.argmax(ypred[0].detach().numpy()))
    p = torch.softmax(ypred[0], dim=0)[label]                                              # :731,734
    (-torch.log(p)).backward()                                                             # :735-736
    g = torch.abs(A.grad)[0]                                                               # :127-130, batch entry 0
    m = torch.sigmoid(g + g.t()).detach().numpy() * np.asarray(adj, np.float64)            # :131-133
    return (m, label) if return_label else m


def grad_graph_closed_form(adj, feat, label, weights, return_grad=False):
    """Hand-derived float64 form of grad_graph_torch (3 or any number of layers, no --bn): dL/dA = sum_l dZ_l H_{l-1}^T, dZ_l the
    gradient at A H_{l-1}; the readout max-pools every layer's columns over all rows, padding rows included."""
    f = np.float64
    A, X = np.asarray(adj, f), np.asarray(feat, f)
    Ws, bs = [], []
    l = 1
    while ("W%d" % l) in weights:
        Ws.append(np.asarray(weights["W%d" % l], f))
        b = weights.get("b%d" % l)
        bs.append(np.zeros(Ws[-1].shape[1], f) if b is None else np.asarray(b, f))
        l += 1
    L = len(Ws)
    offs = np.concatenate([[0], np.cumsum([w.shape[1] for w in Ws])])
    Wp, bp = np.asarray(weights["Wp"], f), np.asarray(weights["bp"], f)
    H, Yh, q = [X], [], []
    for l in range(L):
        Y = (A @ H[-1]) @ Ws[l] + bs[l]
        ql = np.maximum(np.sqrt((Y * Y).sum(1, keepdims=True)), 1e-12)
        Yh.append(Y / ql); q.append(ql)
        H.append(np.maximum(Yh[-1], 0) if l < L - 1 else Yh[-1])
    arg = [H[l + 1].argmax(0) for l in range(L)]
    emb = np.concatenate([H[l + 1].max(0) for l in range(L)])
    logits = Wp @ emb + bp
    label = int(np.argmax(logits)) if int(label) < 0 else int(label)
    p = np.exp(logits - logits.max()); p /= p.sum()
    gl = p.copy(); gl[label] -= 1.0
    dEmb = Wp.T @ gl
    n = A.shape[0]
    dA = np.zeros((n, n), f)
    dH = np.zeros_like(H[L])
    for l in range(L - 1, -1, -1):
        dYh = dH.copy()
        cols = np.arange(offs[l + 1] - offs[l])
        np.add.at(dYh, (arg[l], cols), dEmb[offs[l]:offs[l + 1]])
        if l < L - 1:
            dYh = dYh * (Yh[l] > 0)
        dY = (dYh - Yh[l] * (Yh[l] * dYh).sum(1, keepdims=True)) / q[l]
        dZ = dY @ Ws[l].T
        dA += dZ @ H[l].T
        dH = A.T @ dZ
    G = np.abs(dA)
    out = 1.0 / (1.0 + np.exp(-(G + G.T))) * A
    return (out, dA) if return_grad else out
