"""Graph mode's max-pool readout with its arg-max choices made visible: the torch port of the explainer
(gnnx_oracle.explain_dense_torch) runs unchanged, with the readout of gnnx_oracle.max_pool replaced by one that can

  * record, for every epoch whose backward is used (0 .. E-2) and every pooled column, the winning row, the runner-up and their margin
    in fp32 ulps of the winner, and
  * force a column's arg-max to another row: the row's entry gets (o[winner] - o[row]).detach() plus one ulp added before torch.max,
    so the forward moves by about one ulp and the whole gradient of that column takes the other path.

The readout's backward sends dEmb[k] to one row, the first maximal one.  Two rows less than an fp32 ulp apart send a whole epoch's
gradient of that column down different paths, and the trajectory a faithful fp32 implementation follows may differ from the reference's
by far more than rounding.  admissible() lists the trajectories a correct kernel may follow: the reference's, and one per single
near-tie flip."""
import numpy as np
import torch

import gnnx_oracle as O


class _Pool:
    """max_pool's replacement for one run: forward number t is epoch t."""

    def __init__(self, flips, record, epochs):
        self.flips, self.record, self.epochs = flips or {}, record, epochs
        self.epoch = 0
        self.rec = []

    def __call__(self, outs):
        e = self.epoch
        self.epoch += 1
        pooled = []
        layers = []
        for l, o in enumerate(outs):
            v = o.detach()[0]
            for (fl, c, row) in self.flips.get(e, ()):
                if fl != l:
                    continue
                w = int(torch.argmax(v[:, c]))   # first maximal row, like torch.max
                if w == row:
                    continue
                top = torch.nextafter(v[w, c], torch.tensor(float("inf"), dtype=v.dtype))
                off = torch.zeros_like(o)
                off[0, row, c] = top - v[row, c]     # exact: o[row] + off == nextafter(o[winner])
                o = o + off
                v = o.detach()[0]
            if self.record and e < self.epochs - 1:
                vv = v.numpy().astype(np.float64)
                win = np.argmax(vv, 0)
                cols = np.arange(vv.shape[1])
                best = vv[win, cols]
                # the runner-up is the best row whose value differs from the winner's: copies of the winner (twins, the padded rows
                # that all hold the edge-less constant) would otherwise hide a row under an ulp below them
                rest = np.where(vv == best[None, :], -np.inf, vv)
                run = np.argmax(rest, 0)
                ulp = np.spacing(np.abs(best).astype(np.float32)).astype(np.float64)
                with np.errstate(invalid="ignore"):
                    margin = np.where(np.isfinite(rest[run, cols]), (best - rest[run, cols]) / ulp, np.inf)
                layers.append((win, run, margin))
            pooled.append(torch.max(o, dim=1)[0])
        if layers:
            self.rec.append(layers)
        return pooled


def explain_torch_pool(sub_adj, sub_feat, gt_label, weights, M0, hp=None, bn=False, dtype=torch.float, flips=None, record=False,
                       unconstrained=False):
    """The graph-mode explainer port of the model (attention / MLP head / plain GCN, any L, --bn, unconstrained) in `dtype`, with
    flips = {epoch: [(layer, col, row)]} forcing the arg-max of those pooled columns to `row`.  Returns (mask, sigmoid(feat_mask)) as the
    port does and, with record=True, the record: record[epoch][layer] = (winner rows, runner-up rows, margins in fp32 ulps) per column,
    for epochs 0 .. E-2.  With flips=None the result is bit for bit the port's."""
    hp = hp or O.default_hparams()
    pool = _Pool(flips, record, hp.num_epochs)
    prev = O.set_pool(pool)
    try:
        out, fm = O.explain_dense_torch(sub_adj, sub_feat, gt_label, None, 0, weights, M0, hp, graph_mode=True, bn=bn, return_feat=True,
                                        dtype=dtype, unconstrained=unconstrained)
    finally:
        O.set_pool(prev)
    return (out, fm, pool.rec) if record else (out, fm)


def near_ties(record, ulps=2):
    """[(epoch, layer, col, winner, runner_up, margin)] of every pooled column whose best value and the next different one are less
    than `ulps` fp32 ulps apart.  Rows equal to the winner are not a near tie: torch.max's first maximal row is the defined choice among
    them (twin rows, the padded rows of the edge-less constant, a ReLU column that is 0 in every row)."""
    out = []
    for e, layers in enumerate(record):
        for l, (win, run, margin) in enumerate(layers):
            for c in np.nonzero(margin < ulps)[0]:
                out.append((e, l, int(c), int(win[c]), int(run[c]), float(margin[c])))
    return out


def admissible(sub_adj, sub_feat, gt_label, weights, M0, hp=None, bn=False, ulps=2, unconstrained=False):
    """[(flip, mask, feat_mask)]: the fp32 trajectory (flip None) and, for every near tie of the fp64 run (near_ties(.., ulps)), the fp32
    trajectory whose arg-max at that (epoch, layer, column) is the other row of the pair than the one the fp32 run chose."""
    kw = dict(hp=hp, bn=bn, unconstrained=unconstrained)
    m32, f32, r32 = explain_torch_pool(sub_adj, sub_feat, gt_label, weights, M0, record=True, **kw)
    _, _, r64 = explain_torch_pool(sub_adj, sub_feat, gt_label, weights, M0, dtype=torch.float64, record=True, **kw)
    out = [(None, m32, f32)]
    for e, l, c, w, r, _ in near_ties(r64, ulps):
        row = r if int(r32[e][l][0][c]) == w else w
        m, f = explain_torch_pool(sub_adj, sub_feat, gt_label, weights, M0, flips={e: [(l, c, row)]}, **kw)
        out.append(((e, l, c, row), m, f))
    return out


def nearest_admissible(got, ref, sub_adj, sub_feat, gt_label, weights, M0, hp=None, bn=False, unconstrained=False):
    """rel_l2 of a kernel's edge mask `got` (the entries of np.nonzero(sub_adj)) from the nearest admissible trajectory: the reference's
    own mask `ref`, or an fp32 port trajectory with one near-tie flip."""
    ei, ej = np.nonzero(sub_adj)
    errs = [O.rel_l2(got, ref)]
    errs += [O.rel_l2(got, m[ei, ej]) for f, m, _ in admissible(sub_adj, sub_feat, gt_label, weights, M0, hp, bn, unconstrained=unconstrained)
             if f is not None]
    return min(errs)
