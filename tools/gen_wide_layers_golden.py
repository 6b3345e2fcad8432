"""gen_wide_layers_golden.py -- tests/golden/wide_layers_golden.npz by EXECUTING THE UNMODIFIED REFERENCE on GCNs whose hidden / output
widths are 129 .. 256 (--hidden-dim / --output-dim, models.py:83-190, explainer_main.py:51-56).

The reference's GcnEncoderNode / GcnEncoderGraph (models.py, reference init), biases redrawn from N(0, 0.3) so that they matter, every
parameter then rounded to the nearest float16 value (the model stays float32; the rounding only lets the fixture store the weights in
half the bytes), explained with Explainer.explain (model="exp"):
  * node mode on the rand fixture graph (its own features), nodes 0, 7, 33, 100: 3 layers at 256 / 256 with 30 and 100 epochs and with
    SGD, --bn at 160 / 136, 2 layers at 256 / 20, 5 layers at 144 / 144;
  * graph mode on the 12 graphs of graphs_golden.npz: 3 layers at 256 / 256, --bn with 4 layers at 160 / 160.
Needs the reference tree (oracle/ref_harness.py); deterministic:
    python tools/gen_wide_layers_golden.py

Keys as tools/gen_deep_golden.py writes them, plus
  <case>_wfrom    the case whose <case>_w_* arrays hold this case's weights (float16; cases that share a model store it once)
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
import gen_deep_golden as GD  # noqa: E402
import ref_harness  # noqa: E402
from gen_golden import OUT  # noqa: E402

# name: (L, bn, att, hid, emb, opt, epochs, model seed)
NODE_CASES = {"rand_h256_e30": (3, False, False, 256, 256, "adam", 30, 1300), "rand_h256_e100": (3, False, False, 256, 256, "adam", 100, 1300),
              "rand_h256_sgd": (3, False, False, 256, 256, "sgd", 30, 1300), "rand_bn_h160_o136": (3, True, False, 160, 136, "adam", 30, 1301),
              "rand_L2_h256_o20": (2, False, False, 256, 20, "adam", 30, 1302), "rand_L5_h144": (5, False, False, 144, 144, "adam", 30, 1303)}
GRAPH_CASES = {"graphs_h256": (3, False, False, 256, 256, "adam", 30, 1400), "graphs_bn_L4_h160": (4, True, False, 160, 160, "adam", 30, 1401)}

_deep_model = GD._model


def _half_model(cls, d, C, L, bn, att, hid, emb, seed):
    """gen_deep_golden's model with every parameter rounded to float16 (in place, before the reference sees it)."""
    model, _ = _deep_model(cls, d, C, L, bn, att, hid, emb, seed)
    with torch.no_grad():
        for p_ in model.parameters():
            p_.copy_(p_.half().float())
    # re-read the rounded weights under the fixture's names
    sd = model.state_dict()
    keys = ["conv_first"] + ["conv_block.%d" % i for i in range(L - 2)] + ["conv_last"]
    W = {}
    for l, k in enumerate(keys, 1):
        W["W%d" % l] = sd[k + ".weight"].numpy().astype(np.float32)
        W["b%d" % l] = sd[k + ".bias"].numpy().astype(np.float32)
    W["Wp"] = sd["pred_model.weight"].numpy().astype(np.float32)
    W["bp"] = sd["pred_model.bias"].numpy().astype(np.float32)
    return model, W


def gen(R):
    GD._model = _half_model
    out = {"cases": np.asarray(list(NODE_CASES) + list(GRAPH_CASES))}
    for name, (L, bn, att, hid, emb, opt, epochs, seed) in NODE_CASES.items():
        GD.gen_node_case(R, out, name, L, bn, att, hid, emb, opt, epochs, seed=seed)
    for name, (L, bn, att, hid, emb, opt, epochs, seed) in GRAPH_CASES.items():
        GD.gen_graph_case(R, out, name, L, bn, att, hid, emb, opt, epochs, seed=seed)
    # one copy of each model, as float16 (exact: the parameters were rounded before use)
    kept = {}
    for name, c in list(NODE_CASES.items()) + list(GRAPH_CASES.items()):
        key = (name in GRAPH_CASES, c[7])
        p = name + "_w_"
        names = [k for k in out if k.startswith(p)]
        if key in kept:
            for k in names:
                assert np.array_equal(out[k], out[kept[key] + "_w_" + k[len(p):]]), k
                del out[k]
        else:
            kept[key] = name
            for k in names:
                h = out[k].astype(np.float16)
                assert np.array_equal(h.astype(np.float32), out[k]), k
                out[k] = h
        out[name + "_wfrom"] = np.str_(kept[key])
    path = os.path.join(OUT, "wide_layers_golden.npz")
    np.savez_compressed(path, **out)
    print("  wide-layers golden written (%d bytes)" % os.path.getsize(path))


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen(ref_harness.load())
