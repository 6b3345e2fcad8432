"""CPU: the oracle pieces the graph-mode GPU tests rest on.

  * the host restatement of the kernels' device init (Philox4x32-10 + Box-Muller, gnnx_oracle.philox_m0) against the Random123
    known-answer vectors and the moments of N(0, 1);
  * the feature mask the line-by-line port returns (return_feat=True) against the fp64 closed form's F in graph mode: the kernels
    return sigmoid(F) after num_epochs - 1 updates, explain_closed_form(num_epochs - 1, return_state=True) stops at the same point;
  * the closed form's returned state (M, F and the Adam moments) resumes a run: one step from it equals the uninterrupted run."""
import numpy as np
import pytest

import gnnx_oracle as O
import util
from test_oracle_graph_variants import MODEL_TAGS, dense_m0, model_of


@pytest.fixture(scope="module")
def gv():
    return np.load(util.GOLDEN + "/graph_variants_golden.npz")


@pytest.fixture(scope="module")
def gg():
    return np.load(util.GOLDEN + "/graphs_golden.npz")


def _hex(words):
    return " ".join("%08x" % int(w) for w in words)


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), "d16cfe09 94fdcceb 5001e420 24126ea1"),
])
def test_philox_known_answers(ctr, key, want):
    assert _hex(O.philox4x32_10(ctr, key)) == want


def test_philox_normal_is_standard_normal():
    N = 10 ** 6
    z = O.philox_normal(7, 1279, np.arange(N))
    # 5 standard errors: mean ~ N(0, 1/N), sample variance ~ N(1, 2/N)
    assert abs(z.mean()) < 5 / np.sqrt(N) and abs(z.var() - 1) < 5 * np.sqrt(2 / N), (z.mean(), z.var())
    assert np.abs(z).max() < 6.0
    # keyed by (seed, key, slot): another key or seed gives another stream, the same triple the same number
    assert np.array_equal(z[:100], O.philox_normal(7, 1279, np.arange(100)))
    assert not np.allclose(z[:100], O.philox_normal(7, 1280, np.arange(100)))
    assert not np.allclose(z[:100], O.philox_normal(8, 1279, np.arange(100)))
    assert not np.allclose(z[:100], O.philox_normal(7 + (1 << 32), 1279, np.arange(100)))


def test_philox_m0_scales_by_the_task_size():
    z = O.philox_normal(3, 11, np.arange(50))
    assert np.allclose(O.philox_m0(3, 11, 50, 100), 1 + np.sqrt(2 / 100) * z, rtol=0, atol=1e-15)
    m = O.philox_m0(3, 11, 200000, 40)
    assert abs(m.mean() - 1) < 5 * np.sqrt(0.05 / 200000) and abs(m.std() / np.sqrt(2 / 40) - 1) < 0.01


def _graph_case(gg, gv, tag):
    if tag == "default":
        return {k: gg[k] for k in util.WKEYS}, 3, False
    return model_of(gv, tag)


@pytest.mark.parametrize("tag", ["default"] + [t for t in MODEL_TAGS if t in ("L2", "L4", "bn")])
def test_port_feature_mask_is_the_closed_form_state(gg, gv, tag):
    w, L, bn = _graph_case(gg, gv, tag)
    E = 10
    for g in range(int(gg["num_graphs"])):
        A = gg["adj"][g].astype(np.float64)
        args = (A, gg["feat"][g], int(gg["label"][g]), None, 0, w, dense_m0(gg, g))
        plain = O.explain_dense_torch(*args, hp=O.default_hparams(num_epochs=E), graph_mode=True, bn=bn)
        mask, fm = O.explain_dense_torch(*args, hp=O.default_hparams(num_epochs=E), graph_mode=True, bn=bn, return_feat=True)
        assert np.array_equal(mask, plain)                 # the option changes nothing else
        _, st = O.explain_closed_form(*args, hp=O.default_hparams(num_epochs=E - 1), graph_mode=True, bn=bn, return_state=True)
        ref = 1 / (1 + np.exp(-st["F"]))
        assert fm.shape == (gg["feat"].shape[2],) and np.abs(ref - 0.5).max() > 1e-3   # F has moved from 0
        assert np.abs(fm - ref).max() <= 1e-6, (tag, g, np.abs(fm - ref).max())


def test_port_feature_mask_before_any_update(gg):
    w = {k: gg[k] for k in util.WKEYS}
    A = gg["adj"][2].astype(np.float64)
    _, fm = O.explain_dense_torch(A, gg["feat"][2], int(gg["label"][2]), None, 0, w, dense_m0(gg, 2),
                                  hp=O.default_hparams(num_epochs=1), graph_mode=True, return_feat=True)
    assert np.array_equal(fm, np.full(gg["feat"].shape[2], 0.5))


@pytest.mark.parametrize("bn", [False, True])
def test_closed_form_resumes_from_its_state_graph_mode(gg, gv, bn):
    w, L, _ = _graph_case(gg, gv, "bn" if bn else "default")
    t0 = 7
    for g in (0, 3, 9):
        A = gg["adj"][g].astype(np.float64)
        args = (A, gg["feat"][g], int(gg["label"][g]), None, 0, w, dense_m0(gg, g))
        _, s0 = O.explain_closed_form(*args, hp=O.default_hparams(num_epochs=t0), graph_mode=True, bn=bn, return_state=True)
        _, s1 = O.explain_closed_form(*args, hp=O.default_hparams(num_epochs=t0 + 1), graph_mode=True, bn=bn, return_state=True)
        init = dict(m=s0["mM"], v=s0["vM"], feat=np.stack([s0["F"], s0["mF"], s0["vF"]]), step=t0)
        _, r1 = O.explain_closed_form(A, gg["feat"][g], int(gg["label"][g]), None, 0, w, s0["M"], hp=O.default_hparams(num_epochs=1),
                                      graph_mode=True, bn=bn, return_state=True, init_state=init)
        assert np.abs(s0["vM"]).max() > 0 and np.abs(s0["mF"]).max() > 0
        for k in ("M", "F", "mM", "vM", "mF", "vF"):
            assert np.abs(r1[k] - s1[k]).max() <= 1e-12, (g, k)
