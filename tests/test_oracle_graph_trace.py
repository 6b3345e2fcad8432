"""CPU: pins tests/golden/graph_trace_golden.npz -- what the UNMODIFIED reference prints with print_training=True in graph mode
(loss, mask density, softmax row per epoch; tools/gen_graph_trace_golden.py) -- against the line-by-line port, and the off-edge part of
the printed loss against an fp64 numpy restatement of its recurrence (offedge_sums), the specification of
gx_offedge_regularisers_graphs.

In graph mode the reference's size and entropy terms sum over all max_nodes^2 mask entries (explain.py:755-770): padded rows and
columns, non-edges and the diagonal included.  None of those entries reaches the masked adjacency, so each follows a private Adam
recurrence driven by the two regularisers alone (graph mode has no Laplacian term, explain.py:787-788)."""
import numpy as np
import pytest

import gnnx_oracle as O
import util
from test_oracle_state import dense_m0


def golden():
    return np.load(util.GOLDEN + "/graph_trace_golden.npz")


def graphs():
    return np.load(util.GOLDEN + "/graphs_golden.npz")


def case_hparams(tg, case):
    """The oracle hyper-parameters of a fixture case (a, b or c)."""
    over = dict(size=float(tg["b_size"]), ent=float(tg["b_ent"]), feat_size=float(tg["b_feat_size"])) if case == "b" else {}
    return O.default_hparams(num_epochs=int(tg[case + "_epochs"]), **over)


def offedge_sums(M0, on, epochs, lr=0.1, beta1=0.9, beta2=0.999, eps=1e-8, size=0.005, ent=1.0):
    """(epochs, 2) float64: per epoch (sum sigmoid(M), sum H(sigmoid(M))) over the entries of the (n, n) mask where `on` is False,
    M = the entry after e Adam steps on c_size * sigmoid(M) + c_ent * H(sigmoid(M)) / n^2 (torch.optim.Adam's update, in fp64).
    d/dM of that loss is sigmoid'(M) * (c_size - c_ent * M / n^2), since dH/dsigmoid = log((1 - s) / s) = -M."""
    n = M0.shape[0]
    M = np.asarray(M0, np.float64)[~np.asarray(on, bool)]
    m = np.zeros_like(M)
    v = np.zeros_like(M)
    out = np.zeros((epochs, 2))
    for e in range(epochs):
        S = 1.0 / (1.0 + np.exp(-M))
        out[e] = S.sum(), (-S * np.log(S) - (1 - S) * np.log(1 - S)).sum()
        g = S * (1 - S) * (size - ent * M / (n * n))
        t = e + 1
        m = beta1 * m + (1 - beta1) * g
        v = beta2 * v + (1 - beta2) * g * g
        M = M - lr / (1 - beta1 ** t) * m / (np.sqrt(v) / np.sqrt(1 - beta2 ** t) + eps)
    return out


def _port_trace(gg, g, hp):
    A = gg["adj"][g].astype(np.float64)
    W = {k: gg[k] for k in util.WKEYS}
    M0 = dense_m0(int(gg["max_nodes"]), int(gg["g%d_seed" % g]))
    tr = []
    O.explain_dense_torch(A, gg["feat"][g], int(gg["label"][g]), None, 0, W, M0, hp=hp, graph_mode=True, trace=tr)
    return A, M0, tr


def test_fixture_layout():
    tg, gg = golden(), graphs()
    C = gg["Wp"].shape[0]
    assert list(tg["a_gids"]) == list(range(int(gg["num_graphs"])))
    assert int(tg["a_epochs"]) == int(tg["b_epochs"]) == 30 and int(tg["c_epochs"]) == 12
    for case in "abc":
        for g in tg[case + "_gids"]:
            assert tg["%s_g%d" % (case, g)].shape == (int(tg[case + "_epochs"]), 2 + C)
    # the padded graphs of the stand-in do have padded rows: the off-edge sums cover them
    assert (gg["adj"].sum(axis=2) == 0).any(axis=1).sum() >= 6


@pytest.mark.parametrize("case", ["a", "b"])
def test_port_prints_what_the_reference_prints(case):
    tg, gg = golden(), graphs()
    hp = case_hparams(tg, case)
    for g in [int(x) for x in tg[case + "_gids"]]:
        ref = tg["%s_g%d" % (case, g)]
        _, _, tr = _port_trace(gg, g, hp)
        loss = np.array([r["loss"] for r in tr])
        assert np.abs(loss / ref[:, 0] - 1).max() <= 1e-6, (case, g)
        assert np.abs(np.array([r["density"] for r in tr]) - ref[:, 1]).max() <= 1e-6, (case, g)
        assert np.abs(np.stack([r["pred"] for r in tr]) - ref[:, 2:]).max() <= 2e-7, (case, g)


@pytest.mark.parametrize("case", ["a", "b"])
def test_offedge_restatement_completes_the_printed_loss(case):
    """The port's edge terms plus the fp64 off-edge recurrence give the number the reference printed."""
    tg, gg = golden(), graphs()
    hp = case_hparams(tg, case)
    n = int(gg["max_nodes"])
    for g in [int(x) for x in tg[case + "_gids"]]:
        ref = tg["%s_g%d" % (case, g)]
        A, M0, tr = _port_trace(gg, g, hp)
        off = offedge_sums(M0, A > 0, hp.num_epochs, lr=hp.lr, size=hp.size, ent=hp.ent)
        edges = np.array([r["pred_loss"] + r["size_edges"] + r["ent_edges"] + r["lap"] + r["feat_size"] for r in tr])
        loss = edges + hp.size * off[:, 0] + hp.ent * off[:, 1] / (n * n)
        assert np.abs(loss / ref[:, 0] - 1).max() <= 1e-6, (case, g, np.abs(loss / ref[:, 0] - 1).max())
        # and the port's own split agrees: its off-edge terms are the restatement's
        size_off = np.array([r["size_off"] for r in tr]); ent_off = np.array([r["ent_off"] for r in tr])
        assert np.abs(hp.size * off[:, 0] - size_off).max() <= 1e-6 * np.abs(size_off).max()
        assert np.abs(hp.ent * off[:, 1] / (n * n) - ent_off).max() <= 1e-6 * np.abs(ent_off).max()


def test_coefficients_move_the_offedge_part():
    """Case b is not case a in disguise: its printed loss differs by far more than the tolerances above, and the off-edge part
    scales with c_size and c_ent / max_nodes^2."""
    tg, gg = golden(), graphs()
    n = int(gg["max_nodes"])
    for g in [int(x) for x in tg["b_gids"]]:
        a, b = tg["a_g%d" % g], tg["b_g%d" % g]
        assert np.abs(b[:, 0] / a[:, 0] - 1).min() > 1e-2
        M0 = dense_m0(n, int(gg["g%d_seed" % g]))
        on = gg["adj"][g] > 0
        off_b = offedge_sums(M0, on, 1, size=float(tg["b_size"]), ent=float(tg["b_ent"]))
        off_a = offedge_sums(M0, on, 1)
        # epoch 0 sees M0 itself: the sums agree, only the coefficients differ
        assert np.array_equal(off_a, off_b)
        part_a = 0.005 * off_a[0, 0] + 1.0 * off_a[0, 1] / (n * n)
        part_b = float(tg["b_size"]) * off_b[0, 0] + float(tg["b_ent"]) * off_b[0, 1] / (n * n)
        assert part_b > 5 * part_a
