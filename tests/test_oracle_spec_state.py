"""CPU: the feature-mask parameter F that oracle/kernel_spec.py returns next to the edge mask (return_F=True) against the dense
closed form's state, fp64.  The kernels return sigmoid(F) after num_epochs - 1 updates; explain_closed_form(num_epochs - 1,
return_state=True) stops at the same point (the convention test_masks_match_oracle_random uses for the feature mask)."""
import networkx as nx
import numpy as np
import pytest

import gnnx_oracle as O
import kernel_spec as KS


def _case(N, m, graph_seed, d, C, L, seed, hid=20):
    rng = np.random.default_rng(seed)
    G = nx.barabasi_albert_graph(N, m, seed=graph_seed)
    rowptr, col = O.csr_from_edges(N, np.array(G.edges(), dtype=np.int64))
    feat = rng.normal(size=(N, d)); label = rng.integers(0, C, N); pred_label = rng.integers(0, C, N)
    sc = lambda *s: rng.normal(size=s) * 0.5
    w = {}
    dims = [d] + [hid] * L
    for l in range(1, L + 1):
        w["W%d" % l] = sc(dims[l - 1], dims[l]); w["b%d" % l] = sc(dims[l])
    w["Wp"] = sc(C, hid * L); w["bp"] = sc(C)
    return rowptr, col, feat, label, pred_label, w


def _closed_form_F(srp, scol, sfeat, gt, pl, idx, w, m0, epochs, bn):
    A = O.dense_from_csr(srp, scol)
    ei, ej = np.nonzero(A)
    M0 = np.zeros(A.shape); M0[ei, ej] = m0
    _, st = O.explain_closed_form(A, sfeat, gt, pl, idx, w, M0, hp=O.default_hparams(num_epochs=epochs - 1), bn=bn, return_state=True)
    return st["F"]


@pytest.mark.parametrize("L,bn", [(2, True), (3, False), (3, True), (4, True)])
def test_edge_list_spec_returns_the_closed_form_feature_state(L, bn):
    rowptr, col, feat, label, pred_label, w = _case(70, 2, L, 9, 4, L, 10 * L + int(bn))
    E = 20
    for node in (3, 41):
        idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(rowptr, col, feat, label, node, L)
        m0 = 1 + 0.2 * np.random.default_rng(node).normal(size=len(scol))
        a, _ = KS.explain_pruned_edges(srp, scol, sfeat, slabel[idx], pred_label[nbrs], idx, w, m0, num_epochs=E, bn=bn)
        a2, _, F = KS.explain_pruned_edges(srp, scol, sfeat, slabel[idx], pred_label[nbrs], idx, w, m0, num_epochs=E, bn=bn, return_F=True)
        assert np.array_equal(a, a2)                   # the option changes nothing else
        ref = _closed_form_F(srp, scol, sfeat, slabel[idx], pred_label[nbrs], idx, w, m0, E, bn)
        assert F.shape == (feat.shape[1],) and np.abs(F).max() > 0.1
        assert np.abs(F - ref).max() <= 1e-10, (L, bn, node, np.abs(F - ref).max())


def test_sparse_spec_returns_the_closed_form_feature_state():
    rowptr, col, feat, label, pred_label, w = _case(120, 3, 9, 16, 4, 3, 3)
    E = 12
    for node in (0, 57):
        idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(rowptr, col, feat, label, node, 3)
        m0 = 1 + 0.2 * np.random.default_rng(node).normal(size=len(scol))
        a = KS.explain_pruned_edges_sparse(srp, scol, sfeat, slabel[idx], pred_label[nbrs], idx, w, m0, num_epochs=E, chunk=64)
        a2, F = KS.explain_pruned_edges_sparse(srp, scol, sfeat, slabel[idx], pred_label[nbrs], idx, w, m0, num_epochs=E, chunk=64, return_F=True)
        assert np.array_equal(a, a2)
        ref = _closed_form_F(srp, scol, sfeat, slabel[idx], pred_label[nbrs], idx, w, m0, E, False)
        assert np.abs(F).max() > 0.1
        assert np.abs(F - ref).max() <= 1e-10, (node, np.abs(F - ref).max())


def test_one_epoch_leaves_F_at_zero():
    # num_epochs = 1: no update is taken, F is still its initial zero (the kernels return sigmoid(0) = 0.5)
    rowptr, col, feat, label, pred_label, w = _case(40, 2, 1, 5, 3, 3, 1)
    idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(rowptr, col, feat, label, 7, 3)
    m0 = np.ones(len(scol))
    _, _, F = KS.explain_pruned_edges(srp, scol, sfeat, slabel[idx], pred_label[nbrs], idx, w, m0, num_epochs=1, return_F=True)
    _, F2 = KS.explain_pruned_edges_sparse(srp, scol, sfeat, slabel[idx], pred_label[nbrs], idx, w, m0, num_epochs=1, return_F=True)
    assert not F.any() and not F2.any()
