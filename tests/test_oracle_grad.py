"""CPU: the fp64 specifications of the gradient baseline (Explainer.explain(model="grad"), explain.py:125-133,717-738) that
tests/test_gpu_grad.py holds the kernels to: oracle.grad_closed_form (dense numpy, any number of layers, the diagonal of sub_adj
included) against torch autograd in fp64, kernel_spec.grad_edges_sparse against the dense form, and the fp32 port against the
masks the unmodified reference produced."""
import networkx as nx
import numpy as np
import pytest

import gnnx_oracle as O
import kernel_spec as KS
import util


def _weights(rng, d, C, hid, emb, L=3, scale=0.5):
    dims = [d] + [hid] * (L - 1) + [emb]
    sc = lambda *s: (rng.normal(size=s) * scale).astype(np.float32)
    w = {}
    for l in range(1, L + 1):
        w["W%d" % l] = sc(dims[l - 1], dims[l]); w["b%d" % l] = sc(dims[l])
    w["Wp"] = sc(C, hid * (L - 1) + emb); w["bp"] = sc(C)
    return w


def _case(seed, N, L, d, C, loop_frac):
    """A connected random graph with self loops on a fraction of its nodes, the k-hop neighbourhood of node 0 as the reference builds
    it (adj[nbrs][:, nbrs], diagonal kept)."""
    rng = np.random.default_rng(seed)
    G = nx.connected_watts_strogatz_graph(N, 4, 0.3, seed=seed)
    A = nx.to_numpy_array(G, nodelist=range(N))
    loops = rng.random(N) < loop_frac
    A[np.arange(N), np.arange(N)] = loops
    hop = O.neighborhoods_dense(A[None], L)[0]
    nbrs = np.nonzero(hop[0])[0]
    return A[nbrs][:, nbrs], rng.normal(size=(len(nbrs), d)), int(np.sum(hop[0][:0])), _weights(rng, d, C, 16, 12, L), loops[nbrs]


CASES = [(1, 30, 3, 10, 4, 0.0), (2, 40, 3, 7, 3, 0.3), (3, 24, 2, 5, 5, 1.0), (4, 36, 4, 9, 2, 0.5), (5, 28, 3, 1, 21, 0.2)]


@pytest.mark.parametrize("seed,N,L,d,C,loop_frac", CASES, ids=["plain", "loops30", "L2_loops_all", "L4_loops50", "d1_C21"])
def test_grad_closed_form_matches_autograd_fp64(seed, N, L, d, C, loop_frac):
    """The closed form against torch autograd, both fp64, at every label: every entry of the result, diagonal included."""
    A, X, idx, w, loops = _case(seed, N, L, d, C, loop_frac)
    assert (np.diag(A) > 0).any() == (loop_frac > 0)
    for label in range(C):
        ref = O.grad_baseline_dense_torch(A, X, label, idx, w, dtype=np.float64)
        got = O.grad_closed_form(A, X, label, idx, w)
        assert np.abs(got - ref).max() <= 1e-10, label
    if loop_frac > 0:   # a self loop's own entry sigmoid(2|g_ii|) >= 0.5
        assert (np.diag(got)[loops] >= 0.5).all()


def test_grad_closed_form_isolated_self_loop():
    """A node whose only edge is its self loop: the 1 x 1 sub-adjacency [[1]], result [[sigmoid(2|g|)]]."""
    rng = np.random.default_rng(9)
    w = _weights(rng, 6, 3, 16, 12)
    X = rng.normal(size=(1, 6))
    for label in range(3):
        ref = O.grad_baseline_dense_torch(np.ones((1, 1)), X, label, 0, w, dtype=np.float64)
        got, dA = O.grad_closed_form(np.ones((1, 1)), X, label, 0, w, return_grad=True)
        assert got.shape == (1, 1) and abs(got[0, 0] - ref[0, 0]) <= 1e-10 and got[0, 0] >= 0.5
        assert abs(got[0, 0] - 1 / (1 + np.exp(-2 * abs(dA[0, 0])))) <= 1e-15


def test_grad_closed_form_uses_the_predicted_label():
    """rand fixture nodes whose predicted label differs from their label: the result follows pred_label (autograd at pred_label)
    and differs from the one at label."""
    fx = util.load_fixture("rand")
    nodes = [n for n in range(fx.N) if fx.pred_label[n] != fx.label[n]][:3]
    assert len(nodes) == 3
    for node in nodes:
        idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(fx.rowptr, fx.col, fx.feat, fx.label, node, 3)
        A = O.dense_from_csr(srp, scol)
        got = O.grad_closed_form(A, sfeat, fx.pred_label[node], idx, fx.weights)
        ref = O.grad_baseline_dense_torch(A, sfeat, fx.pred_label[node], idx, fx.weights, dtype=np.float64)
        assert np.abs(got - ref).max() <= 1e-10, node
        other = O.grad_closed_form(A, sfeat, fx.label[node], idx, fx.weights)
        assert np.abs(other - got).max() > 1e-4, node


@pytest.mark.parametrize("seed,N,L,d,C,loop_frac", CASES, ids=["plain", "loops30", "L2_loops_all", "L4_loops50", "d1_C21"])
def test_grad_sparse_matches_dense(seed, N, L, d, C, loop_frac):
    """kernel_spec.grad_edges_sparse (CSR slots + diagonal) against the dense closed form to 1e-12."""
    A, X, idx, w, loops = _case(seed, N, L, d, C, loop_frac)
    off = A * (1 - np.eye(len(A)))
    rp, col = O.csr_from_dense(off)
    r, c = np.nonzero(off)
    for label in (0, C - 1):
        dense = O.grad_closed_form(A, X, label, idx, w)
        slots, diag = KS.grad_edges_sparse(rp, col, X, label, idx, w, loops=loops)
        assert np.abs(slots - dense[r, c]).max() <= 1e-12
        assert np.abs(diag - np.diag(dense)).max() <= 1e-12
        # without the diagonal: the edge list the kernels work on
        slots0, diag0 = KS.grad_edges_sparse(rp, col, X, label, idx, w)
        assert np.abs(slots0 - O.grad_closed_form(off, X, label, idx, w)[r, c]).max() <= 1e-12 and not diag0.any()


def test_grad_sparse_outer_edges_are_half():
    """An edge between two nodes at distance L from the explained node gets no gradient: exactly sigmoid(0) = 0.5 in fp64."""
    A, X, idx, w, _ = _case(1, 30, 3, 10, 4, 0.0)
    rp, col = O.csr_from_dense(A)
    dist = KS.hop_distances(rp, col, idx, 3)
    ei = np.repeat(np.arange(len(A)), np.diff(rp))
    outer = (dist[ei] == 3) & (dist[col] == 3)
    assert outer.any()
    slots, _ = KS.grad_edges_sparse(rp, col, X, 1, idx, w)
    assert (slots[outer] == 0.5).all() and (slots[~outer] != 0.5).all()


@pytest.mark.parametrize("which", ["syn1", "rand"])
def test_grad_port_and_closed_form_match_reference_golden(which):
    """The fp32 port (bit-for-bit the reference's computation) and the fp64 closed form against the masks the unmodified reference
    produced (tests/golden/grad_golden.npz, unchanged)."""
    fx = util.load_fixture(which)
    g = np.load(util.GOLDEN + "/grad_golden.npz")
    for node in [int(x) for x in g[which + "_nodes"]]:
        idx, srp, scol, sfeat, slabel, nbrs = O.extract_neighborhood(fx.rowptr, fx.col, fx.feat, fx.label, node, 3)
        A = O.dense_from_csr(srp, scol)
        r, c = np.nonzero(A)
        ref = g["%s_n%d_mask" % (which, node)]
        port = O.grad_baseline_dense_torch(A, sfeat, int(fx.pred_label[node]), idx, fx.weights)
        assert util.rel_l2(port[r, c], ref) <= 1e-6, node
        c64 = O.grad_closed_form(A, sfeat, int(fx.pred_label[node]), idx, fx.weights)
        assert util.rel_l2(c64[r, c], ref) <= 1e-5 and np.abs(c64[r, c] - ref).max() <= 1e-5, node
