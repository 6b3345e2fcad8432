"""Drop-in for utils/graph_utils.py:neighborhoods of the reference (the only function of that
module on the explainer's path; GraphSampler is a training data loader, out of scope)."""
import numpy as np


def csr_from_dense(adj):
    """Dense (N,N) 0/1 adjacency -> (rowptr int32[N+1], col int32[nnz]), columns ascending per row
    (row-major nonzero order).  Host marshalling only."""
    adj = np.asarray(adj)
    if adj.ndim != 2 or adj.shape[0] != adj.shape[1]:
        raise ValueError("adjacency must be square")
    nz = adj != 0
    vals = adj[nz]
    if vals.size and not np.all(vals == 1):
        raise NotImplementedError("weighted adjacency is not built (reference datasets are 0/1)")
    ei, ej = np.nonzero(nz)
    N = adj.shape[0]
    rowptr = np.zeros(N + 1, dtype=np.int64)
    np.add.at(rowptr, ei + 1, 1)
    return np.cumsum(rowptr).astype(np.int32), ej.astype(np.int32)


def is_sparse(adj):
    """True for a scipy.sparse matrix (scipy is only imported when it is installed)."""
    try:
        import scipy.sparse as sp
    except ImportError:
        return False
    return sp.issparse(adj)


def csr_from_sparse(adj):
    """scipy.sparse (N,N) 0/1 adjacency -> the (rowptr, col) csr_from_dense returns for adj.toarray(), without materialising the
    dense matrix: duplicates summed, explicit zeros dropped, columns ascending per row.  Host marshalling only."""
    if adj.ndim != 2 or adj.shape[0] != adj.shape[1]:
        raise ValueError("adjacency must be square")
    a = adj.tocsr(copy=True)
    a.sum_duplicates()
    a.eliminate_zeros()
    a.sort_indices()
    if a.nnz and not np.all(a.data == 1):
        raise NotImplementedError("weighted adjacency is not built (reference datasets are 0/1)")
    return a.indptr.astype(np.int32), a.indices.astype(np.int32)


def neighborhoods(adj, n_hops, use_cuda=True):
    """utils/graph_utils.py:147-158: (B,N,N) 0/1 -> (B,N,N) int, (A + A^2 + ... + A^k) > 0.

    Computed by libgnnx's integer frontier expansion on CSR (bit-exact, O(edges) instead of dense
    N^3 matmuls).  `use_cuda` is accepted for signature compatibility; the GPU is always used."""
    from .engine import Engine
    adj = np.asarray(adj)
    if adj.ndim != 3:
        raise ValueError("adj must be (B,N,N)")
    out = np.zeros(adj.shape, dtype=int)
    eng = Engine(0)
    try:
        for b in range(adj.shape[0]):
            rowptr, col = csr_from_dense(adj[b])
            N = adj.shape[1]
            # the graph upload API carries features/labels; neighbourhood rows need none of them
            eng.set_graph_csr_structure(rowptr, col)
            out[b] = eng.neighborhood_rows(np.arange(N, dtype=np.int32), n_hops)
    finally:
        eng.close()
    return out
