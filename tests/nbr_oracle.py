"""NumPy restatement of the nearest-genes contract (DESIGN.md §4.25, g2vec_b200/neighbors.py): the float64 chain
over d, vectorised over the pairs of a block of rows, and np.lexsort((j, -s)) for the order."""
import numpy as np


def dots(A, B):
    """dot [len(A), len(B)]: ((0 + a_0 b_0) + a_1 b_1) + ... in ascending d, float64."""
    A = np.asarray(A, dtype=np.float32).astype(np.float64)
    B = np.asarray(B, dtype=np.float32).astype(np.float64)
    acc = np.zeros((A.shape[0], B.shape[0]))
    for d in range(A.shape[1]):
        acc = acc + A[:, d, None] * B[None, :, d]
    return acc


def inv_norms(W):
    W = np.asarray(W, dtype=np.float32).astype(np.float64)
    n = np.zeros(W.shape[0])
    for d in range(W.shape[1]):
        n = n + W[:, d] * W[:, d]
    out = np.zeros_like(n)
    nz = n > 0
    out[nz] = 1.0 / np.sqrt(n[nz])
    return out


def similarities(W, rows=None):
    """s [len(rows), m] of the contract, rows (default all) against every gene."""
    W = np.asarray(W, dtype=np.float32)
    rows = np.arange(W.shape[0]) if rows is None else np.asarray(rows)
    inv = inv_norms(W)
    s = (dots(W[rows], W) * inv[rows, None]) * inv[None, :]
    s[(inv[rows, None] == 0) | (inv[None, :] == 0)] = 0.0
    return s


def nearest(W, k, block=256):
    """(idx int32 [m, k], sim float64 [m, k]) of the contract."""
    W = np.asarray(W, dtype=np.float32)
    m = W.shape[0]
    idx = np.empty((m, k), dtype=np.int32)
    sim = np.empty((m, k))
    j = np.arange(m)
    for r0 in range(0, m, block):
        rows = np.arange(r0, min(m, r0 + block))
        s = similarities(W, rows)
        for t, i in enumerate(rows):
            keep = j != i
            o = np.lexsort((j[keep], -s[t, keep]))[:k]
            idx[i] = j[keep][o]
            sim[i] = s[t, keep][o]
    return idx, sim
