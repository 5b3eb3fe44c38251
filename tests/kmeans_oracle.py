"""NumPy restatement of the best-of-R k-means restarts (DESIGN.md §4.26) -- test infrastructure for
tests/test_kmeans_host.py and tests/test_gpu_kmeans.py:

* ``chain``: the sequential float64 sum from +0 along an axis (np.cumsum is a running sum, one rounding per step; a
  leading +0 makes an all -0 sum +0, as the chain from +0 does);
* ``dist``: the contract's distances, t = x - c and acc = acc + t*t over d ascending (NumPy does not contract to fma);
* ``blocked``: a sum over rows in blocks of kmeans.BLOCK, then over the block partials;
* ``seed_rows``: the k-means++ seeding by an integer inverse CDF, with Python integers for the 64 x 64 -> 128 products;
* ``lloyd``, ``kmeans_lgroups``: one restart and the whole call, the same KMeansResult as kmeans.kmeans_lgroups.
"""
import numpy as np

from g2vec_b200 import kmeans
from tests.reshuffle_oracle import philox4x32_10

_M32 = 0xFFFFFFFF


def draw64(seed, subseq, s):
    """draw64(seed, subseq, s) of csrc/g2v_common.cuh, Python ints in and out."""
    w = [int(x) for x in philox4x32_10(s >> 1, 0, subseq & _M32, subseq >> 32, seed & _M32, (seed >> 32) & _M32)]
    return (w[3] << 32) | w[2] if s & 1 else (w[1] << 32) | w[0]


def draws(seed, r):
    """u_0, u_1, u_2 of restart r."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return [draw64(seed, (1 << 62) + r, t) for t in range(3)]


def chain(a, axis=-1):
    a = np.moveaxis(np.asarray(a, dtype=np.float64), axis, -1)
    z = np.zeros(a.shape[:-1] + (1,))
    return np.cumsum(np.concatenate([z, a], axis=-1), axis=-1)[..., -1]


def dist(X, C):
    """[n, k] float64 distances of the rows of X [n, D] (float64) to the centres C [k, D]."""
    t = X[:, None, :] - C[None, :, :]
    return chain(t * t, axis=-1)


def blocked(v):
    """The blocked sum over the rows of v [n, ...]: a chain inside each block of BLOCK rows, then over the blocks."""
    v = np.asarray(v, dtype=np.float64)
    n = v.shape[0]
    nb = -(-n // kmeans.BLOCK)
    pad = np.zeros((nb * kmeans.BLOCK - n,) + v.shape[1:])   # +0 after the last row leaves its block's chain alone
    parts = chain(np.concatenate([v, pad]).reshape((nb, kmeans.BLOCK) + v.shape[1:]), axis=1)
    return chain(parts, axis=0)


def seed_rows(X, seed, r):
    """The three rows k-means++ picks for restart r."""
    n = X.shape[0]
    u = draws(seed, r)
    rows = [(u[0] * n) >> 64]
    for t in (1, 2):
        Dm = dist(X, X[rows]).min(axis=1)
        mx = Dm.max()
        if mx == 0.0:
            rows.append((u[t] * n) >> 64)
            continue
        q = np.floor((Dm / mx) * 4294967296.0).astype(np.uint64)
        target = (u[t] * int(q.sum())) >> 64
        rows.append(int(np.searchsorted(np.cumsum(q), np.uint64(target), side="right")))
    return rows


def lloyd(X, C, max_iter=kmeans.MAX_ITER):
    """One restart from the centres C [3, D]: (labels, centres, n_iter, inertia)."""
    C = np.array(C, dtype=np.float64)
    prev = None
    for it in range(1, max_iter + 1):
        dd = dist(X, C)
        a = np.argmin(dd, axis=1)                       # the first of equal values: the lower c
        m = dd[np.arange(X.shape[0]), a]
        cnt = np.bincount(a, minlength=3)
        if it == max_iter or (it > 1 and (a == prev).all() and (cnt > 0).all()):
            return a.astype(np.int8), C, it, float(blocked(m))
        new = C.copy()
        for c in range(3):
            if cnt[c]:
                new[c] = blocked(np.where((a == c)[:, None], X, 0.0)) / cnt[c]
        taken = []
        for c in range(3):
            if cnt[c] == 0:
                mm = m.copy()
                mm[taken] = -1.0
                i = int(np.argmax(mm))                  # the first of equal values: the lowest row
                taken.append(i)
                new[c] = X[i]
        C, prev = new, a


def contingency(a, b):
    t = np.zeros((3, 3), dtype=np.int64)
    np.add.at(t, (a.astype(np.int64), b.astype(np.int64)), 1)
    return t


def kmeans_lgroups(W, restarts, seed=0, max_iter=kmeans.MAX_ITER):
    W = kmeans.check_inputs(W, restarts)
    X = W.astype(np.float64)
    R = int(restarts)
    out = [None] * R
    seeds = np.empty((R, 3), dtype=np.int32)
    for r in range(R):
        seeds[r] = seed_rows(X, seed, r)
        out[r] = lloyd(X, X[seeds[r]], max_iter)
    labels = np.stack([o[0] for o in out])
    inertia = np.array([o[3] for o in out])
    best = int(np.argmin(inertia))
    count = np.zeros(X.shape[0], dtype=np.int64)
    reach = 0
    for r in range(R):
        p, hits = kmeans.match(contingency(labels[r], labels[best]))
        reach += hits == X.shape[0]
        count += np.array(p)[labels[r]] == labels[best]
    return kmeans.KMeansResult(labels=labels, centres=np.stack([o[1] for o in out]), inertia=inertia,
                               n_iter=np.array([o[2] for o in out], dtype=np.int32), seeds=seeds, best=best,
                               agreement=count / R, lgroups=kmeans.name_lgroups(labels[best]), reach=reach)
