"""NumPy restatement of the exact t-SNE map (DESIGN.md §4.27), items 1-6 of the contract in its order -- test
infrastructure for tests/test_tsne_host.py and tests/test_gpu_tsne.py:

* ``dist``: d_ij = the chain acc = acc + t*t, t = x_id - x_jd, over d ascending from +0 (NumPy does not contract to fma);
* ``conditional``: scikit-learn's _binary_search_perplexity in float64, vectorised over rows, its sums the sequential
  chains of the Cython loop; (c, beta, steps) with the steps convention of tsne.py;
* ``conditional_from_beta``: c of given betas (to compare the GPU's P with, from the GPU's betas);
* ``joint``: P = (c + c^T) / (2m);
* ``partials``, ``gradient``, ``step``, ``optimize``: the iteration, its j chains vectorised over rows with a loop over
  j inside each block of tsne.BLOCK columns;
* ``kl``: the KL divergence at Y.
"""
import numpy as np

from g2vec_b200 import tsne
from tests.kmeans_oracle import chain


def dist(X):
    """[m, m] float64 distances of the rows of X [m, D] (float64)."""
    X = np.asarray(X, dtype=np.float64)
    acc = np.zeros((X.shape[0], X.shape[0]))
    for d in range(X.shape[1]):
        t = X[:, None, d] - X[None, :, d]
        acc = acc + t * t
    return acc


def _entropy(d, beta, off):
    """S (0 -> float32(1e-8)), H and e/S of every row at its beta, the sums in the Cython loop's order."""
    e = np.where(off, np.exp(-d * beta[:, None]), 0.0)
    S = chain(e, axis=1)
    S = np.where(S == 0.0, float(np.float32(1e-8)), S)
    Pc = e / S[:, None]
    H = np.log(S) + beta * chain(d * Pc, axis=1)
    return S, H, Pc


def conditional(d, perplexity):
    """(c [m, m], beta [m], steps [m] int32) of the distances d [m, m] (float64)."""
    d = np.asarray(d, dtype=np.float64)
    m = d.shape[0]
    off = ~np.eye(m, dtype=bool)
    target = np.log(float(perplexity))
    beta = np.ones(m)
    lo, hi = np.full(m, -np.inf), np.full(m, np.inf)
    steps = np.full(m, tsne.MAX_STEPS, dtype=np.int32)
    done = np.zeros(m, dtype=bool)
    c = np.zeros((m, m))
    for l in range(tsne.MAX_STEPS):
        _, H, Pc = _entropy(d, beta, off)
        c[~done] = Pc[~done]
        diff = H - target
        ok = ~done & (np.abs(diff) <= tsne.TOLERANCE)
        steps[ok] = l
        done |= ok
        if done.all() or l == tsne.MAX_STEPS - 1:
            break
        up = ~done & (diff > 0.0)
        down = ~done & ~(diff > 0.0)
        lo = np.where(up, beta, lo)
        hi = np.where(down, beta, hi)
        beta = np.where(up, np.where(hi == np.inf, beta * 2.0, (beta + hi) / 2.0), beta)
        beta = np.where(down, np.where(lo == -np.inf, beta / 2.0, (beta + lo) / 2.0), beta)
    return c, beta, steps


def conditional_from_beta(d, beta):
    d = np.asarray(d, dtype=np.float64)
    return _entropy(d, np.asarray(beta, dtype=np.float64), ~np.eye(d.shape[0], dtype=bool))[2]


def row_sums(d, beta):
    """S of every row at its beta, before the floor at float32(1e-8)."""
    d = np.asarray(d, dtype=np.float64)
    off = ~np.eye(d.shape[0], dtype=bool)
    return chain(np.where(off, np.exp(-d * np.asarray(beta, dtype=np.float64)[:, None]), 0.0), axis=1)


def entropy(d, beta):
    """H of every row at its beta (to recheck the tolerance)."""
    d = np.asarray(d, dtype=np.float64)
    return _entropy(d, np.asarray(beta, dtype=np.float64), ~np.eye(d.shape[0], dtype=bool))[1]


def joint(c):
    return (c + c.T) / float(2 * c.shape[0])


def blocked(v):
    """The chain of v [m] inside blocks of tsne.BLOCK, then over the block partials."""
    v = np.asarray(v, dtype=np.float64)
    nb = -(-v.shape[0] // tsne.BLOCK)
    pad = np.zeros(nb * tsne.BLOCK - v.shape[0])             # +0 after the last row leaves its block's chain alone
    return chain(chain(np.concatenate([v, pad]).reshape(nb, tsne.BLOCK), axis=1), axis=0)


def partials(P, Y):
    """[nb, 5, m]: per column block the chains over its j != i of w, a t_0, a t_1, r t_0, r t_1."""
    m = Y.shape[0]
    nb = -(-m // tsne.BLOCK)
    out = np.zeros((nb, 5, m))
    rows = np.arange(m)
    for b in range(nb):
        z, a0, a1, r0, r1 = (np.zeros(m) for _ in range(5))
        for j in range(b * tsne.BLOCK, min(m, (b + 1) * tsne.BLOCK)):
            t0 = Y[:, 0] - Y[j, 0]
            t1 = Y[:, 1] - Y[j, 1]
            w = 1.0 / (1.0 + (t0 * t0 + t1 * t1))
            a = P[:, j] * w
            r = w * w
            keep = rows != j
            z = np.where(keep, z + w, z)
            a0 = np.where(keep, a0 + a * t0, a0)
            a1 = np.where(keep, a1 + a * t1, a1)
            r0 = np.where(keep, r0 + r * t0, r0)
            r1 = np.where(keep, r1 + r * t1, r1)
        out[b] = (z, a0, a1, r0, r1)
    return out


def gradient(P, Y, alpha):
    """(g [m, 2], Z): g = 4 ((alpha A) - (R / Z))."""
    rows = chain(partials(P, Y), axis=0)                     # [5, m]
    Z = blocked(rows[0])
    g = 4.0 * ((alpha * rows[1:3].T) - (rows[3:5].T / Z))
    return g, Z


def stage(it):
    """(alpha, momentum, reset of u and the gains) of iteration it."""
    early = it < tsne.EXPLORATION
    return (tsne.EXAGGERATION if early else 1.0), (0.5 if early else 0.8), it in (0, tsne.EXPLORATION)


def step(g, Y, u, gains, it, eta):
    """scikit-learn's _gradient_descent update: (Y, u, gains) after iteration it with the gradient g."""
    _, mu, reset = stage(it)
    if reset:
        u, gains = np.zeros_like(Y), np.ones_like(Y)
    inc = u * g < 0.0
    gains = np.where(inc, gains + 0.2, gains * 0.8)
    gains = np.maximum(gains, 0.01)
    g = g * gains
    u = mu * u - eta * g
    return Y + u, u, gains


def optimize(P, Y0, n_iter, snapshots=()):
    """Y after n_iter iterations from Y0, and {it: Y after it iterations} for it in snapshots."""
    P = np.asarray(P, dtype=np.float64)
    Y = np.array(Y0, dtype=np.float64)
    eta = tsne.learning_rate(Y.shape[0])
    u = gains = None
    snap = {}
    for it in range(n_iter):
        g, _ = gradient(P, Y, stage(it)[0])
        Y, u, gains = step(g, Y, u, gains, it, eta)
        if it + 1 in snapshots:
            snap[it + 1] = Y.copy()
    return Y, snap


def kl(P, Y):
    m = Y.shape[0]
    off = ~np.eye(m, dtype=bool)
    t = Y[:, None, :] - Y[None, :, :]
    w = np.where(off, 1.0 / (1.0 + (t[..., 0] ** 2 + t[..., 1] ** 2)), 0.0)
    q = w / w.sum()
    eps = np.finfo(np.float64).eps
    with np.errstate(divide="ignore"):
        terms = P * np.log(np.maximum(P, eps) / np.maximum(q, eps))
    return float(terms[off].sum())
