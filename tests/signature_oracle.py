"""NumPy float64 restatement of the signature test (DESIGN.md §4.29) -- test infrastructure for
tests/test_signature_host.py and tests/test_gpu_signature.py:

* ``draw64``: draw64(seed, subsequence, s) of csrc/g2v_common.cuh for any subsequence, on perm_oracle's Philox and
  64 x 64 -> high 64 product;
* ``folds`` and ``floyd``: g2v_sig_folds and g2v_sig_draw bit for bit;
* ``standardise``, ``fit``: the training fold's z-scores and damped Newton with np.linalg.cholesky, run to a step of
  1e-13 (tighter than the kernel's 1e-10, so the kernel is compared with the minimiser, not with its own path);
* ``auc_counts`` and ``cv``: out-of-fold scores, AUC and accuracy by counting, and P_random.
"""
import numpy as np

from tests.perm_oracle import mulhi64
from tests.reshuffle_oracle import philox4x32_10

_M32 = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)
SUB_FOLDS = 1 << 61
SUB_RANDOM = (1 << 61) + (1 << 40)


def draw64(seed, subseq, s):
    """draw64(seed, subseq, s) for an int subsequence and an array (or int) of draw numbers s."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    s = np.asarray(s, dtype=np.uint64)
    w = philox4x32_10(s >> np.uint64(1), 0, subseq & 0xFFFFFFFF, (subseq >> 32) & 0xFFFFFFFF, seed & 0xFFFFFFFF,
                      seed >> 32)
    w = [x.astype(np.uint64) for x in w]
    odd = (s & np.uint64(1)).astype(bool)
    return np.where(odd, (w[3] << _S32) | w[2], (w[1] << _S32) | w[0])


def folds(y, K, F, seed):
    """int8 [K, n]: per repeat and class, the class's samples Fisher-Yates shuffled; position t -> fold t mod F."""
    y = np.asarray(y)
    n = y.shape[0]
    out = np.empty((K, n), dtype=np.int8)
    for k in range(K):
        for c in (0, 1):
            idx = np.flatnonzero(y == c)
            m = idx.shape[0]
            if m > 1:
                js = mulhi64(draw64(seed, SUB_FOLDS + 2 * k + c, np.arange(m - 1)),
                             np.arange(m, 1, -1, dtype=np.uint64)).astype(np.int64)
                for s in range(m - 1):
                    i = m - 1 - s
                    idx[i], idx[js[s]] = idx[js[s]], idx[i]
            out[k, idx] = np.arange(m) % F
    return out


def floyd(G, p, seed, r):
    """Random signature r: Floyd's sampling of p of the G genes, ascending int32 [p]."""
    u = draw64(seed, SUB_RANDOM + r, np.arange(p))
    j = np.arange(G - p, G, dtype=np.uint64)
    v = mulhi64(u, j + np.uint64(1)).astype(np.int64)
    chosen = set()
    for t in range(p):
        chosen.add(int(j[t]) if int(v[t]) in chosen else int(v[t]))
    return np.array(sorted(chosen), dtype=np.int32)


def standardise(xtr):
    """(mu, sd) per column of the training rows: mean and population SD; mu = the value, sd = 1 where min == max."""
    mu, sd = xtr.mean(axis=0), xtr.std(axis=0)
    const = xtr.min(axis=0) == xtr.max(axis=0)
    mu[const], sd[const] = xtr[0, const], 1.0
    return mu, sd


def loss(beta, Z1, y):
    eta = Z1 @ beta
    return float(np.sum(np.logaddexp(0.0, eta) - y * eta) + 0.5 * beta[1:] @ beta[1:])


def fit(Z, y, tol=1e-13, max_iter=100):
    """Ridge logistic regression (unpenalised intercept) by damped Newton from 0 with the kernel's Armijo rule (the
    loss may exceed the Armijo bound by its rounding, 2^-40 |L|): (beta [p + 1], iterations, converged)."""
    Z1 = np.hstack([np.ones((Z.shape[0], 1)), Z])
    beta = np.zeros(Z1.shape[1])
    ridge = np.eye(Z1.shape[1]); ridge[0, 0] = 0.0
    L = loss(beta, Z1, y)
    for it in range(1, max_iter + 1):
        sg = 0.5 * (1.0 + np.tanh(0.5 * (Z1 @ beta)))
        g = Z1.T @ (sg - y) + ridge @ beta
        H = (Z1 * (sg * (1.0 - sg))[:, None]).T @ Z1 + ridge
        C = np.linalg.cholesky(H)
        d = np.linalg.solve(C.T, np.linalg.solve(C, g))
        t, gd = 1.0, float(g @ d)
        for h in range(41):
            Lc = loss(beta - t * d, Z1, y)
            if Lc <= L - 1e-4 * t * gd + 2.0 ** -40 * abs(L) or h == 40:
                break
            t *= 0.5
        beta = beta - t * d
        L = Lc
        if t * np.abs(d).max() <= tol:
            return beta, it, True
    return beta, max_iter, False


def auc_counts(s, y):
    """(2 #{pos > neg} + #{pos == neg}) / (2 n_pos n_neg) of scores s with labels y, by brute force."""
    pos, neg = s[y == 1], s[y == 0]
    gt = int((pos[:, None] > neg[None, :]).sum())
    eq = int((pos[:, None] == neg[None, :]).sum())
    return (2 * gt + eq) / (2.0 * len(pos) * len(neg))


def accuracy(s, y):
    return int(((s > 0) == (y == 1)).sum()) / float(len(y))


def cv(x, y, genes, fold):
    """Every fit of the signatures genes [S, p] on the splits fold [K, n]: scores [S, K, n], beta [S, K, F, p + 1],
    auc and acc [S, K, F], n_iter [S, K, F], converged [S, K, F]."""
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y).astype(np.float64)
    S, p = genes.shape
    K, n = fold.shape
    F = int(fold.max()) + 1
    scores = np.empty((S, K, n)); beta = np.empty((S, K, F, p + 1))
    auc = np.empty((S, K, F)); acc = np.empty((S, K, F))
    n_iter = np.empty((S, K, F), dtype=np.int64); conv = np.empty((S, K, F), dtype=bool)
    for s in range(S):
        xs = x[:, genes[s]]
        for k in range(K):
            for f in range(F):
                te = fold[k] == f
                mu, sd = standardise(xs[~te])
                b, it, ok = fit((xs[~te] - mu) / sd, y[~te])
                eta = b[0] + ((xs[te] - mu) / sd) @ b[1:]
                scores[s, k, te] = eta
                beta[s, k, f], n_iter[s, k, f], conv[s, k, f] = b, it, ok
                auc[s, k, f] = auc_counts(eta, y[te])
                acc[s, k, f] = accuracy(eta, y[te])
    return {"scores": scores, "beta": beta, "auc": auc, "acc": acc, "n_iter": n_iter, "converged": conv}


def p_random(auc_mean, R):
    return np.array([(1.0 + (auc_mean[2:] >= auc_mean[s]).sum()) / (R + 1.0) for s in (0, 1)])
