"""NumPy float64 restatement of the survival CV (DESIGN.md §4.33) -- test infrastructure for
tests/test_survival_cv_host.py and tests/test_gpu_survival_cv.py.  It follows the kernel's pass structure and scaled
recurrences, one sample at a time where the kernel goes a tile at a time:

* ``objective``: pass 1 in descending time (S0, S1 under a running shift, l_k = log S0_k, m_k, the loss, the gradient
  and -sum d_k m_k m_k^T), pass 2 in ascending time (C <- C e^{l_k - l_prev} + d_k, omega_i = e^{eta_i - l_k} C);
* ``fit``: damped Newton with np.linalg.cholesky and the kernel's rules, run to a step of 1e-13 (tighter than the
  kernel's 1e-10, so the kernel is compared with the minimiser, not with its own path);
* ``conc_counts``: Harrell's comparable, concordant and tied pairs, counted pair by pair;
* ``cv``: every fit of every signature over the time positions, as survival_cv lays them out.
"""
import math

import numpy as np

from g2vec_b200 import survival
from tests import signature_oracle as so


def layout(time, event):
    """(order, flags, grp): survival.time_groups' order and flags, and the time group of every position."""
    order, _, flags, _, _ = survival.time_groups(time, event)
    end = (flags & 2).astype(bool)
    return order, flags, np.cumsum(np.r_[0, end[:-1]]).astype(np.int64)


def standardise(xs, train):
    """z [n, p] from the training rows' mean and population SD; a feature constant on them gets mu = the value,
    SD = 1, and z = 0 on the training rows."""
    xt = xs[train]
    const = xt.min(axis=0) == xt.max(axis=0)
    mu = np.where(const, xt[0], xt.mean(axis=0))
    sd = np.where(const, 1.0, xt.std(axis=0))
    return (xs - mu) / sd


def objective(z, grp, ev, beta, scratch=None):
    """(L, g, H) of the Breslow ridge objective over the rows of z [m, p] (descending time, grp nondecreasing, ev
    bool).  scratch: a dict that receives the l_k, d_k and omega of the passes."""
    m, p = z.shape
    eta = z @ beta
    M, s0, s1 = -math.inf, 0.0, np.zeros(p)
    L = -float(eta[ev].sum())
    g = beta - z[ev].sum(axis=0)
    Hm = np.zeros((p, p))
    groups = []                                        # (l_k, d_k, first row, last row + 1)
    start = 0
    for i in range(m):
        e = float(eta[i])
        if e > M:
            r = math.exp(M - e) if M > -math.inf else 0.0
            s0 *= r; s1 = s1 * r
            M = e
        w = math.exp(e - M)
        s0 += w; s1 = s1 + w * z[i]
        if i == m - 1 or grp[i + 1] != grp[i]:
            d = int(ev[start:i + 1].sum())
            lk = math.log(s0) + M
            groups.append((lk, d, start, i + 1))
            if d:
                mk = s1 / s0
                L += d * lk
                g = g + d * mk
                Hm -= d * np.outer(mk, mk)
            start = i + 1
    L += 0.5 * float(beta @ beta)
    omega = np.zeros(m)
    C, prev = 0.0, None
    for lk, d, a, b in reversed(groups):
        C = float(d) if prev is None else C * math.exp(lk - prev) + d
        prev = lk
        omega[a:b] = np.exp(eta[a:b] - lk) * C
    H = z.T @ (omega[:, None] * z) + Hm + np.eye(p)
    if scratch is not None:
        scratch.update(groups=groups, omega=omega)
    return L, g, H


def loss(z, grp, ev, beta):
    return objective(z, grp, ev, beta)[0]


def fit(z, grp, ev, step_tol=1e-13, max_iter=100):
    """(beta, n_iter, converged): damped Newton from 0 with the kernel's Armijo rule and loss slack."""
    p = z.shape[1]
    b = np.zeros(p)
    L, g, H = objective(z, grp, ev, b)
    for it in range(1, max_iter + 1):
        Lc_ = np.linalg.cholesky(H)
        d = np.linalg.solve(Lc_.T, np.linalg.solve(Lc_, g))
        gd, t = float(g @ d), 1.0
        for h in range(41):
            bc = b - t * d
            Lc = loss(z, grp, ev, bc)
            if Lc <= L - 1e-4 * t * gd + 2.0 ** -40 * abs(L) or h == 40:
                break
            t *= 0.5
        b = bc
        if t * np.abs(d).max() <= step_tol:
            return b, it, True
        L, g, H = objective(z, grp, ev, b)
    return b, max_iter, False


def conc_counts(eta, grp, ev):
    """(comparable, concordant, tied) over pairs (i, j) with grp[i] > grp[j] (t_i < t_j) and i an event, one row of
    pairs at a time."""
    eta, grp = np.asarray(eta), np.asarray(grp)
    cmp = con = tie = 0
    for i in np.flatnonzero(ev):
        ok = grp < grp[i]
        cmp += int(ok.sum())
        con += int((ok & (eta[i] > eta)).sum())
        tie += int((ok & (eta[i] == eta)).sum())
    return cmp, con, tie


def concordance(cnt):
    cmp, con, tie = cnt
    return (2.0 * con + tie) / (2.0 * cmp) if cmp else math.nan


def cv(xs, flags, grp, genes, fold):
    """Every fit over the time positions: xs [n, G] in position order, genes [S, p], fold [K, n] -> dict of beta
    [S, K, F, p], scores [S, K, n] (out-of-fold eta per position), n_iter, converged."""
    S, p = genes.shape
    K, n = fold.shape
    F = int(fold.max()) + 1
    ev = (flags & 1).astype(bool)
    beta = np.zeros((S, K, F, p))
    scores = np.full((S, K, n), np.nan)
    it = np.zeros((S, K, F), np.int32)
    conv = np.zeros((S, K, F), bool)
    for s in range(S):
        for k in range(K):
            for f in range(F):
                tr = fold[k] != f
                z = standardise(xs[:, genes[s]], tr)
                b, n_it, ok = fit(z[tr], grp[tr], ev[tr])
                beta[s, k, f], it[s, k, f], conv[s, k, f] = b, n_it, ok
                te = ~tr
                scores[s, k, te] = z[te] @ b
    return {"beta": beta, "scores": scores, "n_iter": it, "converged": conv}


def folds(flags, K, F, seed):
    """The splits over the time positions: g2v_sig_folds with y = the event flags."""
    return so.folds((np.asarray(flags) & 1).astype(np.uint8), K, F, seed)
