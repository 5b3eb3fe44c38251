"""NumPy restatement of the permutation Cox score test (DESIGN.md §4.31) -- test infrastructure for
tests/test_survival_host.py and tests/test_gpu_survival.py:

* ``perms``: pi_b of every permutation, Fisher-Yates on the identity vectorised over the permutations with the draws
  of tests/perm_oracle.py (perm_oracle.draw64 / mulhi64);
* ``rows``: the idx rows of g2v_surv_rows, idx[slot[pi_b(s)]] = s;
* ``scan``: T, U and V of g2v_surv_scores, a loop over the time positions on [n_b, G] int64 arrays with the same
  float64 operations in the same order;
* ``tally``: the counts of g2v_dcx_tally (tests/diffcoex_oracle.py);
* ``survival_test``: the whole test on the host.
"""
import numpy as np

from g2vec_b200 import survival
from tests import diffcoex_oracle, perm_oracle

tally = diffcoex_oracle.tally


def perms(n, seed, b_begin, n_b):
    """int64 [n_b, n]: pi_b(s) for b = b_begin + 1 .. b_begin + n_b."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    arr = np.tile(np.arange(n, dtype=np.int64), (n_b, 1))
    b = np.arange(b_begin + 1, b_begin + n_b + 1, dtype=np.uint64)
    ar = np.arange(n_b)
    for i in range(n - 1, 0, -1):
        j = perm_oracle.mulhi64(perm_oracle.draw64(seed, b, n - 1 - i), np.uint64(i + 1)).astype(np.int64)
        xi = arr[:, i].copy()
        arr[:, i] = arr[ar, j]
        arr[ar, j] = xi
    return arr


def rows(slot, seed, b_begin, n_b):
    """uint16 [n_b, n]: idx[r][slot[pi_b(s)]] = s."""
    slot = np.asarray(slot, dtype=np.int64)
    n = slot.shape[0]
    pi = perms(n, seed, b_begin, n_b)
    out = np.empty((n_b, n), dtype=np.uint16)
    out[np.arange(n_b)[:, None], slot[pi]] = np.arange(n, dtype=np.uint16)[None, :]
    return out


def scan(q, idx, flags, a, c):
    """(T, U, V) [n_b, G] float64 of the rows idx [n_b, n] over q [n, G] int64 (|q| <= 2^16)."""
    q = np.asarray(q, dtype=np.int64)
    idx = np.asarray(idx, dtype=np.int64)
    n_b, n = idx.shape
    G = q.shape[1]
    S1 = np.zeros((n_b, G), np.int64); S2 = np.zeros((n_b, G), np.int64); E1 = np.zeros((n_b, G), np.int64)
    U = np.zeros((n_b, G)); V = np.zeros((n_b, G))
    d = 0
    for p in range(n):
        x = q[idx[:, p]]
        S1 += x
        S2 += x * x
        if flags[p] & 1:
            E1 += x
            d += 1
        if flags[p] & 2:
            if d > 0:
                S0 = np.int64(p + 1)
                num_u = S0 * E1 - np.int64(d) * S1
                num_v = S0 * S2 - S1 * S1
                U = U + num_u.astype(np.float64) * a[p]
                V = V + num_v.astype(np.float64) * c[p]
            E1[:] = 0
            d = 0
    T = np.zeros((n_b, G))
    np.divide(U * U, V, out=T, where=V > 0)
    return T, U, V


def observed(prep):
    """(T, U, V) [G] of the observed pairing: the time order itself as the one row."""
    T, U, V = scan(prep["q"], prep["order"][None, :], prep["flags"], prep["a"], prep["c"])
    return T[0], U[0], V[0]


def survival_test(expr, time, event, n_perm, seed=0, chunk=None):
    """The whole test on the host: a SurvivalResult with the bits of survival.survival_test."""
    prep = survival.prepare(expr, time, event, n_perm)
    T_obs, U, V = observed(prep)
    o = np.argsort(-T_obs, kind="stable")
    qr = prep["q"][:, o]
    c = np.zeros(len(o), np.int64); cm = np.zeros(len(o), np.int64)
    chunk = chunk or n_perm
    for b0 in range(0, n_perm, chunk):
        T = scan(qr, rows(prep["slot"], seed, b0, min(chunk, n_perm - b0)), prep["flags"], prep["a"], prep["c"])[0]
        x, y = tally(T, T_obs[o])
        c += x; cm += y
    return survival.finish(prep, T_obs, U, V, o, c, cm, n_perm)
