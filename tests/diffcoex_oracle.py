"""NumPy restatement of the differential co-expression test (DESIGN.md §4.30) -- test infrastructure for
tests/test_diffcoex_host.py and tests/test_gpu_diffcoex.py:

* ``sums``: the exact int64 sums of g2v_dcx_sums' P form, sum_s M[r, s] q_i[s] q_j[s];
* ``stats``: D of every row from the int64 sums of A, B and P, through diffcoex.corr_of / stat_of (the IEEE sequence
  of the kernel's epilogue);
* ``tally``: the counts of g2v_dcx_tally, vectorised (reverse cumulative max for maxT);
* ``maxt_counts_naive``: the step-down maxT counts straight from the definition, O(B E^2);
* ``diffcoex_test``: the whole test on the host, the permutation rows from tests/perm_oracle.py.
"""
import numpy as np

from g2vec_b200 import diffcoex
from tests import perm_oracle


def sums(M, q, pi, pj, block=4096):
    """S [n_b, E] int64 = M[:, :n] . (q[:, pi] * q[:, pj]), exact; q [n, G] int64, |q| <= 2^16."""
    n = q.shape[0]
    Mi = np.asarray(M)[:, :n].astype(np.int64)
    out = np.empty((Mi.shape[0], len(pi)), dtype=np.int64)
    for e0 in range(0, len(pi), block):
        sl = slice(e0, e0 + block)
        out[:, sl] = Mi @ (q[:, pi[sl]] * q[:, pj[sl]])
    return out


def stats(n, k, A, Bq, P, At, Bt, Pt, pi, pj):
    """D [n_b, E] of rows with k selected samples: A, Bq [n_b, G] and P [n_b, E] their sums, At, Bt [G] and Pt [E] the
    totals over all n samples."""
    r1 = diffcoex.corr_of(k, P, A[:, pi], A[:, pj], Bq[:, pi], Bq[:, pj])
    A2, B2, P2 = At[None, :] - A, Bt[None, :] - Bq, Pt[None, :] - P
    r2 = diffcoex.corr_of(n - k, P2, A2[:, pi], A2[:, pj], B2[:, pi], B2[:, pj])
    return diffcoex.stat_of(r1, r2)


def tally(D, D_obs):
    """(count, count_maxt) of the rows of D, everything in rank order."""
    count = (D >= D_obs[None, :]).sum(axis=0)
    u = np.maximum.accumulate(D[:, ::-1], axis=1)[:, ::-1]
    return count.astype(np.int64), (u >= D_obs[None, :]).sum(axis=0).astype(np.int64)


def maxt_counts_naive(D_perm, D_obs):
    """c~_j = #{b : max over ranks k >= j of D_b[r_k] >= D_obs[r_j]}, D_perm [B, E] and D_obs [E] in PAIR order; the
    ranks r sort D_obs descending, ties by pair index.  Returns c~ in rank order."""
    E = D_obs.shape[0]
    r = sorted(range(E), key=lambda e: (-D_obs[e], e))
    out = np.zeros(E, dtype=np.int64)
    for j in range(E):
        for b in range(D_perm.shape[0]):
            if max(D_perm[b, r[kk]] for kk in range(j, E)) >= D_obs[r[j]]:
                out[j] += 1
    return out


def observed_sums(prep):
    """A2, B2 [2, G] and P2 [2, E]: the sums of the all-ones and the observed labellings."""
    q, n, pairs = prep["q"], prep["n"], prep["pairs"]
    M2 = np.stack([np.ones(n, np.uint8), prep["obs"]])
    G = q.shape[1]
    diag = np.arange(G)
    return M2.astype(np.int64) @ q, sums(M2, q, diag, diag), sums(M2, q, pairs[:, 0], pairs[:, 1])


def diffcoex_test(expr, label, pairs, n_perm, seed=0, chunk=None):
    """The whole test on the host: a DiffCoexResult with the bits of diffcoex.diffcoex_test."""
    prep = diffcoex.prepare(expr, label, pairs, n_perm)
    q, n, k = prep["q"], prep["n"], prep["k"]
    G = q.shape[1]
    A2, B2, P2 = observed_sums(prep)
    R_good, R_poor, D_obs = diffcoex.observed(prep, A2, B2, P2)
    o = np.argsort(-D_obs, kind="stable")
    pi, pj = prep["pairs"][o, 0], prep["pairs"][o, 1]
    S_pad = -(-n // 32) * 32
    diag = np.arange(G)
    c = np.zeros(len(o), np.int64); cm = np.zeros(len(o), np.int64)
    chunk = chunk or n_perm
    for b0 in range(0, n_perm, chunk):
        M = perm_oracle.labels(prep["obs"], S_pad, seed, b0, min(chunk, n_perm - b0))
        A = perm_oracle.sums(M, q)
        D = stats(n, k, A, sums(M, q, diag, diag), sums(M, q, pi, pj), A2[0], B2[0], P2[0][o], pi, pj)
        a, b = tally(D, D_obs[o])
        c += a; cm += b
    return diffcoex.finish(prep, R_good, R_poor, D_obs, o, c, cm, n_perm)

