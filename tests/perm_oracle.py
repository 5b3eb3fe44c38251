"""NumPy restatement of the label-permutation test (DESIGN.md §4.24) -- test infrastructure for
tests/test_perm_host.py and tests/test_gpu_perm.py:

* ``labels(obs, S_pad, seed, b_begin, n_b)``: the indicator rows of g2v_perm_labels, Fisher-Yates vectorised over the
  permutations with the Philox4x32-10 of tests/reshuffle_oracle.py and the 64 x 64 -> high 64 product from 32-bit
  halves;
* ``sums``: the int64 matmul of g2v_perm_sums;
* ``tally``: the counts of g2v_perm_tally, vectorised (reverse cumulative max for maxT);
* ``maxt_counts_naive``: the step-down maxT counts straight from the definition, O(B G^2), to pin the fast form;
* ``perm_test``: the whole test on the host, the counts through ``tally``.
"""
import numpy as np

from g2vec_b200 import perm
from tests.reshuffle_oracle import philox4x32_10

_M32 = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def mulhi64(a, b):
    """High 64 bits of the 128-bit product of uint64 arrays, from 32-bit halves."""
    a = np.asarray(a, dtype=np.uint64); b = np.asarray(b, dtype=np.uint64)
    a0, a1, b0, b1 = a & _M32, a >> _S32, b & _M32, b >> _S32
    p00, p01, p10, p11 = a0 * b0, a0 * b1, a1 * b0, a1 * b1
    mid = (p00 >> _S32) + (p01 & _M32) + (p10 & _M32)
    return p11 + (p01 >> _S32) + (p10 >> _S32) + (mid >> _S32)


def draw64(seed, b, s):
    """draw64(seed, 2^63 + b, s) of csrc/g2v_common.cuh for an array of permutation numbers b."""
    b = np.asarray(b, dtype=np.uint64)
    lo, hi = b & _M32, (b >> _S32) | np.uint64(0x80000000)
    w = philox4x32_10(s >> 1, 0, lo, hi, seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    w = [x.astype(np.uint64) for x in w]
    return (w[3] << _S32) | w[2] if s & 1 else (w[1] << _S32) | w[0]


def labels(obs, S_pad, seed, b_begin, n_b):
    """Rows b = b_begin + 1 .. b_begin + n_b: uint8 [n_b, S_pad]."""
    obs = np.asarray(obs, dtype=np.uint8)
    n = obs.shape[0]
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    rows = np.zeros((n_b, S_pad), dtype=np.uint8)
    rows[:, :n] = obs
    b = np.arange(b_begin + 1, b_begin + n_b + 1, dtype=np.uint64)
    ar = np.arange(n_b)
    for i in range(n - 1, 0, -1):
        j = mulhi64(draw64(seed, b, n - 1 - i), np.uint64(i + 1)).astype(np.int64)
        xi = rows[:, i].copy()
        rows[:, i] = rows[ar, j]
        rows[ar, j] = xi
    return rows


def sums(M, q_rank):
    """A = M . q, exact int64: M [n_b, S_pad] (only the first n columns can be 1), q_rank [n, G]."""
    n = q_rank.shape[0]
    return M[:, :n].astype(np.int64) @ q_rank


def tally(A, n, k, Q, W, absN_obs, rho_obs):
    """(count, count_maxt) of the rows of A, all arrays in rank order."""
    N = n * A - k * np.asarray(Q)[None, :]
    count = (np.abs(N) >= absN_obs[None, :]).sum(axis=0)
    rho = perm.rho_of(N, np.asarray(W)[None, :])
    u = np.maximum.accumulate(rho[:, ::-1], axis=1)[:, ::-1]
    return count.astype(np.int64), (u >= rho_obs[None, :]).sum(axis=0).astype(np.int64)


def maxt_counts_naive(rho_perm, rho_obs):
    """c~_j = #{b : max over ranks k >= j of rho_b[r_k] >= rho_obs[r_j]}, rho_perm [B, G] and rho_obs [G] in GENE
    order; the ranks r sort rho_obs descending, ties by gene index.  Returns c~ in rank order."""
    G = rho_obs.shape[0]
    r = sorted(range(G), key=lambda g: (-rho_obs[g], g))
    out = np.zeros(G, dtype=np.int64)
    for j in range(G):
        for b in range(rho_perm.shape[0]):
            if max(rho_perm[b, r[kk]] for kk in range(j, G)) >= rho_obs[r[j]]:
                out[j] += 1
    return out


def perm_test(expr, label, n_perm, seed=0, chunk=None):
    """The whole test on the host: PermResult with the same counts as perm.perm_test."""
    prep = perm.prepare(expr, label, n_perm)
    o, n, k = prep["order"], prep["n"], prep["k"]
    S_pad = -(-n // 32) * 32
    qr = prep["q"][:, o]
    c = np.zeros(len(o), np.int64); cm = np.zeros(len(o), np.int64)
    chunk = chunk or n_perm
    for b0 in range(0, n_perm, chunk):
        M = labels(prep["obs"], S_pad, seed, b0, min(chunk, n_perm - b0))
        a, b = tally(sums(M, qr), n, k, prep["Q"][o], prep["W"][o], np.abs(prep["N_obs"][o]), prep["rho_obs"][o])
        c += a; cm += b
    return perm.finish(prep, c, cm, n_perm)
