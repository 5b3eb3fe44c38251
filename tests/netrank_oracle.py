"""NumPy restatement of the NetRank test (DESIGN.md §4.35) -- test infrastructure for tests/test_netrank_host.py and
tests/test_gpu_netrank.py.  Every float64 operation is the device's, in the device's order (NumPy does not contract
a * b + c into an fma), so the results are the kernels' bits:

* ``seeds(A, n, k, Q, W)``: S [G][n_b] of g2v_nr_seed from the sums A [n_b][G];
* ``step(x, S, net, d)``: one g2v_nr_step over every column, the neighbour sums in CSR order, vectorised over the
  genes by neighbour position (genes in descending degree, so the genes with a p-th neighbour are a prefix);
* ``propagate(S, pairs, d)``: T steps from x = S;
* ``netrank_test``: the whole test on the host, the rows from tests/perm_oracle.py.
"""
import numpy as np

from g2vec_b200 import netrank, perm
from tests import perm_oracle


def seeds(A, n, k, Q, W):
    N = n * np.asarray(A, np.int64) - k * np.asarray(Q, np.int64)[None, :]
    return np.sqrt(perm.rho_of(N, np.asarray(W)[None, :])).T.copy()


class Net:
    """The CSR of the pairs, and per neighbour position p the genes (descending degree) that have a p-th neighbour,
    with that neighbour and its weight."""

    def __init__(self, pairs, G):
        self.rowptr, self.col, self.deg, self.w = netrank.csr(pairs, G)
        self.G = G
        o = netrank.row_order(self.deg)
        dsort = self.deg[o]
        self.pos = []
        for p in range(int(dsort[0]) if G else 0):
            m = int((dsort > p).sum())
            rows = o[:m]
            nb = self.col[self.rowptr[rows].astype(np.int64) + p]
            self.pos.append((rows, nb, self.w[nb]))


def step(x, S, net, d):
    acc = np.zeros_like(x)
    for rows, nb, w in net.pos:
        acc[rows] = acc[rows] + x[nb] * w[:, None]
    return (1.0 - d) * S + d * acc


def propagate(S, pairs, d, net=None):
    net = net or Net(pairs, S.shape[0])
    x = S
    for _ in range(netrank.n_iterations(d)):
        x = step(x, S, net, d)
    return x


def netrank_test(expr, label, pairs, n_perm, damping=0.5, seed=0, chunk=None):
    """The whole test on the host: NetRankResult with the device's bits."""
    x, lab, pairs = netrank.check_inputs(expr, label, pairs, n_perm, damping)
    prep = perm.prepare(x, lab)
    n, k, G = prep["n"], prep["k"], x.shape[1]
    net = Net(pairs, G)
    S_pad = -(-n // 32) * 32
    q, Q, W = prep["q"], prep["Q"], prep["W"]
    M1 = np.zeros((1, S_pad), np.uint8)
    M1[0, :n] = prep["obs"]
    S_obs = seeds(perm_oracle.sums(M1, q), n, k, Q, W)
    score_obs = propagate(S_obs, pairs, damping, net)[:, 0]
    count = np.zeros(G, np.int64)
    chunk = chunk or n_perm
    for b0 in range(0, n_perm, chunk):
        M = perm_oracle.labels(prep["obs"], S_pad, seed, b0, min(chunk, n_perm - b0))
        xs = propagate(seeds(perm_oracle.sums(M, q), n, k, Q, W), pairs, damping, net)
        count += (xs >= score_obs[:, None]).sum(axis=1)
    return netrank.finish(S_obs[:, 0], score_obs, net.deg, count, netrank.n_iterations(damping), n_perm)
