"""The NetRank kernels (csrc/g2v_nr.cu) at ordinary sizes and their tile edges, meant to be executed under
compute-sanitizer on a GPU box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_netrank.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_netrank.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  seed at n_b, G in {1, 33} (one and two
32 x 32 tiles) with ld past n_b; step on a network with degrees 0, 1, 8, 9 and 40 at 1, 33 and 64 columns in tiles of
32; tally at G = 1 and 9 (one and two 8-gene blocks) with n_b = 1 and 33.  Every result is checked against
tests/netrank_oracle.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import test_gpu_netrank as t, netrank_oracle
    from g2vec_b200 import diffcoex
    launches = 0
    rs = np.random.RandomState(0)
    for n_b in (1, 33):
        for G in (1, 33):
            A = rs.randint(-(1 << 20), 1 << 20, size=(n_b, G)).astype(np.int64)
            Q = rs.randint(-(1 << 20), 1 << 20, size=G).astype(np.int64)
            W = np.full(G, 1e30); W[0] = 0.0
            got = t.gpu_seed(A, 40, 17, Q, W, n_b + 3)
            assert np.array_equal(got[:, :n_b], netrank_oracle.seeds(A, 40, 17, Q, W))
            launches += 1
    src = np.r_[np.zeros(40, int), np.full(9, 41), np.full(8, 51), [60]]
    dst = np.r_[np.arange(1, 41), np.arange(42, 51), np.arange(52, 60), [61]]
    pairs = diffcoex.pairs_from_edges(src, dst)                 # genes 62..69 without neighbours
    for cols in (1, 33, 64):
        S = rs.uniform(size=(70, 64))
        got = t.gpu_propagate(S, pairs, 0.5, 32, n_cols=cols)
        assert np.array_equal(got[:, :cols], netrank_oracle.propagate(S[:, :cols], pairs, 0.5))
        launches += 40 * -(-cols // 32)
    for G in (1, 9):
        for n_b in (1, 33):
            x = rs.uniform(size=(G, 40))
            obs = rs.uniform(size=G)
            assert (t.gpu_tally(x, n_b, obs) == (x[:, :n_b] >= obs[:, None]).sum(axis=1)).all()
            launches += 1
    print("sanitizer smoke (netrank) OK: %d launches" % launches)


if __name__ == "__main__":
    main()
