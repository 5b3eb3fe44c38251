"""The differential co-expression kernels (csrc/g2v_dcx.cu) at their tile edges, meant to be executed under
compute-sanitizer on a GPU box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_diffcoex.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_diffcoex.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  sums in both forms at n_b in {1, 129}
(inside and past the 128-row CTA tile), E in {1, 65} (inside and past the 64-pair tile) and n in {3, 33} (one and two
32-sample slabs); tally at E = 1, 129 and 300 (partial 128-pair tiles) with one row and with several rows per CTA.
Every result is checked against tests/diffcoex_oracle.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import test_gpu_diffcoex as t, diffcoex_oracle
    launches = 0
    rs = np.random.RandomState(0)
    for n in (3, 33):
        for nb in (1, 129):
            for E in (1, 65):
                q = rs.randint(-(1 << 16), (1 << 16) + 1, size=(n, 9)).astype(np.int64)
                S_pad = -(-n // 32) * 32
                M = np.zeros((nb, S_pad), np.uint8); M[:, :n] = rs.randint(0, 2, size=(nb, n))
                pi, pj = rs.randint(0, 9, E), rs.randint(0, 9, E)
                assert (t.gpu_sums(M, q, pi, pj) == diffcoex_oracle.sums(M, q, pi, pj)).all()
                launches += 1
    for n, G, E, nb, k in ((8, 6, 1, 1, 4), (40, 12, 65, 129, 10)):
        args = t._stat_case(rs, n, G, E, nb, k)
        M, q, pi, pj, n, k, A, Bq, At, Bt, Pt = args
        want = diffcoex_oracle.stats(n, k, A, Bq, diffcoex_oracle.sums(M, q, pi, pj), At, Bt, Pt, pi, pj)
        assert np.array_equal(t.gpu_stats(*args), want)
        launches += 1
    for E, nb in ((1, 1), (129, 3), (300, 700)):
        D_obs = rs.rand(E)
        D = rs.rand(nb, E)
        got, want = t.gpu_tally(D, D_obs), diffcoex_oracle.tally(D, D_obs)
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
        launches += 1
    print("sanitizer smoke (differential co-expression) OK: %d launches" % launches)


if __name__ == "__main__":
    main()
