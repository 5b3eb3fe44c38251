"""The three permutation-test kernels (csrc/g2v_perm.cu) at their tile edges, meant to be executed under
compute-sanitizer on a GPU box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_perm.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_perm.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  labels at n = 3, 33 and 32768 (one and
several 32-draw rounds, the largest row); sums at n_b, G in {1, 17, 65} (inside, on and past the 64 x 64 CTA tile and
the 32 x 32 warp tile) and S_pad in {32, 160}; tally at G = 1, 129 and 300 (partial 128-gene tiles) with one row and
with several rows per CTA.  Every result is checked against tests/perm_oracle.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import test_gpu_perm as t, perm_oracle
    from g2vec_b200 import perm
    launches = 0
    for n in (3, 33, 32768):
        obs = np.zeros(n, np.uint8); obs[: max(1, n // 3)] = 1
        S_pad = -(-n // 32) * 32
        assert (t.gpu_labels(obs, S_pad, 9, 0, 2) == perm_oracle.labels(obs, S_pad, 9, 0, 2)).all()
        launches += 1
    rs = np.random.RandomState(0)
    for S_pad in (32, 160):
        for nb in (1, 17, 65):
            for G in (1, 17, 65):
                q, pl = t._random_planes(rs, S_pad, G, S_pad)
                M = rs.randint(0, 2, size=(nb, S_pad)).astype(np.uint8)
                assert (t.gpu_sums(M, pl) == perm_oracle.sums(M, q)).all()
                launches += 1
    for n, G, nb in ((12, 1, 1), (40, 129, 3), (60, 300, 700)):
        x, lab = t.cohort(n, max(G, 3), n, n // 3)
        args = t._tally_case(rs, n, G, nb) if G >= 3 else None
        if args is None:
            prep = perm.prepare(x[:, :1], lab)
            A = perm_oracle.sums(perm_oracle.labels(prep["obs"], 32, 1, 0, nb), prep["q"])
            args = (A, n, prep["k"], prep["Q"], prep["W"], np.abs(prep["N_obs"]), prep["rho_obs"])
        got, want = t.gpu_tally(*args), perm_oracle.tally(*args)
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
        launches += 1
    print("sanitizer smoke (permutation test) OK: %d launches" % launches)


if __name__ == "__main__":
    main()
