"""The survival kernels (csrc/g2v_surv.cu) at their tile edges, meant to be executed under compute-sanitizer on a GPU
box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_survival.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_survival.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  rows at n in {3, 33} (one and two
rounds of 32 draws) and n_b in {1, 9}; scores at G in {1, 33} (inside and past the 32-gene warp tile), n_b in {1, 9}
(inside and past the 8-permutation CTA) and n in {3, 33} (one and two 32-position batches).  Every result is checked
against tests/survival_oracle.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from g2vec_b200 import survival
    from tests import test_gpu_survival as t, survival_oracle
    launches = 0
    rs = np.random.RandomState(0)
    for n in (3, 33):
        for nb in (1, 9):
            tt, e = t._records(rs, n)
            slot = survival.time_groups(tt, e)[1]
            assert (t.gpu_rows(slot, 5, 2, nb) == survival_oracle.rows(slot, 5, 2, nb)).all()
            launches += 1
            for G in (1, 33):
                q, idx, flags, a, c = t._score_case(rs, n, G, nb)
                got, want = t.gpu_scores(q, idx, flags, a, c), survival_oracle.scan(q, idx, flags, a, c)
                assert all(np.array_equal(g_, w_) for g_, w_ in zip(got, want))
                launches += 1
    print("sanitizer smoke (survival) OK: %d launches" % launches)


if __name__ == "__main__":
    main()
