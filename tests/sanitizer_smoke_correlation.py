"""The Spearman / bicor transform (csrc/g2v_corr.cu) once per method at every block size the launch picks and at the
sample cap, meant to be executed under compute-sanitizer on a GPU box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_correlation.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_correlation.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  S = 33, 64, 65, 128, 129, 256, 257,
1000, 2049 and 32768 give 32, 32, 64, 64, 128, 128, 256, 512, 1024 and 1024 threads (the bitonic sort's barriers at
every width); a few genes each, with ties and a bicor MAD = 0 gene.  Results are checked against the float64 oracle."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import test_gpu_correlation as t
    from tests.test_correlation_host import cohort
    from g2vec_b200 import _capi
    lib = _capi.load()
    launches = 0
    for S in (33, 64, 65, 128, 129, 256, 257, 1000, 2049, 32768):
        X = cohort(S, 4, S, "heavy")
        X[: S // 2 + 1, 3] = 1.5                       # MAD = 0: bicor's Pearson fallback
        a, b = t._pairs(4)
        for method in t.METHODS:
            t.check_against_oracle(lib, X, method, a, b)
            launches += 1
    print("sanitizer smoke (correlation) OK: %d transforms" % launches)


if __name__ == "__main__":
    main()
