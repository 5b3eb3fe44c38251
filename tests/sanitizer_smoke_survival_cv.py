"""The survival-CV kernels (csrc/g2v_cox.cu) at their edges, meant to be executed under compute-sanitizer on a GPU box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_survival_cv.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_survival_cv.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  Fits and concordance at p = 1 and 128
on the smallest folds, at n = 32768 with F = 2, and the concordance of the largest folds from global memory.  Every
result is checked against tests/survival_cv_oracle.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import test_gpu_survival_cv as t, survival_cv_oracle as oc
    launches = 0
    for n, G, p, F, cap in ((4, 1, 1, 2, None), (10, 128, 128, 5, None), (32768, 2, 2, 2, None), (32768, 2, 2, 2, 0)):
        x, tm, e = t._data(n, G, n, p_event=0.9)
        order, flags, grp = oc.layout(tm, e)
        xs = x[order]
        fold = oc.folds(flags, 1, F, 1)
        genes = np.arange(p)[None, :]
        sc, it, cv, be, cnt = t.gpu_fit(xs, flags, grp, genes, fold, cap)
        want = oc.cv(xs, flags, grp, genes, fold)
        assert cv.all() and np.all(np.abs(be - want["beta"]) <= 1e-8 * np.maximum(1.0, np.abs(want["beta"]).max()))
        ev = (flags & 1).astype(bool)
        for f in range(F):
            te = fold[0] == f
            assert tuple(cnt[0, 0, f]) == oc.conc_counts(sc[0, 0, te], grp[te], ev[te])
        launches += 2
    print("sanitizer smoke (survival CV) OK: %d launches" % launches)


if __name__ == "__main__":
    main()
