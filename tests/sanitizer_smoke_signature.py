"""The signature-test kernels (csrc/g2v_sig.cu) at their edges, meant to be executed under compute-sanitizer on a GPU
box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_signature.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_signature.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  folds at the smallest classes (m_c = F)
and at n = 32768; draws at p = 1 and 128; fits and AUC at p = 1 and 128 on the smallest folds, and at n = 32768.  Every
result is checked against tests/signature_oracle.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import test_gpu_signature as t, signature_oracle as so
    launches = 0
    for y, F in ((np.array([0, 1, 0, 1]), 2), (np.arange(32768) % 2, 5)):
        assert (t.gpu_folds(y, 2, F, 3) == so.folds(y, 2, F, 3)).all()
        launches += 1
    for G, p in ((1, 1), (300, 128)):
        got = t.gpu_draw(G, p, 2, 1, 3)
        assert all((got[q] == so.floyd(G, p, 2, 1 + q)).all() for q in range(3))
        launches += 1
    for n, G, p, F in ((4, 1, 1, 2), (10, 128, 128, 5), (32768, 2, 2, 2)):
        x, y = t._data(n, G, n)
        fold = so.folds(y, 1, F, 1)
        genes = np.arange(p)[None, :]
        sc, it, cv, be, auc, acc = t.gpu_fit(x, y, genes, fold)
        want = so.cv(x, y, genes, fold)
        assert cv.all() and np.all(np.abs(be - want["beta"]) <= 1e-8 * np.maximum(1.0, np.abs(want["beta"]).max()))
        for f in range(F):
            te = fold[0] == f
            assert auc[0, 0, f] == so.auc_counts(sc[0, 0, te], y[te])
        launches += 2
    print("sanitizer smoke (signature test) OK: %d launches" % launches)


if __name__ == "__main__":
    main()
