"""The lasso path kernels (csrc/g2v_lasso.cu) at small sizes and their tile edges, meant to be executed under
compute-sanitizer on a GPU box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_lasso.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_lasso.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  G in {1, 8, 9, 33} (one gene, one and
two 8-gene warp tiles, past a 32-gene CTA of g2v_lasso_grad), n in {31, 32, 33} around n_pad, 3 fits and 65 fits
(past the 64-fit tile of g2v_lasso_grad), one fit per chunk and all fits in one chunk; g2v_lasso_cd's working-set
compaction crosses its 256-thread chunks at G = 300.  Fit 0 is checked against tests/lasso_oracle.py (host KKT and
objective), and the chunkings against each other bit for bit."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from g2vec_b200 import lasso
    from tests import lasso_oracle as orc
    runs = 0
    rs = np.random.RandomState(1)
    cases = [(31, 1, 2, 1), (32, 8, 2, 1), (33, 9, 3, 1), (33, 33, 8, 8), (40, 300, 2, 1)]
    for n, G, F, K in cases:
        x = rs.randn(n, G) + rs.uniform(-1, 1, G)
        lab = np.arange(n) % 2
        x[:, 0] += 0.9 * lab
        a = lasso.lasso_cv(x, lab, folds=F, repeats=K, alpha=0.5 if G == 8 else 1.0)
        b = lasso.lasso_cv(x, lab, folds=F, repeats=K, alpha=0.5 if G == 8 else 1.0, max_chunk_bytes=1)
        for name in ("a0", "beta", "entry", "entry_abs", "kkt", "scores", "auc", "cvm"):
            assert np.array_equal(getattr(a, name), getattr(b, name)), (n, G, name)
        z, mu, sd, const = orc.standardise(x)
        y = lab.astype(np.float64)
        al = a.alpha
        for k in range(a.n_lambda):
            assert a.kkt[0, k] <= 1e-7
            assert orc.kkt(z, y, a.a0[k], a.beta[k], a.lambdas[k], al, const) <= 1e-7 + 1e-12
        runs += 2
    print("sanitizer smoke (lasso) OK: %d lasso_cv calls" % runs)


if __name__ == "__main__":
    main()
