"""The t-SNE kernels (csrc/g2v_tsne.cu) on one small map, meant to be executed under compute-sanitizer on a GPU box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_tsne.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_tsne.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  m = 300 genes crosses a 256-column block
edge of g2v_tsne_grad and of the row blocks of Z, the 64-row distance tiles and the 32-row symmetrisation tiles; D = 33
crosses a 32-d staging chunk; 260 iterations cross the stage switch at 250.  d, P and Y are checked against
tests/tsne_oracle.py (d and Y bit for bit)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import tsne_oracle
    from g2vec_b200 import _capi, tsne
    rs = np.random.RandomState(0)
    W = rs.standard_normal((300, 33)).astype(np.float32)
    before = _capi.launch_count()
    P, beta, steps = tsne.affinities(W, 20.0)
    d = tsne_oracle.dist(W.astype(np.float64))
    np.testing.assert_allclose(P, tsne_oracle.joint(tsne_oracle.conditional_from_beta(d, beta)), rtol=1e-12, atol=0)
    assert (steps < tsne.MAX_STEPS).all()
    Y0 = tsne.pca_init(W)
    Y, kl = tsne.optimize(P, Y0, 260)
    want, _ = tsne_oracle.optimize(P, Y0, 260)
    assert (Y.view(np.int64) == want.view(np.int64)).all() and np.isfinite(kl)
    print("sanitizer smoke (t-SNE) OK: %d launches" % (_capi.launch_count() - before))


if __name__ == "__main__":
    main()
