"""The gene-set enrichment kernels (csrc/g2v_gsea.cu) at their edges, meant to be executed under compute-sanitizer on a
GPU box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_gsea.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_gsea.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  keys and rank at G = 2, 257 and 4097
with one and several rows; ES with sets of 1, 32, 33 and 4096 genes (one warp per CTA at the largest, eight below);
norm with a NaN set.  Every result is checked against tests/gsea_oracle.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import test_gpu_gsea as t, gsea_oracle as go
    launches = 0
    for n, G, nb in ((12, 2, 1), (40, 257, 3), (70, 4097, 2)):
        A, n, k, s, Q, W = t._case(n, G, nb, G)
        key, u = t.gpu_keys(A, n, k, s, Q, W)
        _, wu, wkey = go.keys(A, n, k, s, Q, W)
        assert (key == wkey).all() and (u == wu).all()
        pos = t.gpu_rank(key)
        assert (pos == go.rank(wkey)).all()
        launches += 3
        if G > 33:
            rs = np.random.RandomState(G)
            sizes = [1, 32, 33] + ([4096] if G > 4096 else [])
            members = [rs.choice(G, m, replace=False) for m in sizes]
            ptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
            gene = np.concatenate(members).astype(np.int32)
            assert t._eq(t.gpu_es(pos, u, ptr, gene), go.es(pos, u, ptr, gene))
            launches += 1
    es = np.random.RandomState(1).uniform(-1, 1, (9, 5))
    es[:, 2] = np.abs(es[:, 2])
    obs = np.array([0.5, -0.2, -0.4, 0.0, 0.9])
    for g, w in zip(t.gpu_norm(es, obs), go.norm(es, obs)):
        assert t._eq(g, w) if g.dtype == np.float64 else (g == w).all()
    launches += 1
    print("sanitizer smoke (gene-set test) OK: %d launches" % launches)


if __name__ == "__main__":
    main()
