"""Every kernel of the deterministic mode once (the tiled forward for D = 128, 256, 512 and a generic D, the tile sum,
the batch expansion, the carried tail pass inside a captured loop), meant to be executed under compute-sanitizer on a
GPU box, like tests/sanitizer_smoke.py:

    compute-sanitizer --tool memcheck  python tests/sanitizer_smoke_deterministic.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_deterministic.py

(not a pytest test).  Each run is checked against the default (atomic) path of the same configuration."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def rel_max(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def main():
    import g2vec_b200 as g2v
    from tests import helpers

    V, N, B = 300, 700, 128                      # 560 training windows: 9 tiles, the last one partial
    rowptr, gene, label = helpers.random_windows(N, V, 1, 40, seed=5)
    for D in (128, 256, 512, 40):
        W0, Wo0 = helpers.init_weights(V, D, 1)
        kw = dict(seed=0, W_ih0=W0, W_ho0=Wo0, early_stop=False, log=None)
        # full batch: step 0 eagerly, then a captured chunk with the carried tail pass
        got = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=6, deterministic=True, **kw)
        want = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=6, **kw)
        assert rel_max(got, want) < 1e-4, D
        # mini-batches: tiled forward per batch + batch expansion + dense update
        got = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=2, batch=B, deterministic=True, **kw)
        want = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=2, batch=B, **kw)
        assert rel_max(got, want) < 1e-4, D
    print("deterministic sanitizer smoke OK")


if __name__ == "__main__":
    main()
