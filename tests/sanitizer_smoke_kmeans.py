"""The k-means kernels (csrc/g2v_km.cu) on two small calls, meant to be executed under compute-sanitizer on a GPU box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_kmeans.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_kmeans.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  n = 300, D = 33, R = 5 runs in one
chunk with 4 restarts per assign CTA and two row blocks; n = 600, D = 20, R = 20 in chunks of 8 restarts (16 restarts
per assign CTA in none of them, then the agreement over three chunks), with duplicated rows that empty clusters.  Both
results are checked bit for bit against tests/kmeans_oracle.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import kmeans_oracle
    from g2vec_b200 import _capi, kmeans
    rs = np.random.RandomState(0)
    launches = 0
    W1 = rs.standard_normal((300, 33)).astype(np.float32)
    W2 = np.repeat(rs.standard_normal((150, 20)).astype(np.float32), 4, axis=0)
    per2 = 9 * 600 + 24 * 20 + 3 * (24 * 20 + 20) + 64
    for W, R, chunk in ((W1, 5, None), (W2, 20, 8 * per2)):
        before = _capi.launch_count()
        got = kmeans.kmeans_lgroups(W, R, seed=1, max_chunk_bytes=chunk)
        launches += _capi.launch_count() - before
        want = kmeans_oracle.kmeans_lgroups(W, R, seed=1)
        assert (got.labels == want.labels).all() and (got.seeds == want.seeds).all()
        assert (got.inertia.view(np.int64) == want.inertia.view(np.int64)).all()
        assert (got.centres.view(np.int64) == want.centres.view(np.int64)).all()
        assert (got.agreement.view(np.int64) == want.agreement.view(np.int64)).all()
    print("sanitizer smoke (k-means) OK: %d launches" % launches)


if __name__ == "__main__":
    main()
