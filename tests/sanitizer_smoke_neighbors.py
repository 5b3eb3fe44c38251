"""The nearest-genes kernels (csrc/g2v_nbr.cu) on two small searches, meant to be executed under compute-sanitizer on a
GPU box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_neighbors.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_neighbors.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  m = 64, D = 33, K = 63 runs with one
column split (g2v_nbr_partial writes the result); m = 200, D = 40, K = 64 with several (the lists of the last split
are padded, then g2v_nbr_merge).  Both results are checked bit for bit against tests/nbr_oracle.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import nbr_oracle
    from g2vec_b200 import _capi, neighbors
    lib = _capi.load()
    rs = np.random.RandomState(0)
    launches = 0
    for m, D, K, one_split in ((64, 33, 63, True), (200, 40, 64, False)):
        assert (lib.g2v_nbr_splits(m) == 1) == one_split
        W = rs.standard_normal((m, D)).astype(np.float32)
        W[3] = W[10]                                    # a tie
        before = _capi.launch_count()
        idx, sim = neighbors.nearest_genes(W, K)
        launches += _capi.launch_count() - before
        wi, ws = nbr_oracle.nearest(W, K)
        assert (idx == wi).all() and (sim.view(np.int64) == ws.view(np.int64)).all()
    print("sanitizer smoke (nearest genes) OK: %d launches" % launches)


if __name__ == "__main__":
    main()
