"""Each kernel branch that only odd or large shapes reach, once at a tiny size, meant to be executed under
compute-sanitizer on a GPU box, like tests/sanitizer_smoke.py:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_shapes.py

(not a pytest test): the scalar paths of D % 4 != 0 and the scalar tails of V*D % 4 != 0 (expansions, lazy Adam,
rank-1 prepare, dense update, snapshot), the generic rows kernels with opt-in shared memory (D > 768), the rank-1
update with opt-in shared memory (D > 1536), a 4096-gene window (D = 3, V = 4097), canonicalisation at L > 1024 and
the sampler's fused canonical epilogue on walks longer than 1024 nodes.
Every result is checked against the float64 reference of tests/f64_reference.py."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from tests import test_gpu_cbow_f64 as t, test_gpu_glue_edges as ge
    from g2vec_b200 import _capi
    p = torch.cuda.get_device_properties(0)
    env = {"lib": _capi.load(), "capi": _capi, "sm": p.multi_processor_count, "optin": p.shared_memory_per_block_optin}
    for D, V, n in ((3, 4097, 9), (130, 1201, 9), (769, 1201, 9), (1537, 1201, 9)):
        for mode in ("dyadic", "realistic"):
            t.test_rows_forward_and_backward_entry_points(env, D, V, n, mode, "sum")
        t.test_expansions_lazy_adam_and_rank1(env, D, V, n)
        t.test_dense_update_against_float64_adam_and_sgd(env, D, V, 2)
        t.test_loop_begin_snapshot_copies_every_element(env, D, V)
    ge.test_canonicalise_long_rows_equals_numpy_sort(env["lib"], 1025)
    mp = pytest.MonkeyPatch()
    try:
        ge.test_fused_canonical_walks_longer_than_300_nodes(env["lib"], mp, 1365, "hash")
    finally:
        mp.undo()
    torch.cuda.synchronize()
    print("shapes sanitizer smoke OK")


if __name__ == "__main__":
    main()
