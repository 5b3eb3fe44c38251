"""Every branch of the one-GPU simulation of the multi-GPU exchange (tests/test_gpu_cbow_exchange.py) once at a small
size -- the peer load/store path of g2v_cbow_update_nvl with Adam (host and device alpha) and SGD, the scalar tail,
world 3 with ranks that own nothing, one rank alone, the CUDA-graph replay, and g2v_cbow_loop_counters_nvl followed by
g2v_cbow_loop_decide_best -- meant to be executed under compute-sanitizer on a GPU box, like
tests/sanitizer_smoke.py:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_exchange.py

(not a pytest test).  Each result is checked as the test file checks it."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from g2vec_b200 import _capi
    from tests import test_gpu_cbow_exchange as X
    env = {"lib": _capi.load(), "capi": _capi, "sm": torch.cuda.get_device_properties(0).multi_processor_count}
    # n = 3003 (tail of 3), n = 2 (no float4: only the tail), n = 5 (rank 0 owns the one float4), n = 7 at world 2
    for world, V, D in ((3, 1000, 3), (3, 1, 1), (3, 4, 1), (2, 6, 1)):
        X.test_update_nvl_dyadic_is_the_dense_update_bit_for_bit(env, world, V, D)
        X.test_update_nvl_each_rank_changes_exactly_its_slice(env, world, V, D)
    X.test_update_nvl_realistic_within_float64_bound(env, 3, 1000, 3)
    X.test_update_nvl_twelve_steps_eager_and_graph_replay(env, 3, 1000, 3)
    X.test_counter_exchange_and_decision_on_the_summed_counters(env, 3, "best3")
    torch.cuda.synchronize()
    print("exchange sanitizer smoke OK")


if __name__ == "__main__":
    main()
