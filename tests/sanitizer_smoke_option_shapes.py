"""Each launch branch of the class-weighted and weight-decayed CBOW kernels that tests/test_gpu_cbow_f64_options.py
reaches, once at a small size, meant to be executed under compute-sanitizer on a GPU box, like
tests/sanitizer_smoke_shapes.py:

    compute-sanitizer --tool memcheck  python tests/sanitizer_smoke_option_shapes.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_option_shapes.py

(not a pytest test): the weighted generic rows kernels below and above 48 KB of shared memory and at D % 4 != 0, the
weighted VEC kernels, the loop tail, the weighted generic kernels at the largest admitted D and the refusal of D + 1,
the decayed dense update at V*D % 4 in {1, 2, 3}, the decayed lazy Adam with a W_ho step over two blocks, and the
decayed rank-1 update on a VEC path and with opt-in shared memory.  Every result is checked as the pytest file checks
it."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from tests import test_gpu_cbow_f64_options as t
    from g2vec_b200 import _capi
    p = torch.cuda.get_device_properties(0)
    env = {"lib": _capi.load(), "capi": _capi, "sm": p.multi_processor_count, "optin": p.shared_memory_per_block_optin}
    for D, V, n in ((3, 1201, 9), (132, 1201, 9), (128, 1201, 9), (769, 1201, 9), (1000, 1201, 9)):
        for mode, reduce in (("dyadic", "sum"), ("realistic", "mean")):
            t.test_class_weighted_routes_at_every_shape(env, D, V, n, mode, reduce, t.CW_DYADIC)
        t.test_lazy_decay_on_the_problem_rows(env, D, V, n)
    t.test_lazy_decay_on_the_problem_rows(env, 300, 1201, 9)
    t.test_largest_hidden_size_runs_weighted_and_the_next_is_refused(env)
    for D, V in ((1, 4097), (130, 1001), (3, 1001)):
        t.test_dense_decay_at_every_tail(env, D, V, 2, t.LAM)
    for D in (3, 256, 1537):
        t.test_rank1_decay_at_every_path(env, D)
    torch.cuda.synchronize()
    print("option shapes sanitizer smoke OK")


if __name__ == "__main__":
    main()
