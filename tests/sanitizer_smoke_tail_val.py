"""Every branch of g2v_cbow_loop_tail_val once -- D = 128, 256, 512, sum and mean, with and without class weights,
empty windows, a list shorter than one chunk, empty training or validation lists -- and a device loop whose chunks
replay as CUDA graphs, meant to be executed under compute-sanitizer on a GPU box, like tests/sanitizer_smoke.py:

    compute-sanitizer --tool memcheck  python tests/sanitizer_smoke_tail_val.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_tail_val.py
    compute-sanitizer --tool synccheck python tests/sanitizer_smoke_tail_val.py

(not a pytest test).  Each result is checked against g2v_cbow_loop_tail and g2v_cbow_eval_certified."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import numpy as np
    import torch
    import g2vec_b200 as g2v
    from g2vec_b200 import _capi
    from tests import helpers
    from tests import test_gpu_cbow_tail_val as t
    lib = _capi.load()
    V, N = 300, 700
    perm = np.random.RandomState(3).permutation(N).astype(np.int32)
    cu = lambda a: torch.from_numpy(a.copy()).cuda()
    for D in (128, 256, 512):
        case = t._case(V, D, N, 0, 40, seed=D)                       # includes empty windows
        for reduce in (_capi.REDUCE_SUM, _capi.REDUCE_MEAN):
            for cw in (None, (0.5, 2.0)):
                t._compare(lib, case, cu(perm[:500]), cu(perm[500:]), V, D, reduce, cw)
        for n_tr, n_va in ((0, 9), (9, 0), (1, 3)):
            t._compare(lib, case, cu(perm[:n_tr]), cu(perm[n_tr:n_tr + n_va]), V, D, _capi.REDUCE_SUM, None)
    rowptr, gene, label = helpers.random_windows(N, V, 1, 40, seed=5)
    W0, Wo0 = helpers.init_weights(V, 128, 1)
    _, info = g2v.train_cbow(rowptr, gene, label, V, 128, 0.05, max_epoch=11, seed=0, W_ih0=W0, W_ho0=Wo0, log=None,
                             early_stop=False, return_info=True)
    assert info["graph"]
    print("tail_val sanitizer smoke OK")


if __name__ == "__main__":
    main()
