"""The two kernels of early stopping with patience (g2v_cbow_loop_decide_best, g2v_cbow_loop_keep_best) inside short
runs whose chunks replay as CUDA graphs, meant to be executed under compute-sanitizer on a GPU box, like
tests/sanitizer_smoke.py:

    compute-sanitizer --tool memcheck  python tests/sanitizer_smoke_patience.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_patience.py

(not a pytest test).  Each run's vectors are checked against a run without early stopping that ends at its best step."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import g2vec_b200 as g2v
    from tests import helpers

    V, N, D = 300, 700, 40                       # D not a multiple of 4: the copy's scalar tail runs too
    rowptr, gene, label = helpers.random_windows(N, V, 1, 40, seed=5)
    W0, Wo0 = helpers.init_weights(V, D, 1)
    for algo, det in (("rows", True), ("rank1", False)):
        kw = dict(seed=0, W_ih0=W0, W_ho0=Wo0, log=None, algo=algo, deterministic=det)
        # 11 steps: step 0 eagerly, then two captured 5-step chunks
        got, info = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, max_epoch=11, patience=3, return_info=True, **kw)
        want = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, max_epoch=info["best_step"] + 1, early_stop=False, **kw)
        assert info["graph"] and got.tobytes() == want.tobytes(), (algo, info["stop_step"], info["best_step"])
    print("patience sanitizer smoke OK")


if __name__ == "__main__":
    main()
