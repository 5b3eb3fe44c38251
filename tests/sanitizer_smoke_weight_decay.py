"""The weight-decay instantiations of the optimizer kernels (dense, lazy, rank-1) inside short runs whose full-batch
chunks replay as CUDA graphs, and in the host-driven mini-batch loop, meant to be executed under compute-sanitizer on a
GPU box, like tests/sanitizer_smoke.py:

    compute-sanitizer --tool memcheck  python tests/sanitizer_smoke_weight_decay.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_weight_decay.py

(not a pytest test).  D = 40 takes the scalar paths, D = 128 the float4 ones.  Each bit-reproducible run is repeated and
compared bit for bit, and a run at weight_decay = 0 against one without the argument."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import g2vec_b200 as g2v
    from tests import helpers

    V, N = 300, 700
    rowptr, gene, label = helpers.random_windows(N, V, 1, 40, seed=5)
    for D in (40, 128):
        W0, Wo0 = helpers.init_weights(V, D, 1)
        for algo, det, batch, opt in (("rows", True, 0, "adam"), ("rows", True, 0, "sgd"), ("rank1", False, 0, "adam"),
                                      ("rank1", False, 0, "sgd"), ("rows", True, 100, "lazy_adam"),
                                      ("rows", False, 100, "adam")):
            kw = dict(seed=0, W_ih0=W0, W_ho0=Wo0, log=None, algo=algo, deterministic=det, batch=batch, optimizer=opt,
                      early_stop=False, max_epoch=11)       # full batch: step 0 eagerly, then two captured 5-step chunks
            a = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, weight_decay=0.01, **kw)
            if det or algo == "rank1":
                b = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, weight_decay=0.01, **kw)
                assert a.tobytes() == b.tobytes(), (D, algo, opt, batch)
                c = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, weight_decay=0.0, **kw)
                d = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, **kw)
                assert c.tobytes() == d.tobytes() != a.tobytes(), (D, algo, opt, batch)
    print("weight decay sanitizer smoke OK")


if __name__ == "__main__":
    main()
