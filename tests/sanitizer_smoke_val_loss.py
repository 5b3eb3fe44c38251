"""The validation-loss monitor's kernels (g2v_cbow_val_loss, g2v_cbow_st_prepare, g2v_cbow_loop_decide[_best]_score)
inside short runs whose chunks replay as CUDA graphs, and in the host-driven mini-batch loop, meant to be executed under
compute-sanitizer on a GPU box, like tests/sanitizer_smoke.py:

    compute-sanitizer --tool memcheck  python tests/sanitizer_smoke_val_loss.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_val_loss.py

(not a pytest test).  Each run's stop and best steps are checked against the loss rule on its own loss trajectory, and
the rank1 and deterministic runs are repeated bit for bit."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import g2vec_b200 as g2v
    from tests import helpers, val_loss_oracle as vo

    V, N, D = 300, 700, 40
    rowptr, gene, label = helpers.random_windows(N, V, 0, 40, seed=5)
    W0, Wo0 = helpers.init_weights(V, D, 1)
    n_va = N - int(N * 0.8)
    for algo, det, batch, opt, patience in (("rows", True, 0, "adam", 1), ("rows", False, 0, "adam", 3),
                                            ("rank1", False, 0, "adam", 2), ("rows", False, 100, "lazy_adam", 2)):
        kw = dict(seed=0, W_ih0=W0, W_ho0=Wo0, log=None, algo=algo, deterministic=det, batch=batch, optimizer=opt,
                  patience=patience, monitor="val_loss", lr_patience=2, lr_factor=0.5, return_info=True)
        # 16 steps at most: step 0 eagerly, then captured 5-step chunks (full batch)
        W, info = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, max_epoch=16, **kw)
        Qs = [int(round(l * n_va * 2 ** 24)) for l in info["val_loss"]]
        assert (info["stop_step"], info["best_step"]) == vo.apply_rule(Qs, patience), (algo, batch, info["stop_step"])
        assert info["graph"] == (batch == 0)
        if det or algo == "rank1":
            W2, info2 = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, max_epoch=16, **kw)
            assert W.tobytes() == W2.tobytes() and info2["val_loss"] == info["val_loss"], algo
    print("val loss sanitizer smoke OK")


if __name__ == "__main__":
    main()
