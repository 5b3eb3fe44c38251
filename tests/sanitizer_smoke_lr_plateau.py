"""The two kernels of the reduce-on-plateau learning rate (g2v_cbow_lr_plateau, g2v_cbow_adam_tick_lr) inside short
runs whose chunks replay as CUDA graphs, and in the host-driven mini-batch loop, meant to be executed under
compute-sanitizer on a GPU box, like tests/sanitizer_smoke.py:

    compute-sanitizer --tool memcheck  python tests/sanitizer_smoke_lr_plateau.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_lr_plateau.py

(not a pytest test).  Each run's rates are checked against the rule on its own validation counts, and a schedule that
never fires against a run without one, bit for bit."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import g2vec_b200 as g2v
    from tests import helpers, lr_plateau_oracle as lro

    V, N, D = 300, 700, 40
    rowptr, gene, label = helpers.random_windows(N, V, 1, 40, seed=5)
    W0, Wo0 = helpers.init_weights(V, D, 1)
    for algo, det, batch, opt in (("rows", True, 0, "adam"), ("rank1", False, 0, "adam"),
                                  ("rows", False, 100, "lazy_adam")):
        kw = dict(seed=0, W_ih0=W0, W_ho0=Wo0, log=None, algo=algo, deterministic=det, batch=batch, optimizer=opt,
                  early_stop=False)
        # 11 steps: step 0 eagerly, then two captured 5-step chunks (full batch)
        _, info = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, max_epoch=11, lr_patience=1, lr_factor=0.5,
                                 return_info=True, **kw)
        used, cuts, _ = lro.rates(lro.val_counts(info), 0.05, 1, 0.5)
        assert info["lr"] == [float(r) for r in used] and info["lr_reductions"] == cuts, (algo, batch)
        assert info["graph"] == (batch == 0)
        if det or algo == "rank1":
            a = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, max_epoch=11, lr_patience=100, **kw)
            b = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, max_epoch=11, **kw)
            assert a.tobytes() == b.tobytes(), algo
    print("lr plateau sanitizer smoke OK")


if __name__ == "__main__":
    main()
