"""Tiny reshuffled lazy_adam run (epoch-order kernel + batch-plan builder + lazy steps), and the builder on lists that
reach its every path (segments of 1-2, 3-32, 33-4096 and more than 4096 positions; several waves), meant to be
executed under compute-sanitizer on a GPU box, like tests/sanitizer_smoke.py:

    compute-sanitizer --tool memcheck  python tests/sanitizer_smoke_reshuffle.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_reshuffle.py

(not a pytest test).  The training result is checked against the CPU restatement fed the restated epoch orders, the
plans against the torch.sort construction the builder replaced."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def check_plans(g2v):
    import torch
    from g2vec_b200 import cbow
    from tests import helpers, reshuffle_oracle as ro
    rs = np.random.RandomState(9)
    for V, N, lmax, hub, Bs in ((50, 5000, 5, True, (40, 4500)), (200_000, 300, 30, False, (8,))):
        lens = rs.randint(1, lmax + 1, size=N)
        rowptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        gene = np.concatenate([np.sort(rs.choice(V, size=k, replace=False)) for k in lens]).astype(np.int32)
        if hub:
            gene[rowptr[:-1]] = 0                    # gene 0 in every window: a segment per batch of B positions
        label = (rs.rand(N) < 0.5).astype(np.uint8)
        W0, Wo0 = helpers.init_weights(V, 8, 0)
        m = g2v.CbowModel(rowptr, gene, label, V, 8, W0, Wo0, optimizer="lazy_adam")
        wd = torch.from_numpy(rs.permutation(N).astype(np.int32)).cuda()
        for B in Bs:                                 # V = 200k, B = 8: 38 batches in waves of 20
            got = [x.cpu().numpy() for x in cbow.batch_plan(m, wd, B)]
            want = ro.batch_plan_torch(m.rowptr, m.gene, V, wd, B)
            assert all(a.shape == b.shape and (a == b).all() for a, b in zip(got, want)), (V, B)


def main():
    import g2vec_b200 as g2v
    import oracle
    from tests import helpers, reshuffle_oracle as ro

    V, N, D, B = 400, 300, 32, 64
    rowptr, gene, label = helpers.random_windows(N, V, 1, 40, seed=5)
    W0, Wo0 = helpers.init_weights(V, D, 1)
    tr, _ = oracle.split_indices(N, 0)
    want, _ = ro.lazy_minibatch_train_orders(rowptr, gene, label, ro.epoch_orders(tr, 0, 3), W0, Wo0, 0.005, B)
    got = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=3, seed=0, W_ih0=W0, W_ho0=Wo0, early_stop=False,
                         log=None, batch=B, optimizer="lazy_adam", reshuffle=True)
    err = float(np.abs(got - want).max() / np.abs(want).max())
    assert err < 1e-4, err
    check_plans(g2v)
    print("reshuffle sanitizer smoke OK")


if __name__ == "__main__":
    main()
