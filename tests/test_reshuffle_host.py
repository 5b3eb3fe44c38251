"""CPU checks of reshuffled mini-batch epochs (DESIGN.md §4.12): the NumPy restatement of the epoch permutation P
against the pure-Python Philox oracle, its bijectivity and its rank dealing, the oracle loops that take one order per
epoch, and the command line's --reshuffle option."""
import numpy as np
import pytest

import oracle
from tests import helpers, lazy_adam_oracle, reshuffle_oracle as ro


def test_vectorised_philox_equals_the_oracle():
    rs = np.random.RandomState(0)
    for _ in range(20):
        ctr = [int(x) for x in rs.randint(0, 2 ** 32, size=4, dtype=np.uint64)]
        key = [int(x) for x in rs.randint(0, 2 ** 32, size=2, dtype=np.uint64)]
        got = [int(w[()]) for w in ro.philox4x32_10(*ctr, *key)]
        assert got == oracle.philox4x32_10(ctr, key)


def test_round_function_is_the_oracle_philox():
    """One Feistel round of P restated with oracle.philox4x32_10 on scalars."""
    n, seed, epoch = 1000, (7 << 32) | 3, 4
    h = ro.half_bits(n)
    assert h == 5                                   # 2^10 = 1024 >= 1000
    for x in (0, 1, 517, 1023):
        L, R = x >> h, x & ((1 << h) - 1)
        for r in range(4):
            w = oracle.philox4x32_10([R, ro.DOMAIN | r, epoch, n], [seed & 0xFFFFFFFF, seed >> 32])
            L, R = R, L ^ (w[0] & ((1 << h) - 1))
        assert int(ro.feistel(np.array([x], dtype=np.uint64), h, seed, epoch, n)[0]) == (L << h) | R


@pytest.mark.parametrize("n", [1, 2, 3, 1000, 2 ** 20 + 3])
def test_perm_is_a_bijection(n):
    for seed, epoch in ((0, 1), (12345, 7)):
        p = ro.perm(seed, epoch, n)
        assert p.dtype == np.int64 and p.shape == (n,)
        assert (np.sort(p) == np.arange(n)).all()


def test_perm_depends_on_seed_epoch_and_n():
    a = ro.perm(0, 1, 1000)
    assert (a != np.arange(1000)).mean() > 0.9
    assert (a != ro.perm(0, 2, 1000)).mean() > 0.9
    assert (a != ro.perm(1, 1, 1000)).mean() > 0.9
    assert (a == ro.perm(0, 1, 1000)).all()


@pytest.mark.parametrize("world", [2, 3, 8])
def test_rank_shares_interleave_into_the_one_rank_list(world):
    tr = np.random.RandomState(1).permutation(1003).astype(np.int64)
    one = ro.epoch_list(tr, 5, 3)
    back = np.empty_like(one)
    for r in range(world):
        back[r::world] = ro.epoch_list(tr, 5, 3, r, world)
    assert (back == one).all()


def test_order_loops_with_fixed_orders_equal_the_fixed_batch_loops():
    V, N, D, B = 200, 300, 16, 64
    rowptr, gene, label = helpers.random_windows(N, V, 1, 12, seed=3)
    W0, Wo0 = helpers.init_weights(V, D, 1)
    tr, _ = oracle.split_indices(N, 0)
    a = lazy_adam_oracle.lazy_minibatch_train(rowptr, gene, label, tr, W0, Wo0, 0.005, B, 2)
    b = ro.lazy_minibatch_train_orders(rowptr, gene, label, [tr, tr], W0, Wo0, 0.005, B)
    assert all((x == y).all() for x, y in zip(a, b))
    c = ro.lazy_minibatch_train_orders(rowptr, gene, label, ro.epoch_orders(tr, 0, 2), W0, Wo0, 0.005, B)
    assert not (c[0] == a[0]).all()
    d = ro.dense_minibatch_train_orders(rowptr, gene, label, ro.epoch_orders(tr, 0, 2), W0, Wo0, 0.005, B, "sgd")
    assert np.isfinite(d[0]).all()


def test_command_line_reshuffle_option(capsys):
    from g2vec_b200 import cli
    base = ["e.tsv", "c.tsv", "n.tsv", "out"]
    assert cli.parse_arguments(base).reshuffle is False
    assert cli.parse_arguments(base + ["--batch", "64", "--reshuffle"]).reshuffle is True
    with pytest.raises(SystemExit):
        cli.parse_arguments(base + ["--reshuffle"])
    assert "--reshuffle needs mini-batches" in capsys.readouterr().err
