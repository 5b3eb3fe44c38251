"""Decoupled weight decay (DESIGN.md §4.18) on the host: the float64 trainer of tests/weight_decay_oracle.py against
tests/lr_plateau_oracle.adam64_train at λ = 0, the rows it decays, and the checks of ``weight_decay`` in train_cbow /
check_config and of ``--weight-decay`` on the command line.  CPU."""
import numpy as np
import pytest

from g2vec_b200 import cbow, cli
from tests import helpers, lr_plateau_oracle as lro, weight_decay_oracle as wdo

F32 = np.float32


def _problem(seed=3, N=60, V=40, D=8):
    """Windows over genes 0..V-9 only: the last 8 rows of W_ih never receive a gradient."""
    rowptr, gene, label = helpers.random_windows(N, V - 8, 2, 6, seed)
    W0, Wo0 = helpers.init_weights(V, D, seed)
    return rowptr, gene, label, W0, Wo0


@pytest.mark.parametrize("batch,lazy", [(0, False), (16, False), (16, True), (0, True)])
def test_zero_decay_is_the_adam_trainer(batch, lazy):
    rowptr, gene, label, W0, Wo0 = _problem()
    tr = np.arange(48)
    lists = [tr, tr[::-1], tr]
    rates = [F32(0.01), F32(0.005), F32(0.005)]
    want = lro.adam64_train(rowptr, gene, label, lists, W0, Wo0, rates, batch=batch, lazy=lazy)
    got = wdo.train64(rowptr, gene, label, lists, W0, Wo0, rates, weight_decay=0.0, batch=batch,
                      optimizer="lazy_adam" if lazy else "adam")
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("optimizer", ["adam", "sgd"])
def test_rows_without_gradient_end_at_the_decay_factor(optimizer):
    rowptr, gene, label, W0, Wo0 = _problem()
    used = np.unique(gene)
    unused = np.setdiff1d(np.arange(W0.shape[0]), used)
    assert len(unused) > 0
    lam, steps = 0.05, 7
    W, _ = wdo.train64(rowptr, gene, label, [np.arange(60)] * steps, W0, Wo0, [0.01] * steps, weight_decay=lam,
                       optimizer=optimizer)
    want = W0[unused].astype(np.float64) * wdo.decay_factor(lam, steps)
    assert np.allclose(W[unused], want, rtol=1e-14, atol=0)
    assert wdo.decay_factor(lam, steps) == (1 - float(F32(lam))) ** steps
    # the float32 iterate of the kernels stays within `steps` roundings of it
    w32 = wdo.decay32(W0[unused], lam, steps).astype(np.float64)
    assert np.abs(w32 - want).max() <= steps * 2 * 2.0 ** -24 * np.abs(W0).max()


def test_lazy_decays_only_the_gathered_rows():
    rowptr, gene, label, W0, Wo0 = _problem()
    lam = 0.1
    win = np.arange(20)                                   # one batch: the genes of windows 0..19
    touched = np.unique(gene[rowptr[0]:rowptr[20]])
    rest = np.setdiff1d(np.arange(W0.shape[0]), touched)
    assert len(rest) > 0
    W, Wo = wdo.train64(rowptr, gene, label, [win], W0, Wo0, [0.01], weight_decay=lam, optimizer="lazy_adam")
    assert np.array_equal(W[rest], W0[rest].astype(np.float64))
    Wd, Wod = wdo.train64(rowptr, gene, label, [win], W0, Wo0, [0.01], weight_decay=lam, optimizer="adam")
    assert np.allclose(Wd[rest], W0[rest].astype(np.float64) * (1 - float(F32(lam))), rtol=1e-15, atol=0)
    # the gathered rows and W_ho take the same step in both (one step from zero moments)
    assert np.allclose(W[touched], Wd[touched], rtol=1e-13, atol=0) and np.allclose(Wo, Wod, rtol=1e-13, atol=0)


def test_the_decay_is_applied_once_per_batch():
    rowptr, gene, label, W0, Wo0 = _problem()
    unused = np.setdiff1d(np.arange(W0.shape[0]), np.unique(gene))
    W, _ = wdo.train64(rowptr, gene, label, [np.arange(60)] * 2, W0, Wo0, [0.01] * 2, weight_decay=0.02, batch=16)
    # 4 batches per epoch, 2 epochs: 8 decays
    assert np.allclose(W[unused], W0[unused].astype(np.float64) * wdo.decay_factor(0.02, 8), rtol=1e-14, atol=0)


def test_decay32_rounds_each_operation_on_its_own():
    w = np.array([1.0, -3.0, 0.1, 1e-30, 0.0], np.float32)
    lam = F32(0.01)
    want = np.array([F32(x - F32(lam * x)) for x in w], np.float32)
    assert wdo.decay32(w, 0.01).view(np.int32).tolist() == want.view(np.int32).tolist()


BAD = [-1, -1e-9, 1, 1.0, 1 + 1e-9, 1 - 1e-9, float("nan"), float("inf"), -float("inf"), True, "0.1", None]


@pytest.mark.parametrize("wd", BAD)
def test_check_config_and_train_cbow_refuse_bad_values(wd):
    with pytest.raises(ValueError, match="weight_decay"):
        cbow.check_config("rows", "adam", False, weight_decay=wd)
    rowptr = np.array([0, 1, 2, 3], np.int32)
    with pytest.raises(ValueError, match="weight_decay"):
        cbow.train_cbow(rowptr, np.zeros(3, np.int32), np.zeros(3, np.uint8), 4, 8, 0.01, log=None, weight_decay=wd)


def test_check_config_accepts_every_trainer_configuration():
    for wd in (0, 0.0, 1e-4, 0.5, np.float32(0.01), np.float64(0.999)):
        for algo, opt in (("rows", "adam"), ("rows", "sgd"), ("rows", "lazy_adam"), ("rank1", "adam"), ("rank1", "sgd")):
            cbow.check_config(algo, opt, False, weight_decay=wd)
        cbow.check_config("rows", "adam", True, batch=64, reshuffle=True, weight_decay=wd, lr_patience=2)
        cbow.check_config("rows", "sgd", False, several_gpus=True, weight_decay=wd)


def test_command_line_arguments():
    base = ["E", "C", "N", "R"]
    assert cli.parse_arguments(base).weight_decay == 0.0
    assert cli.parse_arguments(base + ["--weight-decay", "0.01"]).weight_decay == 0.01
    assert cli.parse_arguments(base + ["--weight-decay", "0"]).weight_decay == 0.0
    cli.parse_arguments(base + ["--weight-decay", "1e-3", "--optimizer", "lazy_adam", "--batch", "64"])
    for bad in ("-1", "1", "nan", "inf", "-inf", "1.5", "0.99999999"):
        with pytest.raises(SystemExit):
            cli.parse_arguments(base + ["--weight-decay", bad])
