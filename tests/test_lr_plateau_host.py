"""The reduce-on-plateau learning rate (DESIGN.md §4.17) on the host: the rule of tests/lr_plateau_oracle.py on worked
sequences, the host readers of the device state (g2vec_b200.cbow.lr_rates / lr_cut), the reduction lines of the loop
log, and the checks of the arguments in train_cbow and on the command line.  CPU."""
import numpy as np
import pytest
import torch

from g2vec_b200 import cbow, cli
from tests import lr_plateau_oracle as lro

F32 = np.float32


def test_a_tie_is_not_an_improvement():
    # best 5 at step 0; 5 and 5 tie it: two steps without improvement cut the rate at step 2
    used, cuts, last = lro.rates([5, 5, 5, 6, 6, 6], 0.01, 2, factor=0.5)
    assert cuts == [2, 5]
    assert used == [F32(0.01)] * 3 + [F32(0.005)] * 3 and last == F32(0.0025)


def test_wait_restarts_after_a_reduction():
    # K = 2: steps 1, 2 cut at 2; wait starts again, so steps 3, 4 cut at 4 -- not at 3
    _, cuts, _ = lro.rates([9, 1, 1, 1, 1, 1], 1.0, 2, factor=0.5)
    assert cuts == [2, 4]
    # an improvement in between restarts it as well
    _, cuts, _ = lro.rates([9, 1, 10, 1, 1, 11, 1], 1.0, 2, factor=0.5)
    assert cuts == [4]


def test_wait_restarts_at_the_min_lr_floor_without_a_reduction():
    used, cuts, last = lro.rates([9, 1, 1, 1, 1, 1, 1], 1.0, 2, factor=0.5, min_lr=0.4)
    # 1.0 -> 0.5 at step 2; 0.5 -> max(0.25, 0.4) = 0.4 at step 4; at step 6 the rate is at the floor: no cut
    assert cuts == [2, 4] and last == F32(0.4)
    assert used == [F32(1.0)] * 3 + [F32(0.5)] * 2 + [F32(0.4)] * 2


def test_patience_one_cuts_on_every_step_without_improvement():
    used, cuts, _ = lro.rates([3, 4, 4, 2, 5, 5], 1.0, 1, factor=0.5)
    assert cuts == [2, 3, 5]
    assert used == [F32(1), F32(1), F32(1), F32(0.5), F32(0.25), F32(0.25)]


def test_patience_larger_than_the_run_never_cuts():
    used, cuts, last = lro.rates([7] * 30, 0.005, 31)
    assert cuts == [] and used == [F32(0.005)] * 30 and last == F32(0.005)


def test_the_product_is_rounded_to_float32():
    used, cuts, last = lro.rates([1, 0, 0, 0], 0.005, 1, factor=0.1)
    want = F32(0.005)
    for _ in range(3):
        want = F32(want * F32(0.1))
    assert last == want and cuts == [1, 2, 3]
    assert float(last) != 0.005 * 0.1 ** 3                  # the float64 product differs from the float32 one
    assert all(isinstance(r, np.float32) for r in used)


def _state(lr, factor, min_lr, rates_used, steps):
    """A host copy of a g2v_cbow_lr_plateau state after ``steps`` decisions, as set_lr_plateau lays it out."""
    cap = len(rates_used)
    head = torch.tensor([1, -1, 0, 0, steps, cap, 0, 0], dtype=torch.int64)
    f = torch.zeros(4 + cap + (cap & 1), dtype=torch.float32)
    f[:3] = torch.tensor([lr, factor, min_lr])
    f[4:4 + cap] = torch.tensor(rates_used)
    return torch.cat([head, f.view(torch.int64)])


def test_host_readers_of_the_device_state():
    used, cuts, last = lro.rates([3, 4, 4, 2, 5, 5], 1.0, 1, factor=0.5)
    st = _state(float(last), 0.5, 0.0, [float(r) for r in used], 6)
    got_rates, got_cuts = cbow.lr_rates(st)
    assert got_rates == [float(r) for r in used] and got_cuts == cuts == [2, 3, 5]
    assert [cbow.lr_cut(st, s) for s in range(6)] == [None, None, 0.5, 0.25, None, 0.125]
    # mid-run: three steps decided, the rate after step 2 is the current one
    st3 = _state(0.5, 0.5, 0.0, [1.0, 1.0, 1.0, 0.0, 0.0, 0.0], 3)
    assert cbow.lr_rates(st3) == ([1.0, 1.0, 1.0], [2]) and cbow.lr_cut(st3, 2) == 0.5


def test_the_log_prints_one_line_per_reduction_between_the_epoch_lines():
    used, _, last = lro.rates([3, 4, 4, 2, 5, 5], 0.005, 1, factor=0.1)
    st = _state(float(last), 0.1, 0.0, [float(r) for r in used], 6)
    lines = []
    log = cbow._LoopLog(10, 10, lines.append, None)
    log.plateau = st
    for s, v in enumerate([3, 4, 4, 2, 5, 5]):
        log.step(s, [0, 0, v, 5], True, False)
    cut = [l for l in lines if "learning rate" in l]
    assert cut == ["    - Epoch: 002\tlearning rate -> 0.0005", "    - Epoch: 003\tlearning rate -> 5e-05",
                   "    - Epoch: 005\tlearning rate -> 5e-06"]
    assert lines.index(cut[0]) > lines.index([l for l in lines if l.startswith("    - Epoch: 000\tACC")][0])
    assert lines.index(cut[-1]) > lines.index([l for l in lines if l.startswith("    - Epoch: 005\tACC")][0])
    # without a plateau state nothing is printed
    lines2 = []
    log = cbow._LoopLog(10, 10, lines2.append, None)
    for s, v in enumerate([3, 4, 4, 2, 5, 5]):
        log.step(s, [0, 0, v, 5], True, False)
    assert not any("learning rate" in l for l in lines2) and len(lines2) == 2


@pytest.mark.parametrize("kw,msg", [
    (dict(lr_patience=-1), "lr_patience"), (dict(lr_patience=1.5), "lr_patience"), (dict(lr_patience=True), "lr_patience"),
    (dict(lr_patience=1, lr_factor=0.0), "lr_factor"), (dict(lr_patience=1, lr_factor=1.0), "lr_factor"),
    (dict(lr_patience=1, lr_factor=1.5), "lr_factor"), (dict(lr_patience=1, lr_factor=float("nan")), "lr_factor"),
    (dict(lr_patience=1, lr_factor=1 - 1e-9), "lr_factor"), (dict(lr_patience=1, lr_factor="0.5"), "lr_factor"),
    (dict(lr_patience=1, min_lr=-1e-3), "min_lr"), (dict(lr_patience=1, min_lr=float("inf")), "min_lr"),
    (dict(lr_patience=1, min_lr=float("nan")), "min_lr"),
    (dict(lr_patience=2, optimizer="sgd"), "sgd"),
])
def test_train_cbow_refuses_bad_arguments_before_any_device_work(kw, msg):
    rowptr = np.array([0, 1, 2, 3], np.int32)
    with pytest.raises(ValueError, match=msg):
        cbow.train_cbow(rowptr, np.zeros(3, np.int32), np.zeros(3, np.uint8), 4, 8, 0.01, log=None, **kw)


def test_check_config_accepts_the_schedule_with_adam_and_lazy_adam_and_sgd_when_off():
    for opt in ("adam", "lazy_adam"):
        cbow.check_config("rows", opt, False, lr_patience=3, lr_factor=0.5, min_lr=1e-6)
    cbow.check_config("rank1", "adam", False, lr_patience=1, lr_factor=np.float32(0.25), min_lr=0)
    cbow.check_config("rows", "sgd", False, lr_patience=0, lr_factor=0.1, min_lr=0.0)


def test_command_line_arguments():
    base = ["E", "C", "N", "R"]
    a = cli.parse_arguments(base)
    assert (a.lr_patience, a.lr_factor, a.min_lr) == (0, 0.1, 0.0)
    a = cli.parse_arguments(base + ["--lr-patience", "3", "--lr-factor", "0.5", "--min-lr", "1e-5"])
    assert (a.lr_patience, a.lr_factor, a.min_lr) == (3, 0.5, 1e-5)
    cli.parse_arguments(base + ["--lr-patience", "2", "--optimizer", "lazy_adam"])
    cli.parse_arguments(base + ["--optimizer", "sgd"])
    for bad in (["--lr-patience", "-1"], ["--lr-factor", "0"], ["--lr-factor", "1"], ["--lr-factor", "2"],
                ["--min-lr", "-0.1"], ["--min-lr", "inf"], ["--lr-patience", "1", "--optimizer", "sgd"]):
        with pytest.raises(SystemExit):
            cli.parse_arguments(base + bad)
