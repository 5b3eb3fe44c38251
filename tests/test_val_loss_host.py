"""The validation-loss monitor (DESIGN.md §4.19) on the host: the fixed-point terms, both rules and their sentinels on
hand-made Q trajectories, the loop log (g2vec_b200.cbow._LoopLog), the argument checks, and the trajectories of the two
golden problems under the CPU oracle (tests/val_loss_oracle.py).  CPU."""
import math

import numpy as np
import pytest

from g2vec_b200 import cbow
from tests import helpers, patience_oracle, val_loss_oracle as vo

STEPS = {"cbow_small.npz": 40, "cbow_ex.npz": 25}
_runs = {}


def trajectory(name):
    """(golden, validation counts, training counts, Q) of STEPS[name] full-batch steps without early stopping."""
    if name not in _runs:
        g = helpers.cbow_golden(name)
        _, hist, Qs, stop, _ = vo.cbow_train(g["rowptr"], g["gene"], g["label"], g["tr"], g["va"], g["W0"], g["Wo0"],
                                             g["lr"], max_steps=STEPS[name], patience=STEPS[name] + 1)
        assert stop is None and len(Qs) == STEPS[name]
        val = np.rint(np.array([h[1] for h in hist]) * len(g["va"])).astype(np.int64)
        trc = np.rint(np.array([h[2] for h in hist]) * len(g["tr"])).astype(np.int64)
        _runs[name] = (g, val, trc, Qs)
    return _runs[name]


def feed(n_tr, n_va, counts, Qs, patience, monitor="val_loss"):
    lines = []
    log = cbow._LoopLog(n_tr, n_va, lines.append, patience, monitor=monitor)
    for s, (v, q) in enumerate(zip(counts, Qs)):
        acc = [0, 0, int(v), 1]
        if log.step(s, acc, True, log.stops(acc, q), q):
            return log, lines, s
    log.end()
    return log, lines, None


def test_fixed_point_terms():
    ln2 = int(np.rint(math.log(2.0) * 2 ** 24))
    assert list(vo.q_terms([0.0, 0.0], [0, 1])) == [ln2, ln2]
    cap = 64 * 2 ** 24
    assert list(vo.q_terms([np.inf, -np.inf, np.nan, 1e3, -1e3], [0, 1, 1, 0, 1])) == [cap] * 5
    assert list(vo.q_terms([1e3, -1e3, 60.0], [1, 0, 0])) == [0, 0, int(np.rint((60 + math.log1p(math.exp(-60))) * 2 ** 24))]
    # the bound of the header: fewer than 2^32 windows keep Q < 2^62, so the score 2^62 - Q stays positive
    assert (2 ** 32 - 1) * cap < cbow.SCORE_TOP
    assert cbow.val_loss_mean(3 * 2 ** 24, 2) == 1.5 and cbow.val_loss_mean(0, 0) == 0.0


@pytest.mark.parametrize("patience", [1, 2, 3])
def test_early_stop_rule_on_hand_made_trajectories(patience):
    cases = [[5, 4, 4, 3, 6, 7, 8, 2, 9, 9, 9],       # ties become the best (the later step)
             [10, 11, 12, 13, 1],                     # the first step is the best until the end
             [2 ** 62 - 1, 2 ** 62 - 2, 2 ** 62],     # the largest Q a list can have is still above the sentinel
             [7], [3, 3, 3, 3]]
    for Qs in cases:
        want = vo.apply_rule(Qs, patience)
        log, _, stop = feed(10, 10, [0] * len(Qs), Qs, patience)
        assert (stop, log.best_step) == want
        # the score form the device decides on gives the same: higher score = lower Q
        assert patience_oracle.apply_rule([cbow.SCORE_TOP - q for q in Qs], patience) == want
    assert vo.apply_rule([5, 4, 4, 3, 6], 1) == (4, 3)
    assert vo.apply_rule([5, 4, 4, 3, 6, 7, 8, 2], 3) == (6, 3)
    assert vo.apply_rule([1, 2], 1) == (1, 0)          # the first step is always the best, whatever its Q
    assert vo.apply_rule([9, 9, 9], 1) == (None, 2)    # ties: the later step


def test_plateau_rule_on_the_loss():
    used, cuts, _ = vo.rates([5, 5, 4, 4, 4, 3, 9, 9], 0.01, 2)
    assert cuts == [4, 7]                               # a tie is no improvement; the first step always improves
    used, cuts, _ = vo.rates([2 ** 62 - 1, 2 ** 62 - 1], 0.01, 1)
    assert cuts == [1]                                  # the first step beats the -1 sentinel even at the largest Q


def test_log_lines_with_and_without_the_loss():
    n_va = 4
    Qs = [4 * 2 ** 24, 3 * 2 ** 24, 2 * 2 ** 24, 5 * 2 ** 24]
    log, lines, stop = feed(8, n_va, [1, 2, 2, 2], Qs, 1)
    assert stop == 3 and log.best_step == 2
    assert lines[0].startswith("    - Epoch: 000\tACC[val]=0.2500\tACC[tr]=0.1250\tLOSS[val]=1.000000 (")
    assert lines[-1].startswith("    - Epoch(stop): 002\tACC[val]=0.5000\tACC[tr]=0.1250\tLOSS[val]=0.500000 (")
    assert log.losses == [1.0, 0.75, 0.5, 1.25]
    # Epoch(best) carries the loss too
    log, lines, stop = feed(8, n_va, [1, 2, 2, 2], Qs, 5)
    assert stop is None and lines[-1] == "    - Epoch(best): 002\tACC[val]=0.5000\tACC[tr]=0.1250\tLOSS[val]=0.500000"
    # val_acc: the lines of the accuracy rule, with no loss
    log, lines, stop = feed(8, n_va, [1, 2, 2, 1], Qs, 1, monitor="val_acc")
    assert stop == 3 and log.best_step == 2 and log.losses == []
    assert lines[0].startswith("    - Epoch: 000\tACC[val]=0.2500\tACC[tr]=0.1250 (")
    assert lines[-1].startswith("    - Epoch(stop): 002\tACC[val]=0.5000\tACC[tr]=0.1250 (")
    assert not any("LOSS" in l for l in lines)


@pytest.mark.parametrize("name,want_loss,want_acc", [("cbow_small.npz", (25, 24), (8, 7)),
                                                     ("cbow_ex.npz", (11, 10), (14, 13))])
def test_golden_trajectories_pick_different_steps(name, want_loss, want_acc):
    g, val, trc, Qs = trajectory(name)
    assert vo.apply_rule(Qs, 1) == want_loss
    assert patience_oracle.apply_rule(val, 1) == want_acc
    log, lines, stop = feed(len(g["tr"]), len(g["va"]), val, Qs, 1)
    assert (stop, log.best_step) == want_loss
    assert "LOSS[val]=%.6f" % vo.mean_loss(Qs[want_loss[1]], len(g["va"])) in lines[-1]
    log, lines, stop = feed(len(g["tr"]), len(g["va"]), val, Qs, 1, monitor="val_acc")
    assert (stop, log.best_step) == want_acc
    # the loss changes by far more than float32 rounding at the decisions
    for s in (want_loss[0], want_loss[1]):
        assert abs(Qs[s] - Qs[s - 1]) / (len(g["va"]) << 24) > 1e-4


def test_golden_trainer_stops_where_the_rule_says():
    g = helpers.cbow_golden("cbow_small.npz")
    W, hist, Qs, stop, best = vo.cbow_train(g["rowptr"], g["gene"], g["label"], g["tr"], g["va"], g["W0"], g["Wo0"],
                                            g["lr"], max_steps=60, patience=1)
    assert (stop, best) == (25, 24) and len(Qs) == 26
    assert abs(vo.mean_loss(Qs[24], len(g["va"])) - 0.53718) < 1e-5


def test_float32_logits_follow_the_lane_order():
    rs = np.random.RandomState(3)
    rowptr, gene, label = helpers.random_windows(40, 200, 0, 60, 4)
    s = rs.standard_normal(200).astype(np.float32)
    win = np.arange(40)
    z32 = vo.logits32(rowptr, gene, win, s)
    z64 = np.array([s[gene[rowptr[i]:rowptr[i + 1]]].astype(np.float64).sum() for i in win])
    assert np.allclose(z32, z64, rtol=0, atol=1e-4)
    assert all(z32[i] == 0 for i in win if rowptr[i] == rowptr[i + 1])


@pytest.mark.parametrize("bad", ["loss", "val_accuracy", None, 1, ""])
def test_monitor_is_refused_before_device_work(bad):
    with pytest.raises(ValueError, match="monitor"):
        cbow.check_config("rows", "adam", False, monitor=bad)
    with pytest.raises(ValueError, match="monitor"):
        cbow.train_cbow(np.array([0, 1, 2, 3]), np.array([0, 1, 0]), np.array([0, 1, 0]), 2, 4, 0.005, log=None,
                        monitor=bad)
    for good in cbow.MONITORS:
        cbow.check_config("rows", "adam", False, monitor=good)


def test_command_line_monitor():
    from g2vec_b200 import cli
    assert cli.parse_arguments(["E", "C", "N", "R"]).monitor == "val_acc"
    assert cli.parse_arguments(["E", "C", "N", "R", "--monitor", "val_loss"]).monitor == "val_loss"
    for bad in ("loss", "VAL_LOSS", ""):
        with pytest.raises(SystemExit):
            cli.parse_arguments(["E", "C", "N", "R", "--monitor", bad])
    assert "--monitor" in cli.__doc__ and "LOSS[val]" in cli.__doc__
