"""Early stopping with patience (DESIGN.md §4.15) on the host: the loop log and its rule (g2vec_b200.cbow._LoopLog)
fed with the per-step counters of the two golden problems, the CPU restatement of the training loop
(tests/patience_oracle.py), and the checks of the argument.  CPU."""
import numpy as np
import pytest

import oracle
from g2vec_b200 import cbow
from tests import helpers, patience_oracle

# (golden, patience) -> (stop step, best step): the full-batch trajectories of the CPU oracle
TABLE = {("cbow_small.npz", 1): (8, 7), ("cbow_small.npz", 3): (10, 7), ("cbow_small.npz", 5): (12, 7),
         ("cbow_small.npz", 10): (53, 43),
         ("cbow_ex.npz", 1): (14, 13), ("cbow_ex.npz", 3): (16, 13), ("cbow_ex.npz", 5): (23, 18),
         ("cbow_ex.npz", 10): (28, 18)}
STEPS = {"cbow_small.npz": 120, "cbow_ex.npz": 70}
_runs = {}


def trajectory(name):
    """(golden, correct validation counts, correct training counts) of STEPS[name] steps without early stopping."""
    if name not in _runs:
        g = helpers.cbow_golden(name)
        _, hist, stop, best = patience_oracle.cbow_train(g["rowptr"], g["gene"], g["label"], g["tr"], g["va"], g["W0"],
                                                         g["Wo0"], g["lr"], max_steps=STEPS[name],
                                                         patience=STEPS[name] + 1)
        assert stop is None and len(hist) == STEPS[name]
        n_tr, n_va = len(g["tr"]), len(g["va"])
        val = np.rint(np.array([h[1] for h in hist]) * n_va).astype(np.int64)
        trc = np.rint(np.array([h[2] for h in hist]) * n_tr).astype(np.int64)
        _runs[name] = (g, val, trc)
    return _runs[name]


def feed(name, patience, max_steps=None, carried=False):
    """Run _LoopLog over the trajectory as the device loop does (the stop decided by the rule); returns (log, lines)."""
    g, val, trc = trajectory(name)
    lines = []
    log = cbow._LoopLog(len(g["tr"]), len(g["va"]), lines.append, patience)
    for s in range(len(val) if max_steps is None else max_steps):
        shown = carried or s % 5 == 0
        acc = [0, trc[s - 1] if s else 0, val[s], trc[s] if shown else 0]
        if log.step(s, acc, shown, log.stops(acc)):
            return log, lines, s
    log.end()
    return log, lines, None


def test_patience_one_prints_the_reference_log_from_the_golden_counters():
    g = helpers.cbow_golden("cbow_ex.npz")
    n_tr, n_va = len(g["tr"]), len(g["va"])
    val = np.rint(g["acc_val"].astype(np.float64) * n_va).astype(np.int64)
    trc = np.rint(g["acc_tr"].astype(np.float64) * n_tr).astype(np.int64)
    stop = g["stop_step"]
    for patience in (1, None):           # None: what the loops pass without early stopping -- it never stops
        lines = []
        log = cbow._LoopLog(n_tr, n_va, lines.append, patience)
        for s in range(len(val)):
            shown = s % 5 == 0
            acc = [0, trc[s - 1] if s else 0, val[s], trc[s] if shown else 0]
            assert log.stops(acc) == (patience == 1 and s == stop)
            assert log.step(s, acc, shown, log.stops(acc)) == (patience == 1 and s == stop)
        strip = lambda l: l.split(" (")[0]
        ref = [strip(l) for l in g["log"].splitlines()[1:-1]]
        if patience == 1:
            assert [strip(l) for l in lines] == ref
            assert log.best_step == stop - 1
        else:
            assert [strip(l) for l in lines] == ref[:-1]        # no Epoch(stop) line
            assert log.best_step == stop


@pytest.mark.parametrize("name", ["cbow_small.npz", "cbow_ex.npz"])
@pytest.mark.parametrize("patience", [1, 3, 5, 10])
def test_loop_log_gives_the_stop_and_best_steps_and_names_the_best_step(name, patience):
    want_stop, want_best = TABLE[(name, patience)]
    g, val, trc = trajectory(name)
    for carried in (False, True):
        log, lines, stop = feed(name, patience, carried=carried)
        assert (stop, log.best_step) == (want_stop, want_best)
        assert patience_oracle.apply_rule(val, patience) == (want_stop, want_best)
        f32 = np.float32
        a_val = f32(val[want_best]) / f32(len(g["va"]))
        a_tr = f32(trc[want_best]) / f32(len(g["tr"]))
        assert lines[-1].startswith("    - Epoch(stop): %03d\tACC[val]=%.4f\tACC[tr]=%.4f (" % (want_best, a_val, a_tr))
        assert not any("Epoch(best)" in l for l in lines)
        assert sum(l.startswith("    - Epoch: ") for l in lines) == want_stop // 5 + 1
        assert [h[0] for h in log.hist] == list(range(want_stop + 1))
        assert all(h[2] is not None for h in log.hist[:-1])


def test_a_run_that_reaches_max_epoch_prints_the_best_epoch():
    g, val, trc = trajectory("cbow_ex.npz")
    # patience 10: best 18, the bad steps 19..24 pending at max_epoch = 25
    log, lines, stop = feed("cbow_ex.npz", 10, max_steps=25, carried=True)
    assert stop is None and log.best_step == 18
    f32 = np.float32
    assert lines[-1] == "    - Epoch(best): 018\tACC[val]=%.4f\tACC[tr]=%.4f" % (f32(val[18]) / f32(len(g["va"])),
                                                                              f32(trc[18]) / f32(len(g["tr"])))
    # the last step is the best one: no extra line
    log, lines, stop = feed("cbow_ex.npz", 10, max_steps=19, carried=True)
    assert stop is None and log.best_step == 18 and not any("Epoch(best)" in l for l in lines)
    # patience 1 never ends a run with a better earlier step
    log, lines, stop = feed("cbow_ex.npz", 1, max_steps=13)
    assert stop is None and log.best_step == 12 and not any("Epoch(best)" in l for l in lines)


@pytest.mark.parametrize("name", ["cbow_small.npz", "cbow_ex.npz"])
def test_patience_oracle_reproduces_the_table_and_keeps_the_best_weights(name):
    g = helpers.cbow_golden(name)
    args = (g["rowptr"], g["gene"], g["label"], g["tr"], g["va"], g["W0"], g["Wo0"], g["lr"])
    _, val, _ = trajectory(name)
    for patience in (1, 3, 5, 10):
        want_stop, want_best = TABLE[(name, patience)]
        W, hist, stop, best = patience_oracle.cbow_train(*args, max_steps=want_stop + 1, patience=patience)
        assert (stop, best) == (want_stop, want_best) and len(hist) == want_stop + 1
        W_best, _, _, _ = oracle.cbow_train(*args, max_steps=want_best + 1, early_stop=False)
        assert W.tobytes() == W_best.tobytes()
    # patience 1 is the reference's rule: the same run as oracle.cbow_train, bit for bit
    W1, hist1, stop1, _ = patience_oracle.cbow_train(*args, max_steps=500, patience=1)
    W0, hist0, stop0, _ = oracle.cbow_train(*args, max_steps=500)
    assert stop1 == stop0 == g["stop_step"] and hist1 == hist0 and W1.tobytes() == W0.tobytes()
    assert [round(h[1] * len(g["va"])) for h in hist1] == list(val[:stop1 + 1])


@pytest.mark.parametrize("bad", [0, -3, 2.0, 1.5, "5", True, None])
def test_patience_must_be_a_positive_int(bad):
    with pytest.raises(ValueError, match="patience"):
        cbow.check_config("rows", "adam", False, patience=bad)
    with pytest.raises(ValueError, match="patience"):          # refused before any device work
        cbow.train_cbow(np.array([0, 1, 2, 3]), np.array([0, 1, 0]), np.array([0, 1, 0]), 2, 4, 0.005, log=None,
                        patience=bad)
    for good in (1, 2, np.int64(7)):
        cbow.check_config("rows", "adam", False, patience=good)


def test_command_line_patience():
    from g2vec_b200 import cli
    assert cli.parse_arguments(["E", "C", "N", "R"]).patience == 1
    assert cli.parse_arguments(["E", "C", "N", "R", "--patience", "5"]).patience == 5
    for bad in ("0", "-1", "1.5", "x"):
        with pytest.raises(SystemExit):
            cli.parse_arguments(["E", "C", "N", "R", "--patience", bad])
