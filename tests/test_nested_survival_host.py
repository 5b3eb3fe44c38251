"""CPU checks of the nested survival cross-validation (g2vec_b200/nested_survival.py; DESIGN.md §4.36): the options and
every refusal (each before the library loads), check_inputs, the loop's bookkeeping with the device steps replaced,
the summaries and P_random against hand-computed values, and the writers' exact bytes."""
import math

import numpy as np
import pytest

from g2vec_b200 import cli, nested_survival as ns, pipeline, signature, survival, survival_cv
from g2vec_b200.nested_survival import NestedSurvivalResult

BASE = ["E", "C", "N", "R"]


# ------------------------------------------------------------------------------------------- options, refusals
def test_nested_survival_options(capsys):
    a = cli.parse_arguments(BASE)
    assert (a.nested_survival_cv, a.nested_survival_cv_repeats) == (0, 1)
    assert "nested_survival_cv=0, nested_survival_cv_repeats=1" in repr(a)
    a = cli.parse_arguments(BASE + ["--survival", "S", "--nested-survival-cv", "100", "--nested-survival-cv-repeats",
                                    "100", "-n", "64"])
    assert (a.nested_survival_cv, a.nested_survival_cv_repeats) == (100, 100)
    assert cli.parse_arguments(BASE + ["--survival", "S", "--nested-survival-cv", "2"]).nested_survival_cv == 2
    for bad in (["--survival", "S", "--nested-survival-cv", "1"], ["--survival", "S", "--nested-survival-cv", "101"],
                ["--survival", "S", "--nested-survival-cv", "-1"], ["--nested-survival-cv-repeats", "0"],
                ["--nested-survival-cv-repeats", "101"], ["--nested-survival-cv", "3"],
                ["--survival", "S", "--nested-survival-cv", "5", "-n", "65"]):
        with pytest.raises(SystemExit):
            cli.parse_arguments(BASE + bad)
    err = capsys.readouterr().err
    assert "--nested-survival-cv needs --survival FILE" in err and "--nested-survival-cv needs -n <= 64" in err
    assert cli.parse_arguments(BASE + ["--survival", "S", "-n", "65"]).numBiomarker == 65


def _no_device(monkeypatch):
    from g2vec_b200 import _capi

    def boom(*a, **k):
        raise AssertionError("the device was used")
    monkeypatch.setattr(_capi, "load", boom)
    monkeypatch.setattr(cli, "_distributed", boom)
    monkeypatch.setattr(pipeline, "walk_windows", boom)


def test_command_line_refuses_torchrun_before_the_device(tmp_path, capsys, monkeypatch):
    _no_device(monkeypatch)
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(SystemExit) as e:
        cli.main([str(tmp_path / n) for n in BASE] + ["--survival", "S", "--nested-survival-cv", "3"])
    assert e.value.code == 1
    out = capsys.readouterr().out
    assert out.startswith("ERROR: --nested-survival-cv: the nested loop runs on one GPU") and ">>> 0." not in out


def _survival_file(tmp_path, samples, n_events):
    sf = tmp_path / "s.tsv"
    with open(sf, "w") as f:
        f.write("SAMPLE\tTIME\tEVENT\n")
        f.writelines("%s\t%s\t%s\n" % ((s, "NA", "NA") if i % 10 == 9 else (s, i, int(i < n_events)))
                     for i, s in enumerate(samples))
    return str(sf)


@pytest.mark.parametrize("extra,msg", [(["--nested-survival-cv", "4"], "F = 4 folds need at least F events, got 3"),
                                       (["--nested-survival-cv", "3", "--nested-survival-cv-repeats", "2", "-n", "65"],
                                        None)])
def test_command_line_refuses_bad_inputs_after_step_2_before_the_device(tmp_path, capsys, monkeypatch, extra, msg):
    from g2vec_b200 import _capi
    from tests import helpers
    ef, cf, nf, _ = helpers.write_ex_tsv(tmp_path)
    samples = open(ef).readline().rstrip("\n").split("\t")[1:]
    sf = _survival_file(tmp_path, samples, 3)
    monkeypatch.setattr(_capi, "load", lambda *a, **k: (_ for _ in ()).throw(AssertionError("library")))
    monkeypatch.setattr(pipeline, "walk_windows", lambda *a, **k: (_ for _ in ()).throw(AssertionError("step 3")))
    with pytest.raises(SystemExit) as e:
        cli.main([ef, cf, nf, str(tmp_path / "r"), "--survival", sf] + extra)
    out = capsys.readouterr().out
    if msg is None:                                   # refused while parsing
        assert e.value.code == 2 and out == ""
        return
    assert e.value.code == 1
    assert "ERROR: --nested-survival-cv: " + msg in out and ">>> 3." not in out


def _inputs(n=40, G=30, seed=8):
    rs = np.random.RandomState(seed)
    x = rs.standard_normal((n, G))
    t = np.round(rs.exponential(10.0, n) / 3.0) * 3.0
    e = (rs.uniform(size=n) < 0.6).astype(np.int64)
    e[0] = 1
    return x, t, e, rs.randint(0, 2, n)


def test_check_inputs_refuses_before_anything_is_uploaded(monkeypatch):
    _no_device(monkeypatch)
    x, t, e, lab = _inputs()
    t[[4, 9]] = np.nan                                 # samples without a record are left out
    xx, tt, ee, used = ns.check_inputs(x, t, e, lab, 3, 2, p=20)
    assert xx.shape == (38, 30) and not used[[4, 9]].any() and used.sum() == 38 and (tt == t[used]).all()
    ev = e.copy(); ev[:] = 0; ev[:2] = 1
    with pytest.raises(ValueError, match="F = 3 folds need at least F events, got 2"):
        ns.check_inputs(x, t, ev, lab, 3, 1)
    th = t.copy(); th[5:] = np.nan; eh = e.copy(); eh[:5] = 1
    with pytest.raises(ValueError, match="F = 3 folds need at least 2 F samples, got 4"):
        ns.check_inputs(x, th, eh, lab, 3, 1)
    with pytest.raises(ValueError, match="both labels"):
        ns.check_inputs(x, t, e, np.zeros(40, int), 2, 1)
    for F, K, p in ((1, 1, 5), (101, 1, 5), (2.5, 1, 5), (3, 0, 5), (3, 101, 5), (3, 1, 0), (3, 1, 129)):
        with pytest.raises(ValueError):
            ns.check_inputs(np.hstack([x] * 5), t, e, lab, F, K, p=p)


# ------------------------------------------------------------------------------- the loop, device steps replaced
def test_loop_hands_selection_and_fits_exactly_their_training_samples(monkeypatch):
    """pipeline.select, survival_cv.cox_fits and survival.rank_genes replaced by host fakes: selection must get every
    expression sample outside the test fold (those without a record and of other labels included), each fit's Cox rows
    must train on the survival samples outside it, and the loop must count what the fakes return."""
    N, G, K, F = 30, 8, 2, 3
    rs = np.random.RandomState(3)
    x = rs.standard_normal((N, G)).astype(np.float32)
    y = np.array([0, 1] * 15); y[[0, 5, 11]] = 7
    t = rs.exponential(5.0, N); t[[2, 5, 17, 23]] = np.nan
    e = (np.arange(N) % 3 != 0).astype(np.int64)
    used = np.isfinite(t)
    n = int(used.sum())                                # 26 survival samples
    idx = np.flatnonzero(used)
    genes = np.array(["g%d" % i for i in range(G)])
    fold = np.array([[0, 1, 2] * 9, [2, 1, 0] * 9], np.int8)[:, :n]
    seen, ranked, calls = [], [], []

    def fake_select(expr, label, src, dst, gg, args, log=None):
        seen.append((expr.copy(), label.copy()))
        j = len(seen) - 1
        return pipeline.Selection(vectors=None, lgroup=np.array([0, 1, 2, 0, 1, 2, 0, 1]),
                                  biomarkers=[gg[j % 8], gg[(j + 1) % 8]], gene_freq={}, n_windows=100 + j,
                                  info={"best_step": j}, kmeans=None)

    def fake_rank(xx, tt, ee):
        ranked.append((xx.copy(), tt.copy(), ee.copy()))
        return np.arange(xx.shape[1])[::-1]

    def fake_cox_fits(xx, tt, ee, head, R, KK, FF, seed, fold=None, cap=None, max_chunk_bytes=None):
        calls.append((xx.copy(), tt.copy(), ee.copy(), head.copy(), KK, FF, None if fold is None else fold.copy(), cap))
        H = head.shape[0]
        j = len(calls) - 1
        counts = np.zeros((H, KK, FF, 3), np.int64)
        counts[..., 0] = 4
        counts[..., 1] = 3 if j == 0 else 2
        counts[..., 2] = j % 2
        scores = np.tile(np.arange(tt.shape[0]) + 100.0 * j, (H, KK, 1))
        return head, fold, counts, None, np.ones((H, KK, FF), np.uint8), None, scores
    monkeypatch.setattr(pipeline, "select", fake_select)
    monkeypatch.setattr(survival, "rank_genes", fake_rank)
    monkeypatch.setattr(survival_cv, "cox_fits", fake_cox_fits)
    args = cli.parse_arguments(BASE + ["--survival", "S", "--nested-survival-cv", "3", "--nested-survival-cv-repeats",
                                       "2", "--seed", "9"])
    lines = []
    res = ns.nested_survival_cv(x, y, t, e, None, None, genes, args, ["g2", "g5"], random_c=[0.5, 0.9, np.nan],
                                fold=fold, log=lines.append)
    assert len(seen) == 6 and len(calls) == 7 and len(ranked) == 7
    xu = x[used].astype(np.float64)
    assert calls[0][4:6] == (2, 3) and (calls[0][6] == fold).all() and calls[0][7] == 9
    assert calls[0][0].tobytes() == xu.tobytes() and (calls[0][3][0] == [2, 5]).all()
    assert (calls[0][3][2] == [6, 7]).all()           # top_z: the first 2 of the ranking, ascending
    for j, (ex, lab) in enumerate(seen):
        k, f = divmod(j, 3)
        test = fold[k] == f
        rows = np.setdiff1d(np.arange(N), idx[test])
        assert ex.tobytes() == x[rows].tobytes() and (lab == y[rows]).all()
        assert {2, 5, 17, 23} <= set(rows)            # no record: never tested, always trained on
        assert (lab == 7).sum() == len({0, 5, 11} - set(idx[test]))          # other labels passed along
        xx, tt, ee, head, KK, FF, row, cap = calls[j + 1]
        assert (KK, FF) == (1, 2) and (row == (~test)[None, :].astype(np.int8)).all() and cap == int(test.sum())
        three = np.stack([res.biomarkers[k][f], signature.top_t(x[rows], y[rows], 2), [6, 7]])
        cols = np.unique(three)                        # only the head's genes are uploaded
        assert (cols[head] == three).all() and (tt == t[used]).all() and (ee == e[used]).all()
        assert xx.tobytes() == np.ascontiguousarray(xu[:, cols]).tobytes()
        rx, rt, re_ = ranked[j + 1]                    # top_z of the training survival samples only
        assert rx.tobytes() == xu[~test].tobytes() and (rt == t[used][~test]).all() and (re_ == e[used][~test]).all()
        assert res.n_train[k, f] == rows.shape[0] and res.n_test[k, f] == test.sum()
        assert res.n_test_events[k, f] == e[used][test].sum()
        assert (res.scores[k, test] == np.flatnonzero(test) + 100.0 * (j + 1)).all()
    assert (res.n_train + res.n_test == N).all()
    assert (res.c[3:] == 0.75).all() and res.c[0, 0, 0] == 5 / 8 and res.c[2, 1, 2] == 4 / 8
    assert np.allclose(res.c_mean, [(5 / 8 + 0.5) / 2] * 3 + [0.75] * 3, rtol=0, atol=1e-15)
    assert res.optimism == res.c_mean[3] - res.c_mean[0] and res.p_random == 2 / 4
    assert res.stop_epoch.tolist() == [[0, 1, 2], [3, 4, 5]] and res.n_windows[1, 2] == 105
    assert res.biomarkers[0][0] == [0, 1] and res.biomarkers[1][2] == [5, 6]
    assert res.selected.tolist() == [1, 2, 2, 2, 2, 2, 1, 0] and res.converged == res.n_fits == 36
    assert res.jaccard[0, 0] == 0.0 and res.jaccard[0, 2] == 1 / 3
    assert np.array_equal(res.risk[0], res.scores.mean(axis=0)) and res.group.shape == (1, n)
    assert len(lines) == 6 and lines[0] == ("nested survival CV: repeat 1/2, fold 1/3: 21 training samples, 9 test "
                                            "samples (6 events), 100 windows, stop epoch 0, 2 genes: C 0.625 (nested "
                                            "biomarkers), 0.625 (nested top |t|), 0.625 (nested top |Z|)")


# ------------------------------------------------------------------------------------ summaries and writers
def test_summaries_and_p_random_against_hand_computed_values():
    c = np.array([[[0.5, 0.7], [0.6, np.nan]], [[0.4, 0.6], [0.5, 0.5]], [[np.nan, np.nan], [np.nan, np.nan]],
                  [[0.9, 0.9], [0.8, 1.0]], [[0.7, 0.9], [0.8, 0.8]], [[0.6, 0.6], [0.6, 0.6]]])
    m, sd, opt, pr = ns.summarise(c, random_c=[0.5, 0.6, 0.7, np.nan])
    assert np.allclose(m[[0, 1, 3, 4, 5]], [0.6, 0.5, 0.9, 0.8, 0.6], rtol=0, atol=1e-15) and math.isnan(m[2])
    # per-repeat means of nested_biomarkers: 0.6 and 0.6 (the NaN fold left out) -> SD 0
    assert abs(sd[0]) < 1e-15 and abs(sd[3] - 0.0) < 1e-15 and abs(sd[1] - 0.0) < 1e-15
    assert opt == m[3] - m[0] and pr == (1 + 2) / 5.0                  # 0.6 and 0.7 >= 0.6; NaN never counts
    one = ns.summarise(c[:, :1])
    assert np.isnan(one[1]).all() and math.isnan(one[3])


def _result():
    K, F, n = 1, 2, 4
    c = np.array([[[0.75, 0.5]], [[0.625, 0.5]], [[0.5, np.nan]], [[0.875, 1.0]], [[0.75, 0.875]], [[0.5, 0.5]]])
    m, sd, opt, pr = ns.summarise(c, random_c=[0.5, 0.7, 0.2])
    sel = np.array([2, 1, 0, 1])
    return NestedSurvivalResult(
        folds=np.array([[0, 1, 0, 1]], np.int8), n_train=np.array([[20, 21]]), n_test=np.array([[3, 2]]),
        n_test_events=np.array([[2, 1]]), n_windows=np.array([[300, 310]]), stop_epoch=np.array([[4, -1]]),
        biomarkers=[[[0, 1], [0, 3]]], counts=np.zeros((6, K, F, 3), np.int64), c=c,
        jaccard=np.array([[1.0, 1 / 3]]), selected=sel, selected_good=np.array([1, 1, 0, 0]),
        selected_poor=np.array([1, 0, 0, 1]), frequency=sel / 2.0, c_mean=m, c_sd=sd, optimism=opt, p_random=pr,
        converged=11, n_fits=12, scores=np.zeros((K, n)), risk=np.array([[0.5, -0.25, 1.0, -1.0]]),
        group=np.array([[1, 0, 1, 0]], np.int8), logrank_z=np.array([2.5]), logrank_p=np.array([0.0124]),
        hr=np.array([2.0]), hr_low=np.array([1.1]), hr_high=np.array([3.6]))


def test_writers_and_summary_line(tmp_path):
    r = _result()
    genes = np.array(["A", "B", "C", "D"])
    line = ns.summary(r)
    assert line == ("nested survival CV: 2-fold x 1 repeats, 2.0 genes per fit: C 0.625 (nested biomarkers), 0.562 "
                    "(nested top |t|), 0.500 (nested top |Z|), 0.938 (biomarkers), 0.812 (top |t|), 0.500 (top |Z|); "
                    "optimism 0.312; mean Jaccard with the biomarkers 0.667; nested risk groups: log-rank Z = 2.5000, "
                    "P = 0.0124, HR 2.000 (1.100, 3.600); P_random 0.5; 1 of 12 fits did not converge")
    assert ns.summary(r._replace(p_random=float("nan"), converged=12)).endswith("HR 2.000 (1.100, 3.600)")
    prefix = str(tmp_path / "x")
    cli.write_nested_survival_cv(prefix, genes, r)
    assert open(prefix + "_nested_survival_cv.txt").read() == (
        "Repeat\tFold\tN_train\tN_test\tN_test_events\tN_windows\tStop_epoch\tSize\tC_nested\tC_nested_top_t\t"
        "C_nested_top_z\tC_biomarkers\tC_top_t\tC_top_z\tJaccard\tBiomarkers\n"
        "1\t1\t20\t3\t2\t300\t4\t2\t0.750000\t0.625000\t0.500000\t0.875000\t0.750000\t0.500000\t1.000000\tA,B\n"
        "1\t2\t21\t2\t1\t310\t-1\t2\t0.500000\t0.500000\tnan\t1.000000\t0.875000\t0.500000\t0.333333\tA,D\n"
        + line + "\n")
    cli.write_risk(prefix, ["S0", "S1", "S2", "S3"], [1.5, 2.0, 30.25, 4.0], [1, 0, 1, 1], r,
                   suffix="_nested_survival_risk.txt")
    assert open(prefix + "_nested_survival_risk.txt").read() == (
        "SAMPLE\tTIME\tEVENT\tRISK\tGROUP\nS0\t1.5\t1\t0.500000\t1\nS1\t2\t0\t-0.250000\t0\n"
        "S2\t30.25\t1\t1.000000\t1\nS3\t4\t1\t-1.000000\t0\n")
    cli.write_nested_selection(prefix, genes, np.array([0, 1, 2, 1]), r, ["A", "B"],
                               suffix="_nested_survival_selection.txt")
    assert open(prefix + "_nested_survival_selection.txt").read() == (
        "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tBiomarker\tSelected\tFrequency\tSelectedGood\tSelectedPoor\n"
        "A\t0\t1\t2\t1.000000\t1\t1\nB\t1\t1\t1\t0.500000\t1\t0\nC\t2\t0\t0\t0.000000\t0\t0\n"
        "D\t1\t0\t1\t0.500000\t0\t1\n")


def test_shared_writers_keep_their_file_names_by_default(tmp_path):
    r = _result()
    genes = np.array(["A", "B", "C", "D"])
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    cli.write_risk(a, ["S0", "S1", "S2", "S3"], [1.5, 2.0, 30.25, 4.0], [1, 0, 1, 1], r)
    cli.write_risk(b, ["S0", "S1", "S2", "S3"], [1.5, 2.0, 30.25, 4.0], [1, 0, 1, 1], r,
                   suffix="_nested_survival_risk.txt")
    assert open(a + "_risk.txt", "rb").read() == open(b + "_nested_survival_risk.txt", "rb").read()
    cli.write_nested_selection(a, genes, np.array([0, 1, 2, 1]), r, ["A"])
    cli.write_nested_selection(b, genes, np.array([0, 1, 2, 1]), r, ["A"], suffix="_nested_survival_selection.txt")
    assert open(a + "_nested_selection.txt", "rb").read() == open(b + "_nested_survival_selection.txt", "rb").read()
    import os
    assert sorted(os.listdir(str(tmp_path))) == ["a_nested_selection.txt", "a_risk.txt",
                                                 "b_nested_survival_risk.txt", "b_nested_survival_selection.txt"]
