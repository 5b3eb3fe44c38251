"""CPU checks of the nested cross-validation (g2vec_b200/nested.py; DESIGN.md §4.34): the options and every refusal
(each before any device use), the two-fold row, the selection counts, Jaccard, the summaries and P_random against
hand-computed values, the loop's bookkeeping with the device steps replaced, and the writers' exact formats."""
import numpy as np
import pytest

from g2vec_b200 import cli, nested, pipeline, signature
from g2vec_b200.nested import NestedResult
from tests.test_perm_host import cohort

BASE = ["E", "C", "N", "R"]


# ------------------------------------------------------------------------------------------- options, refusals
def test_nested_options():
    a = cli.parse_arguments(BASE)
    assert (a.nested_cv, a.nested_cv_repeats) == (0, 1)
    a = cli.parse_arguments(BASE + ["--nested-cv", "100", "--nested-cv-repeats", "100", "-n", "64"])
    assert (a.nested_cv, a.nested_cv_repeats) == (100, 100)
    assert cli.parse_arguments(BASE + ["--nested-cv", "2"]).nested_cv == 2
    for bad in (["--nested-cv", "1"], ["--nested-cv", "101"], ["--nested-cv", "-1"], ["--nested-cv-repeats", "0"],
                ["--nested-cv-repeats", "101"], ["--nested-cv", "5", "-n", "65"]):
        with pytest.raises(SystemExit):
            cli.parse_arguments(BASE + bad)
    assert cli.parse_arguments(BASE + ["-n", "65"]).numBiomarker == 65


def _no_device(monkeypatch):
    from g2vec_b200 import _capi

    def boom(*a, **k):
        raise AssertionError("the device was used")
    monkeypatch.setattr(_capi, "load", boom)
    monkeypatch.setattr(cli, "_distributed", boom)
    monkeypatch.setattr(pipeline, "walk_windows", boom)


def test_command_line_refuses_too_many_folds_before_the_device(tmp_path, capsys, monkeypatch):
    from tests import helpers
    ef, cf, nf, _ = helpers.write_ex_tsv(tmp_path)
    monkeypatch.setattr(pipeline, "walk_windows", lambda *a, **k: (_ for _ in ()).throw(AssertionError("step 3")))
    with pytest.raises(SystemExit) as e:
        cli.main([ef, cf, nf, str(tmp_path / "r"), "--nested-cv", "59"])       # 77 good, 58 poor samples
    assert e.value.code == 1
    out = capsys.readouterr().out
    assert "ERROR: --nested-cv: F = 59 folds need at least F samples of each label, got 77 and 58" in out
    assert ">>> 3." not in out


def test_command_line_refuses_torchrun_before_the_device(tmp_path, capsys, monkeypatch):
    _no_device(monkeypatch)
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(SystemExit) as e:
        cli.main([str(tmp_path / n) for n in ("E", "C", "N", "R")] + ["--nested-cv", "3"])
    assert e.value.code == 1
    out = capsys.readouterr().out
    assert out.startswith("ERROR: --nested-cv: the nested loop runs on one GPU") and ">>> 0." not in out


def test_check_inputs_refuses_before_anything_is_uploaded(monkeypatch):
    _no_device(monkeypatch)
    x, y = cohort(30, 20, 1, 10)
    xx, lab, used = nested.check_inputs(x, y, 10, 3, p=20)
    assert xx.dtype == np.float64 and used.all() and (lab == y).all()
    for F, K, p in ((1, 1, 5), (101, 1, 5), (11, 1, 5), (2.5, 1, 5), (3, 0, 5), (3, 101, 5), (3, 1, 0), (3, 1, 129)):
        with pytest.raises(ValueError):
            nested.check_inputs(x, y, F, K, p=p)
    with pytest.raises(ValueError, match="both labels"):
        nested.check_inputs(x, np.zeros(30, int), 2, 1)
    xn = x.copy(); xn[0, 0] = np.inf
    with pytest.raises(ValueError, match="finite"):
        nested.check_inputs(xn, y, 2, 1)
    y3 = y.copy(); y3[:4] = 2                         # samples of other labels are left out
    xx, lab, used = nested.check_inputs(x, y3, 2, 1)
    assert xx.shape[0] == 26 and not used[:4].any() and used[4:].all()


# ---------------------------------------------------------------------------------------------- host helpers
def test_two_fold_row_from_a_k_by_f_fold_array():
    fold = np.array([[0, 1, 2, 0, 1, 2], [2, 2, 1, 1, 0, 0]], np.int8)
    assert nested.two_fold_row(fold, 0, 0).tolist() == [[0, 1, 1, 0, 1, 1]]
    assert nested.two_fold_row(fold, 1, 2).tolist() == [[0, 0, 1, 1, 1, 1]]
    assert nested.two_fold_row(fold, 1, 0).dtype == np.int8 and nested.two_fold_row(fold, 1, 0).shape == (1, 6)


def test_selection_counts_frequency_and_jaccard():
    lg = [np.array([0, 1, 2, 0, 1, 2]), np.array([1, 1, 0, 0, 2, 2]), np.array([0, 0, 1, 1, 2, 2])]
    lists = [[0, 1, 3], [0, 2], [0, 1, 2, 3]]
    sel, good, poor = nested.selection_counts(lists, lg, 6)
    assert sel.tolist() == [3, 2, 2, 2, 0, 0]
    assert good.tolist() == [2, 1, 1, 1, 0, 0] and poor.tolist() == [1, 1, 1, 1, 0, 0]
    assert nested.jaccard([0, 1, 3], [1, 3, 4, 5]) == 2 / 5 and nested.jaccard([], []) == 1.0
    assert nested.jaccard([2], [1]) == 0.0


def test_summaries_and_p_random_against_hand_computed_values():
    auc = np.array([[[0.5, 0.7], [0.6, 0.8]], [[0.4, 0.6], [0.5, 0.5]], [[0.9, 0.9], [0.8, 1.0]],
                    [[0.7, 0.9], [0.8, 0.8]]])
    acc = auc - 0.1
    m, sd, am, opt, pr = nested.summarise(auc, acc, random_auc=[0.5, 0.65, 0.7, 0.2])
    assert np.allclose(m, [0.65, 0.5, 0.9, 0.8], rtol=0, atol=1e-15) and np.allclose(am, m - 0.1, atol=1e-15)
    # per-repeat means of nested_biomarkers: 0.6, 0.7 -> SD (ddof 1) = 0.1 / sqrt 2
    assert abs(sd[0] - 0.1 / np.sqrt(2)) < 1e-15 and abs(sd[3] - 0.0) < 1e-15
    assert opt == m[2] - m[0] and pr == (1 + 2) / 5.0              # 0.65 and 0.7 >= 0.65
    one = nested.summarise(auc[:, :1], acc[:, :1])
    assert np.isnan(one[1]).all() and np.isnan(one[4])


def _result():
    K, F = 1, 2
    auc = np.array([[[0.75, 0.5]], [[0.625, 0.5]], [[0.875, 1.0]], [[0.75, 0.875]]])
    acc = np.full((4, K, F), 0.5)
    m, sd, am, opt, pr = nested.summarise(auc, acc, random_auc=[0.5, 0.7, 0.2])
    sel = np.array([2, 1, 0, 1])
    return NestedResult(folds=np.array([[0, 1, 0, 1]], np.int8), n_train=np.array([[20, 21]]),
                        n_test=np.array([[21, 20]]), n_windows=np.array([[300, 310]]), stop_epoch=np.array([[4, -1]]),
                        biomarkers=[[[0, 1], [0, 3]]], auc=auc, acc=acc, jaccard=np.array([[1.0, 1 / 3]]),
                        selected=sel, selected_good=np.array([1, 1, 0, 0]), selected_poor=np.array([1, 0, 0, 1]),
                        frequency=sel / 2.0, auc_mean=m, auc_sd=sd, acc_mean=am, optimism=opt, p_random=pr,
                        converged=7, n_fits=8)


def test_writers_and_summary_line(tmp_path):
    r = _result()
    genes = np.array(["A", "B", "C", "D"])
    line = nested.summary(r)
    assert line == ("nested CV: 2-fold x 1 repeats, 2.0 genes per fit: AUC 0.625 (nested biomarkers), 0.562 (nested "
                    "top |t|), 0.938 (biomarkers), 0.812 (top |t|); optimism 0.312; mean Jaccard with the biomarkers "
                    "0.667; P_random 0.5; 1 of 8 fits did not converge")
    cli.write_nested_cv(str(tmp_path / "x"), genes, r)
    rows = open(str(tmp_path / "x_nested_cv.txt")).read().splitlines()
    assert rows == ["Repeat\tFold\tN_train\tN_test\tN_windows\tStop_epoch\tSize\tAUC_nested\tACC_nested\t"
                    "AUC_nested_top_t\tACC_nested_top_t\tAUC_biomarkers\tAUC_top_t\tJaccard\tBiomarkers",
                    "1\t1\t20\t21\t300\t4\t2\t0.750000\t0.500000\t0.625000\t0.500000\t0.875000\t0.750000\t1.000000\tA,B",
                    "1\t2\t21\t20\t310\t-1\t2\t0.500000\t0.500000\t0.500000\t0.500000\t1.000000\t0.875000\t0.333333\tA,D",
                    line]
    cli.write_nested_selection(str(tmp_path / "x"), genes, np.array([0, 1, 2, 1]), r, ["A", "B"])
    rows = open(str(tmp_path / "x_nested_selection.txt")).read().splitlines()
    assert rows == ["GeneSymbol\tLgroup(0:good,1:poor,2:other)\tBiomarker\tSelected\tFrequency\tSelectedGood\t"
                    "SelectedPoor",
                    "A\t0\t1\t2\t1.000000\t1\t1", "B\t1\t1\t1\t0.500000\t1\t0", "C\t2\t0\t0\t0.000000\t0\t0",
                    "D\t1\t0\t1\t0.500000\t0\t1"]
    r2 = r._replace(p_random=float("nan"), converged=8)
    assert nested.summary(r2).endswith("mean Jaccard with the biomarkers 0.667")


# ------------------------------------------------------------------------------- the loop, device steps replaced
def test_loop_passes_only_training_samples_and_counts_what_it_gets(monkeypatch):
    """pipeline.select and signature.cv_fits replaced by host fakes: the loop must hand select the training samples
    of each outer fit only (labels of other values dropped), score each fit's list on its own two-fold row, and count
    what the fakes return."""
    rs = np.random.RandomState(3)
    x = rs.standard_normal((24, 8)).astype(np.float32)
    y = np.array([0, 1] * 12); y[[0, 5]] = 7
    genes = np.array(["g%d" % i for i in range(8)])
    fold = np.array([[0, 1, 2] * 7 + [0], [2, 1, 0] * 7 + [2]], np.int8)[:, :22]
    used = np.flatnonzero(y != 7)
    seen = []

    def fake_select(expr, label, src, dst, gg, args, log=None):
        seen.append((expr.copy(), label.copy()))
        k = len(seen) - 1
        lg = np.array([0, 1, 2, 0, 1, 2, 0, 1])
        return pipeline.Selection(vectors=None, lgroup=lg, biomarkers=[gg[k % 8], gg[(k + 1) % 8]], gene_freq={},
                                  n_windows=100 + k, info={"best_step": k}, kmeans=None)

    calls = []

    def fake_cv_fits(xx, lab, head, R, K, F, seed, fold=None, cap=None, max_chunk_bytes=None):
        calls.append((head.copy(), K, F, None if fold is None else fold.copy(), cap))
        auc = np.full((head.shape[0], K, F), 0.25 * len(calls)); acc = auc / 2
        return head, fold, auc, acc, None, np.ones(auc.shape, np.uint8), None
    monkeypatch.setattr(pipeline, "select", fake_select)
    monkeypatch.setattr(signature, "cv_fits", fake_cv_fits)
    args = cli.parse_arguments(BASE + ["--nested-cv", "3", "--nested-cv-repeats", "2", "--seed", "9"])
    res = nested.nested_cv(x, y, None, None, genes, args, ["g2", "g5"], fold=fold)
    assert len(seen) == 6 and len(calls) == 7
    for j, (e, lab) in enumerate(seen):
        k, f = divmod(j, 3)
        rows = used[fold[k] != f]
        assert e.tobytes() == x[rows].tobytes() and (lab == y[rows]).all() and (lab != 7).all()
        head, K, F, row, cap = calls[j + 1]
        assert (K, F) == (1, 2) and (row == nested.two_fold_row(fold, k, f)).all() and cap == int((fold[k] == f).sum())
    assert calls[0][1:3] == (2, 3) and calls[0][4] == 8 and (calls[0][3] == fold).all()
    assert (res.auc[2:] == 0.25).all() and res.auc[0, 1, 2] == 0.25 * 7 and res.n_windows[1, 2] == 105
    assert res.stop_epoch.tolist() == [[0, 1, 2], [3, 4, 5]] and (res.n_train + res.n_test == 22).all()
    assert res.biomarkers[0][0] == [0, 1] and res.biomarkers[1][2] == [5, 6]
    assert res.selected.tolist() == [1, 2, 2, 2, 2, 2, 1, 0] and res.converged == res.n_fits == 24
    assert res.jaccard[0, 0] == 0.0 and res.jaccard[0, 2] == 1 / 3        # {g0, g1} and {g2, g3} against {g2, g5}
