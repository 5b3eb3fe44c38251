"""Nested cross-validation of the selection on the H100 (g2vec_b200/nested.py, g2vec_b200/pipeline.py; DESIGN.md
§4.34): one implementation of steps 3-6, no leakage of the test fold, the two-fold-row scoring against a K x F call,
the comparison rows against signature_cv, a null and a planted cohort, and the command line.

The null cohort's bounds come from a host run of the top_t half (signature.top_t on the training samples, scikit-learn's
LogisticRegression(C=1) on the same stratified folds) over the seeds 0..199 of tests/nested_cohorts.module_cohort at
K = 3, F = 3, p = 20: the non-nested top_t AUC had mean 0.697, SD 0.045 and minimum 0.543; the nested top_t AUC mean
0.499, SD 0.057 and largest distance from 1/2 0.151.  The bounds below, top_t > 0.55 and |nested - 1/2| < 0.2, are
3.3 and 3.5 SDs out."""
import os

import numpy as np
import pytest

from g2vec_b200 import cli, nested, pipeline, signature
from tests import nested_cohorts as nc

pytestmark = pytest.mark.gpu


def _args(*extra):
    return cli.parse_arguments(["E", "C", "N", "R"] + list(extra))


def _run_cohort(seed, planted, extra, random_rows=0):
    x, y, genes, (src, dst) = nc.module_cohort(seed, planted=planted)
    args = _args(*extra)
    full = pipeline.select(x, y, src, dst, genes, args)
    pos = {g: i for i, g in enumerate(genes)}
    sig = None
    if random_rows:
        sig = signature.signature_cv(x, y, np.array([pos[g] for g in full.biomarkers]), random_rows,
                                     folds=args.nested_cv, repeats=args.nested_cv_repeats, seed=args.seed)
    res = nested.nested_cv(x, y, src, dst, genes, args, full.biomarkers,
                           random_auc=None if sig is None else sig.auc_mean[2:])
    return x, y, genes, full, res, sig


# ------------------------------------------------------------------------------------------ one selection rule
def test_selection_functions_write_the_files_of_the_command_line(tmp_path, capsys):
    from tests import helpers
    ef, cf, nf, _ = helpers.write_ex_tsv(tmp_path)
    base = ["-r", "2", "-e", "5", "--seed", "3", "--deterministic"]
    a = str(tmp_path / "main")
    cli.main([ef, cf, nf, a] + base)
    capsys.readouterr()
    data = cli.load_data(ef)
    data["label"] = cli.match_labels(cli.load_clinical(cf), data["sample"])
    data, network = cli.restrict(data, cli.load_network(nf))
    src, dst = pipeline.edge_arrays(data["gene"], network["edge"])
    sel = pipeline.select(data["expr"], data["label"], src, dst, data["gene"], cli.parse_arguments([ef, cf, nf, a] + base))
    b = str(tmp_path / "fn")
    cli.write_biomarkers(b, sel.biomarkers)
    cli.write_lgroups(b, sel.lgroup, data["gene"])
    cli.write_vectors(b, data["gene"], sel.vectors)
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt"):
        assert open(a + suffix, "rb").read() == open(b + suffix, "rb").read(), suffix
    assert capsys.readouterr().out == ""                       # select is silent without a log
    assert sel.n_windows > 0 and sel.info["best_step"] is not None and sel.kmeans is None


# ---------------------------------------------------------------------------------------------- no leakage
def test_the_test_fold_reaches_neither_the_selection_nor_the_fit():
    x, y, genes, (src, dst) = nc.module_cohort(5, planted=True)
    args = _args("-r", "2", "-e", "30", "-n", "10", "--seed", "1", "--deterministic", "--nested-cv", "3")
    full = pipeline.select(x, y, src, dst, genes, args)
    kept = {}
    a = nested.nested_cv(x, y, src, dst, genes, args, full.biomarkers,
                         on_fit=lambda k, f, s: kept.setdefault(("a", k, f), s))
    test = a.folds[0] == 0
    rs = np.random.RandomState(99)
    x2, y2 = x.copy(), y.copy()
    x2[test] = rs.standard_normal((int(test.sum()), x.shape[1])).astype(np.float32) * 3.0 + 1.0
    y2[test] = 1 - y2[test]
    b = nested.nested_cv(x2, y2, src, dst, genes, args, full.biomarkers, fold=a.folds,
                         on_fit=lambda k, f, s: kept.setdefault(("b", k, f), s))
    sa, sb = kept[("a", 0, 0)], kept[("b", 0, 0)]
    assert sa.vectors.dtype == np.float32 and sa.vectors.tobytes() == sb.vectors.tobytes()
    assert (sa.lgroup == sb.lgroup).all() and sa.biomarkers == sb.biomarkers and sa.n_windows == sb.n_windows
    assert a.biomarkers[0][0] == b.biomarkers[0][0]
    for field in ("n_train", "n_test", "n_windows", "stop_epoch", "jaccard"):
        assert getattr(a, field)[0, 0] == getattr(b, field)[0, 0], field
    assert a.auc[0, 0, 0] != b.auc[0, 0, 0] and a.auc[1, 0, 0] != b.auc[1, 0, 0]
    assert a.acc[0, 0, 0] != b.acc[0, 0, 0]


# ------------------------------------------------------------------------------------------------- scoring
def _ex():
    from tests.helpers import GOLDEN
    e = np.load(os.path.join(GOLDEN, "ex_expr.npz"))
    lab = np.load(os.path.join(GOLDEN, "ex_graph.npz"))["label"]
    used = (lab == 0) | (lab == 1)
    return e["expr"][used].astype(np.float64), lab[used]


def test_two_fold_row_gives_the_bits_of_fit_k_f_of_a_k_by_f_call():
    from tests.test_gpu_signature import gpu_fit, gpu_folds
    x, y = _ex()
    K, F, seed = 3, 4, 5
    folds = gpu_folds(y, K, F, seed)
    for k in range(K):                                # repeat k's split depends on (labels, F, seed, k) only
        assert (gpu_folds(y, 1 + k, F, seed)[k] == folds[k]).all() and (gpu_folds(y, 6, F, seed)[:K] == folds).all()
    genes = np.stack([np.arange(0, 7000, 100), signature.top_t(x, y, 70)]).astype(np.int32)
    sc, _, _, _, auc, acc = gpu_fit(x, y, genes, folds)
    for k, f in ((0, 0), (1, 3), (2, 1)):
        row = nested.two_fold_row(folds, k, f)
        test = row[0] == 0
        sc2, _, _, _, auc2, acc2 = gpu_fit(x, y, genes, row)
        assert sc2[:, 0, test].tobytes() == sc[:, k, test].tobytes()
        assert auc2[:, 0, 0].tobytes() == auc[:, k, f].tobytes() and acc2[:, 0, 0].tobytes() == acc[:, k, f].tobytes()
        a, c, conv = nested.score_fit(x, y, folds, k, f, genes, seed=seed)      # only the head's genes uploaded
        assert a.tobytes() == auc[:, k, f].tobytes() and c.tobytes() == acc[:, k, f].tobytes() and conv.all()


# ---------------------------------------------------------------------------------------- null and planted
def test_null_cohort_nested_aucs_are_one_half_and_comparison_rows_are_signature_cvs():
    extra = ("-r", "2", "-e", "100", "-n", "10", "--seed", "2", "--deterministic", "--nested-cv", "3",
             "--nested-cv-repeats", "3")
    x, y, genes, full, res, sig = _run_cohort(7, False, extra, random_rows=50)
    assert res.auc_mean[3] > 0.55                                   # top_t chosen with every label: optimistic
    assert abs(res.auc_mean[0] - 0.5) < 0.2 and abs(res.auc_mean[1] - 0.5) < 0.2
    assert res.auc[2:].tobytes() == sig.auc[:2].tobytes() and res.acc[2:].tobytes() == sig.acc[:2].tobytes()
    assert (res.folds == sig.folds).all()
    rnd = sig.auc_mean[2:]
    assert res.p_random == (1.0 + (rnd >= res.auc_mean[0]).sum()) / 51.0
    assert res.optimism == res.auc_mean[2] - res.auc_mean[0]
    sizes = sum(len(b) for row in res.biomarkers for b in row)
    assert res.selected.sum() == sizes and (res.selected == res.selected_good + res.selected_poor).all()
    assert (res.frequency == res.selected / 9.0).all() and res.converged == res.n_fits == 36
    assert (res.n_train + res.n_test == 120).all()


def test_planted_module_is_predicted_and_selected_far_above_chance():
    """G2Vec's L-groups on a 400-gene cohort move between outer fits (genes in the L-group named "other" are never
    selected), so a planted gene is not selected in every fit; the module is selected far more often than the rest."""
    extra = ("-r", "10", "-e", "100", "-n", "10", "--seed", "4", "--deterministic", "--nested-cv", "5")
    x, y, genes, full, res, _ = _run_cohort(3, True, extra)
    assert res.auc_mean[0] > 0.85, res.auc_mean
    rest = np.setdiff1d(np.arange(len(genes)), nc.PLANTED)
    freq = res.frequency[nc.PLANTED]
    assert (freq >= 0.4).all() and freq.mean() > 5 * res.frequency[rest].mean(), freq


# ------------------------------------------------------------------------------------------------------- CLI
def test_command_line_writes_both_files_and_leaves_the_other_files_alone(tmp_path, capsys):
    from tests import helpers
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    base = ["-r", "2", "-e", "5", "--deterministic"]
    a, b, c = (str(tmp_path / n) for n in ("plain", "nested", "again"))
    cli.main([ef, cf, nf, a] + base)
    log_a = capsys.readouterr().out
    cli.main([ef, cf, nf, b] + base + ["--nested-cv", "3"])
    log_b = capsys.readouterr().out
    cli.main([ef, cf, nf, c] + base + ["--nested-cv", "3"])
    capsys.readouterr()
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt"):
        assert open(a + suffix, "rb").read() == open(b + suffix, "rb").read(), suffix
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt", "_nested_cv.txt", "_nested_selection.txt"):
        assert open(b + suffix, "rb").read() == open(c + suffix, "rb").read(), suffix
    assert not os.path.exists(a + "_nested_cv.txt")
    import re
    untimed = lambda log, prefix: [re.sub(r" \([0-9.]+ sec\)$", "", l).replace(prefix, "RES")
                                   for l in log.splitlines()]
    extra = [l for l in untimed(log_b, b) if l not in untimed(log_a, a)]
    assert len(extra) == 7 and extra[0].startswith("Namespace(") and "nested_cv=3" in extra[0]
    assert all(extra[1 + j].startswith("    nested CV: repeat 1/1, fold %d/3: " % (j + 1)) for j in range(3))
    assert extra[4].startswith("    nested CV: 3-fold x 1 repeats, ")
    assert extra[5:] == ["    RES_nested_cv.txt", "    RES_nested_selection.txt"]
    rows = open(b + "_nested_cv.txt").read().splitlines()
    assert rows[0].split("\t") == ["Repeat", "Fold", "N_train", "N_test", "N_windows", "Stop_epoch", "Size",
                                   "AUC_nested", "ACC_nested", "AUC_nested_top_t", "ACC_nested_top_t",
                                   "AUC_biomarkers", "AUC_top_t", "Jaccard", "Biomarkers"]
    assert len(rows) == 5 and rows[4] == extra[4].strip()
    gset = set(genes)
    for j, r in enumerate(rows[1:4]):
        col = r.split("\t")
        assert len(col) == 15 and col[:2] == ["1", str(j + 1)] and int(col[2]) + int(col[3]) == 135
        bm = col[14].split(",")
        assert int(col[6]) == len(bm) <= 100 and set(bm) <= gset and bm == sorted(bm)
        assert all(0.0 <= float(v) <= 1.0 for v in col[7:14])
    sel = open(b + "_nested_selection.txt").read().splitlines()
    lg = open(b + "_lgroups.txt").read().splitlines()
    assert sel[0] == ("GeneSymbol\tLgroup(0:good,1:poor,2:other)\tBiomarker\tSelected\tFrequency\tSelectedGood\t"
                      "SelectedPoor")
    assert len(sel) == len(lg) and [s.split("\t")[:2] for s in sel[1:]] == [s.split("\t") for s in lg[1:]]
    counts = np.array([[int(v) for v in (s.split("\t")[3], s.split("\t")[5], s.split("\t")[6])] for s in sel[1:]])
    assert (counts[:, 0] == counts[:, 1] + counts[:, 2]).all()
    assert counts[:, 0].sum() == sum(int(r.split("\t")[6]) for r in rows[1:4])
