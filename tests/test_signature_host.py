"""CPU checks of the signature test (DESIGN.md §4.29): the oracle against scikit-learn's pipeline and roc_auc_score,
the stratified folds, Floyd's draws, the constant-gene rule, every refusal (raised before the library is loaded), the
options, the writer and the summary line."""
import os

import numpy as np
import pytest

from g2vec_b200 import cli, signature
from g2vec_b200.signature import SignatureResult, check_inputs, summarise, summary
from tests import signature_oracle as so
from tests.test_perm_host import cohort


def _ex():
    from tests.helpers import GOLDEN
    e = np.load(os.path.join(GOLDEN, "ex_expr.npz"))
    lab = np.load(os.path.join(GOLDEN, "ex_graph.npz"))["label"]
    used = (lab == 0) | (lab == 1)
    return e["expr"][used].astype(np.float64), lab[used]


def _sklearn_fit(xtr, ytr):
    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler
    return make_pipeline(StandardScaler(), LogisticRegression(C=1.0, tol=1e-12, max_iter=10000)).fit(xtr, ytr)


# ------------------------------------------------------------------------------------------- oracle vs sklearn
@pytest.mark.parametrize("which", ["seeded", "ex"])
def test_oracle_fits_equal_scikit_learns_pipeline(which):
    from sklearn.metrics import roc_auc_score
    if which == "seeded":
        x, y = cohort(90, 40, 3)
        x[:, :4] += 0.8 * y[:, None]
        genes = np.array([[0, 1, 2, 3, 10, 20, 30], [5, 6, 7, 8, 9, 11, 12]])
    else:
        x, y = _ex()
        genes = np.array([np.arange(0, 7523, 301)[:20], np.arange(7, 7523, 377)[:20]])
    fold = so.folds(y, 2, 5, 4)
    want = so.cv(x, y, genes, fold)
    assert want["converged"].all()
    for s in range(genes.shape[0]):
        for k in range(2):
            for f in range(5):
                te = fold[k] == f
                m = _sklearn_fit(x[~te][:, genes[s]], y[~te])
                lr = m[-1]
                b = want["beta"][s, k, f]
                assert abs(lr.intercept_[0] - b[0]) <= 1e-6 and np.abs(lr.coef_[0] - b[1:]).max() <= 1e-6
                d = m.decision_function(x[te][:, genes[s]])
                eta = want["scores"][s, k, te]
                assert np.abs(d - eta).max() <= 1e-5            # coefficient errors of 1e-6 times |z|
                gap = np.abs(eta[y[te] == 1][:, None] - eta[y[te] == 0][None, :]).min()
                if gap > 1e-6:                          # no near-tie the two fits could order differently
                    assert want["auc"][s, k, f] == pytest.approx(roc_auc_score(y[te], d), abs=1e-15)


def test_oracle_auc_is_roc_auc_score_with_ties():
    from sklearn.metrics import roc_auc_score
    rs = np.random.RandomState(0)
    for _ in range(50):
        m = int(rs.randint(2, 40))
        y = rs.randint(0, 2, m)
        y[:2] = (0, 1)
        s = rs.randint(-3, 4, m).astype(np.float64)     # many ties
        assert so.auc_counts(s, y) == pytest.approx(roc_auc_score(y, s), abs=1e-15)
        assert so.accuracy(s, y) == np.mean((s > 0) == (y == 1))


def test_constant_gene_is_z_zero_and_leaves_the_fit_of_the_others():
    x, y = cohort(60, 6, 2)
    x[:, 3] = 4.25
    fold = so.folds(y, 1, 3, 0)
    a = so.cv(x, y, np.array([[0, 1, 3]]), fold)
    b = so.cv(x, y, np.array([[0, 1]]), fold)
    assert (a["beta"][..., 3] == 0).all()
    assert np.abs(a["beta"][..., :3] - b["beta"]).max() <= 1e-12
    mu, sd = so.standardise(x[:, [3, 0]])
    assert mu[0] == 4.25 and sd[0] == 1.0


# ---------------------------------------------------------------------------------------------- folds, draws
@pytest.mark.parametrize("F", [2, 3, 5, 10])
def test_folds_are_stratified(F):
    for m0, m1 in ((F, F), (F + 1, 2 * F - 1), (5 * F + 3, 3 * F)):
        y = np.array([0] * m0 + [1] * m1)
        np.random.RandomState(m0).shuffle(y)
        fold = so.folds(y, 4, F, 9)
        for k in range(4):
            for c, m in ((0, m0), (1, m1)):
                sizes = np.bincount(fold[k][y == c], minlength=F)
                assert sizes.max() - sizes.min() <= 1 and sizes.sum() == m and sizes.min() >= 1
        assert not (fold[0] == fold[1]).all() or m0 + m1 <= 4


def test_floyd_rows_are_distinct_sorted_and_uniform():
    from scipy import stats
    G, p, R = 40, 7, 4000
    rows = np.array([so.floyd(G, p, 13, r) for r in range(1, R + 1)])
    assert (np.diff(rows, axis=1) > 0).all() and rows.min() >= 0 and rows.max() < G
    counts = np.bincount(rows.ravel(), minlength=G)
    assert stats.chisquare(counts).pvalue > 1e-3
    assert (so.floyd(5, 5, 0, 1) == np.arange(5)).all()


def test_draw64_is_perm_oracles_stream():
    from tests import perm_oracle
    b = np.array([0, 5, 1 << 40], dtype=np.uint64)
    for s in range(4):
        want = perm_oracle.draw64(7, b, s)
        got = [so.draw64(7, (1 << 63) + int(v), s) for v in b]
        assert (np.array(got, dtype=np.uint64) == want).all()


# ------------------------------------------------------------------------------------------------- refusals
def test_check_inputs_refuses_before_anything_is_uploaded():
    x, y = cohort(30, 20, 1, 10)
    check_inputs(x, y, 5, 10, 10, 3)
    bad = [dict(n_random=0), dict(n_random=65537), dict(n_random=2.5), dict(folds=1), dict(folds=101),
           dict(folds=11), dict(repeats=0), dict(repeats=101), dict(p=0), dict(p=21), dict(p=129),
           dict(n_random=65536, folds=10, repeats=100)]
    for kw in bad:
        args = dict(p=5, n_random=10, folds=5, repeats=3)
        args.update(kw)
        with pytest.raises(ValueError, match="signature test"):
            check_inputs(x, y, args["p"], args["n_random"], args["folds"], args["repeats"])
    with pytest.raises(ValueError, match="both labels"):
        check_inputs(x, np.zeros(30, int), 5, 10, 2, 1)
    xn = x.copy(); xn[0, 0] = np.nan
    with pytest.raises(ValueError, match="finite"):
        check_inputs(xn, y, 5, 10, 2, 1)


def test_signature_cv_refuses_without_touching_the_device(monkeypatch):
    from g2vec_b200 import _capi

    def boom():
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(_capi, "load", boom)
    x, y = cohort(30, 20, 1)
    for sig, R in (([1, 1, 2], 5), ([0, 20], 5), ([-1, 2], 5), ([0.5, 2.0], 5), ([1, 2], 0), (list(range(20)) * 7, 5)):
        with pytest.raises(ValueError, match="signature test"):
            signature.signature_cv(x, y, np.array(sig), R, folds=3, repeats=2)


# ----------------------------------------------------------------------------------------------- CLI, writer
def test_signature_options():
    base = ["E", "C", "N", "R"]
    a = cli.parse_arguments(base)
    assert (a.signature_cv, a.signature_folds, a.signature_repeats) == (0, 5, 10)
    a = cli.parse_arguments(base + ["--signature-cv", "65536", "--signature-folds", "100", "--signature-repeats", "1",
                                    "-n", "64"])
    assert (a.signature_cv, a.signature_folds, a.signature_repeats) == (65536, 100, 1)
    for bad in (["--signature-cv", "-1"], ["--signature-cv", "65537"], ["--signature-folds", "1"],
                ["--signature-folds", "101"], ["--signature-repeats", "0"], ["--signature-repeats", "101"],
                ["--signature-cv", "5", "-n", "65"]):
        with pytest.raises(SystemExit):
            cli.parse_arguments(base + bad)
    assert cli.parse_arguments(base + ["-n", "65"]).numBiomarker == 65


def test_command_line_refuses_too_many_folds_before_the_gpu(tmp_path, capsys):
    from tests import helpers
    ef, cf, nf, _ = helpers.write_ex_tsv(tmp_path)
    with pytest.raises(SystemExit) as e:
        cli.main([ef, cf, nf, str(tmp_path / "r"), "--signature-cv", "5", "--signature-folds", "100"])
    assert e.value.code == 1
    out = capsys.readouterr().out
    assert "ERROR: --signature-cv: signature test: F = 100 folds need at least F samples" in out
    assert ">>> 3." not in out


def _result(R=3, K=2, F=2, p=3):
    rs = np.random.RandomState(1)
    S = R + 2
    auc = rs.uniform(0.3, 0.9, (S, K, F)); acc = rs.uniform(0.3, 0.9, (S, K, F))
    auc_mean, auc_sd, acc_mean, p_random = summarise(auc, acc, R)
    genes = np.array([[0, 1, 2], [1, 2, 3], [2, 5, 6], [0, 4, 6], [3, 4, 5]], np.int32)[:S]
    return SignatureResult(names=["biomarkers", "top_t"] + ["random_%d" % r for r in range(1, R + 1)], genes=genes,
                           folds=np.zeros((K, 4), np.int8), auc=auc, acc=acc, n_iter=np.ones((S, K, F), np.int32),
                           converged=S * K * F - 1, beta=np.zeros((2, K, F, p + 1)), auc_mean=auc_mean,
                           auc_sd=auc_sd, acc_mean=acc_mean, p_random=p_random)


def test_summarise_and_p_random():
    r = _result()
    assert (r.p_random == so.p_random(r.auc_mean, 3)).all()
    assert r.auc_mean[0] == r.auc[0].mean() and r.auc_sd[1] == np.std(r.auc[1].mean(axis=1), ddof=1)
    one = summarise(r.auc[:, :1], r.acc[:, :1], 3)
    assert np.isnan(one[1]).all()


def test_writer_and_summary(tmp_path):
    r = _result()
    genes = np.array(["G%d" % i for i in range(7)])
    cli.write_signature(str(tmp_path / "x"), genes, r, ["G0", "G2", "G6"])
    rows = open(str(tmp_path / "x_signature.txt")).read().splitlines()
    assert rows[0] == "Signature\tSize\tAUC\tAUC_SD\tAccuracy\tP_random\tBiomarkers" and len(rows) == 6
    assert rows[1] == "biomarkers\t3\t%.6f\t%.6f\t%.6f\t%.6g\t2" % (r.auc_mean[0], r.auc_sd[0], r.acc_mean[0],
                                                                    r.p_random[0])
    assert rows[2].startswith("top_t\t3\t") and rows[2].endswith("\t1")
    assert rows[3].split("\t")[5] == "nan" and rows[3].endswith("\t2")
    line = summary(r)
    lo, hi = np.percentile(r.auc_mean[2:], [2.5, 97.5])
    assert line == ("signature CV: 2-fold x 2 repeats, 3 genes: AUC %.3f (biomarkers), %.3f (top |t|), random mean "
                    "%.3f [%.3f, %.3f]; P_random %.3g / %.3g; 1 of 20 fits did not converge"
                    % (r.auc_mean[0], r.auc_mean[1], r.auc_mean[2:].mean(), lo, hi, r.p_random[0], r.p_random[1]))
