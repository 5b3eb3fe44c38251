"""Host side of the lasso path (DESIGN.md §4.37), no GPU: the float64 oracle against independent solvers, the lambda
sequence, the stop rules, top_lasso's order, the lambda_min / lambda_1se rule and check_inputs' refusals."""
import numpy as np
import pytest
from scipy.optimize import minimize

from g2vec_b200 import lasso
from tests import lasso_oracle as orc


def small(n, G, seed):
    rs = np.random.RandomState(seed)
    x = rs.randn(n, G) + rs.uniform(-1, 2, G)
    lab = (rs.rand(n) < 0.45).astype(np.float64)
    lab[:2] = [0, 1]
    x[:, :3] += 0.7 * lab[:, None]
    return x, lab


def split_solve(z, y, lam, alpha):
    """beta = b+ - b-, both >= 0, by L-BFGS-B; returns (b0, beta, objective)."""
    n, G = z.shape

    def fg(v):
        b0, bp, bm = v[0], v[1:G + 1], v[G + 1:]
        beta = bp - bm
        eta = b0 + z @ beta
        p = 1.0 / (1.0 + np.exp(-eta))
        f = np.mean(np.logaddexp(0.0, eta) - y * eta) + lam * (alpha * (bp + bm).sum()
                                                                + 0.5 * (1 - alpha) * (beta ** 2).sum())
        gs = z.T @ (p - y) / n + lam * (1 - alpha) * beta
        return f, np.concatenate([[np.mean(p - y)], gs + lam * alpha, -gs + lam * alpha])
    bounds = [(None, None)] + [(0, None)] * (2 * G)
    r = minimize(fg, np.zeros(2 * G + 1), jac=True, method="L-BFGS-B", bounds=bounds,
                 options=dict(ftol=1e-15, gtol=1e-12, maxiter=20000, maxcor=50))
    return r.x[0], r.x[1:G + 1] - r.x[G + 1:], r.fun


@pytest.mark.parametrize("alpha", [1.0, 0.5])
def test_oracle_matches_split_variable_solve_at_g_below_n(alpha):
    x, y = small(60, 8, 1)
    z, mu, sd, const = orc.standardise(x)
    lams = orc.lambdas(z, y, alpha)
    for k in (5, 20, 40):
        b0, beta = orc.solve(z, y, np.log(y.mean() / (1 - y.mean())), np.zeros(8), lams[k], alpha)
        _, beta_s, _ = split_solve(z, y, lams[k], alpha)
        np.testing.assert_allclose(beta, beta_s, atol=1e-6)
        assert orc.kkt(z, y, b0, beta, lams[k], alpha) <= 1e-9


def test_oracle_objective_matches_split_solve_p_much_greater_than_n():
    x, y = small(20, 60, 2)
    z, mu, sd, const = orc.standardise(x)
    lams = orc.lambdas(z, y, 1.0)
    for k in (10, 30):
        b0, beta = orc.solve(z, y, 0.0, np.zeros(60), lams[k], 1.0)
        _, _, f_s = split_solve(z, y, lams[k], 1.0)
        f = orc.objective(z, y, b0, beta, lams[k], 1.0)
        assert f <= f_s * (1 + 1e-9)


def test_lambda_max_gives_zero_and_certifies():
    x, y = small(40, 10, 3)
    z, mu, sd, const = orc.standardise(x)
    lam = orc.lambdas(z, y, 1.0)[0]
    b0, beta = orc.solve(z, y, np.log(y.mean() / (1 - y.mean())), np.zeros(10), lam, 1.0)
    assert not beta.any() and orc.kkt(z, y, b0, beta, lam, 1.0) <= 1e-9
    np.testing.assert_allclose(lasso.lambda_path(lam, 40, 10), orc.lambdas(z, y, 1.0), rtol=1e-15)
    assert lasso.lambda_path(1.0, 10, 40)[-1] == pytest.approx(0.01)
    assert lasso.lambda_path(1.0, 40, 10)[-1] == pytest.approx(1e-4)


def test_stop_rules():
    rs = np.random.RandomState(4)
    x = rs.randn(40, 10)
    y = (np.arange(40) % 2).astype(np.float64)
    x[:, 0] += 6.0 * y                                 # separable: the deviance rule ends the path
    fit = orc.path(x, y, 1.0)
    assert fit["L"] < 100 and fit["dev_ratio"][-1] > 0.999
    old = orc.MAX_ACTIVE
    orc.MAX_ACTIVE = 2                                 # the active cap ends the path before the third gene enters
    try:
        x2, y2 = small(40, 10, 5)
        capped = orc.path(x2, y2, 1.0)
    finally:
        orc.MAX_ACTIVE = old
    assert (capped["entry"] >= 0).sum() <= 2 and capped["L"] < 100


def test_top_lasso_order():
    entry = np.array([3, -1, 1, 3, 1, 0, 3])
    eabs = np.array([0.2, 0.0, 0.5, 0.2, 0.7, 0.1, 0.3])
    assert lasso.top_lasso(entry, eabs, 10).tolist() == [5, 4, 2, 6, 0, 3]
    assert lasso.top_lasso(entry, eabs, 3).tolist() == [5, 4, 2]


def test_lambda_min_and_1se_rule():
    cvm = np.array([1.0, 0.8, 0.62, 0.6, 0.61, 0.7])
    cvsd = np.array([0.1, 0.1, 0.05, 0.03, 0.05, 0.1])
    assert lasso.pick(cvm, cvsd) == (3, 2)
    dev = np.ones((3, 1, 6)); dev[1] *= 0.5
    fold = np.array([[0, 1, 0, 1, 0, 1]])
    cvm2, cvsd2, i_min, i_1se = lasso.cv_summary(dev, fold, 2)
    assert cvm2.tolist() == [1.0, 0.5, 1.0] and i_min == 1 and not cvsd2.any()


def unequal_folds(rs, K, F, n):
    """[K, n] folds with every fold non-empty and sizes that differ."""
    folds = np.empty((K, n), dtype=np.int8)
    for k in range(K):
        f = np.concatenate([np.arange(F), rs.randint(0, F, n - F)])
        rs.shuffle(f)
        folds[k] = f
    return folds


@pytest.mark.parametrize("L,K,F,n", [(7, 1, 2, 5), (30, 1, 5, 23), (20, 3, 4, 17), (12, 10, 10, 101)])
def test_cv_summary_matches_independent_cv_glmnet(L, K, F, n):
    rs = np.random.RandomState(L * 1000 + K * 100 + n)
    folds = unequal_folds(rs, K, F, n)
    sizes = [np.bincount(folds[k], minlength=F) for k in range(K)]
    assert all(s.min() >= 1 for s in sizes) and (K * F == 2 or len(np.unique(np.concatenate(sizes))) > 1)
    dev = rs.gamma(2.0, 0.6, (L, K, n))
    # ties in cvm: equal rows have equal cvm bit for bit, so both rules must take the first of them
    dev[3] = dev[5] = dev[:].min(axis=0)
    dev[4] = dev[3]
    got = lasso.cv_summary(dev, folds, F)
    want = orc.cv_glmnet(dev, folds, F)
    np.testing.assert_allclose(got[0], want[0], rtol=1e-13)
    np.testing.assert_allclose(got[1], want[1], rtol=1e-12)
    assert got[2:] == want[2:] == (3, want[3])
    assert want[3] <= 3 and want[0][want[3]] <= want[0][3] + want[1][3]
    assert want[3] == 0 or want[0][want[3] - 1] > want[0][3] + want[1][3]
    # cvsd at K F = 2 from its definition: two fold means, weights N_0 and N_1
    if K * F == 2:
        m = np.array([dev[:, 0, folds[0] == f].mean(axis=1) for f in range(2)])       # [2, L]
        N = np.bincount(folds[0], minlength=2).astype(np.float64)
        cvm = (N[:, None] * m).sum(axis=0) / n
        np.testing.assert_allclose(want[1], np.sqrt((N[:, None] * (m - cvm) ** 2).sum(axis=0) / n), rtol=1e-12)


def test_heldout_deviance_clamps_at_glmnet_bound():
    eta = np.array([-40.0, -3.0, 0.0, 2.5, 40.0, 11.6, -11.6])
    y = np.array([1, 0, 1, 1, 0, 1, 0])
    d = orc.heldout_deviance(eta, y)
    p = 1 / (1 + np.exp(-eta))
    assert d[0] == pytest.approx(-2 * np.log(1e-5), rel=1e-15)         # clamped from below
    # y = 0, p clamped to 1 - 1e-5: 1 - (1 - 1e-5) is 1e-5 to 7e-12 relative in float64
    assert d[4] == pytest.approx(-2 * np.log(1e-5), rel=1e-11)
    np.testing.assert_allclose(d[[1, 2, 3]], [-2 * np.log(1 - p[1]), 2 * np.log(2), -2 * np.log(p[3])], rtol=1e-14)
    assert d[5] == pytest.approx(-2 * np.log(1 - 1e-5), rel=1e-12)     # sigmoid(11.6) > 1 - 1e-5
    assert d[6] == pytest.approx(-2 * np.log(1 - 1e-5), rel=1e-12)


@pytest.mark.parametrize("kw,msg", [(dict(folds=1), "number of folds F"), (dict(folds=101), "number of folds F"),
                                    (dict(repeats=0), "number of repeats K"), (dict(repeats=101), "repeats K"),
                                    (dict(alpha=0.0), "alpha"), (dict(alpha=1.5), "alpha"),
                                    (dict(alpha=float("nan")), "alpha"), (dict(folds=30), "at least F samples")])
def test_check_inputs_refuses(kw, msg):
    x, y = small(40, 10, 6)
    args = dict(folds=5, repeats=1, alpha=1.0)
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        lasso.check_inputs(x, y.astype(np.int64), **args)


@pytest.mark.parametrize("argv,msg", [(["--lasso", "1"], "--lasso must be 0 (off) or an integer in [2, 100]"),
                                      (["--lasso", "101"], "--lasso must be 0 (off) or an integer in [2, 100]"),
                                      (["--lasso", "-1"], "--lasso must be 0 (off) or an integer in [2, 100]"),
                                      (["--lasso-repeats", "0"], "--lasso-repeats must be an integer in [1, 100]"),
                                      (["--lasso-repeats", "101"], "--lasso-repeats must be an integer in [1, 100]"),
                                      (["--lasso-alpha", "0"], "--lasso-alpha must be a finite number in (0, 1]"),
                                      (["--lasso-alpha", "1.01"], "--lasso-alpha must be a finite number in (0, 1]"),
                                      (["--lasso-alpha", "nan"], "--lasso-alpha must be a finite number in (0, 1]"),
                                      (["--lasso-alpha", "inf"], "--lasso-alpha must be a finite number in (0, 1]")])
def test_parse_arguments_refuses(argv, msg, capsys):
    from g2vec_b200 import cli
    with pytest.raises(SystemExit):
        cli.parse_arguments(["e", "c", "n", "r"] + argv)
    assert msg in capsys.readouterr().err


def test_parse_arguments_defaults():
    from g2vec_b200 import cli
    a = cli.parse_arguments(["e", "c", "n", "r"])
    assert (a.lasso, a.lasso_repeats, a.lasso_alpha) == (0, 1, 1.0)


def fake_result():
    L, G, K, F = 3, 4, 1, 2
    return lasso.LassoResult(alpha=0.5, lambdas=np.array([0.4, 0.2, 0.1]), n_lambda=L, a0=np.zeros(L),
                             beta=np.array([[0, 0, 0, 0], [0.5, 0, 0, 0], [0.75, -0.25, 0, 0]]),
                             df=np.array([0, 1, 2]), dev_ratio=np.array([0.0, 0.1, 0.25]),
                             cvm=np.array([1.4, 1.2, 1.3]), cvsd=np.array([0.1, 0.05, 0.2]),
                             auc=np.array([[[0.5, 0.5]], [[0.7, 0.8]], [[0.6, 0.7]]]), auc_mean=np.array([0.5, 0.75, 0.65]),
                             i_min=1, i_1se=1, folds=np.array([[0, 1, 0, 1]], dtype=np.int8),
                             entry=np.array([[1, 2, -1, -1], [1, -1, -1, -1], [0, 2, 1, -1]], dtype=np.int16),
                             entry_abs=np.array([[0.5, 0.25, 0, 0], [0.3, 0, 0, 0], [0.1, 0.2, 0.3, 0]]),
                             n_iter=np.zeros((3, L), dtype=np.int32), kkt=np.zeros((3, L)), converged=8, fits=3,
                             scores=np.zeros((L, K, 4)))


def test_writers_formats(tmp_path):
    from g2vec_b200 import cli
    res = fake_result()
    genes = ["A", "B", "C", "D"]
    line = lasso.summary(res, np.array([0, 2]))
    assert line == ("lasso: alpha 0.5, 2-fold x 1 repeats, 3 of 100 lambdas; lambda_min 0.2 (1 genes, CV deviance "
                    "1.2000, AUC 0.750), lambda_1se 0.2 (1 genes, CV deviance 1.2000, AUC 0.750); top_lasso(2) "
                    "Jaccard 0.333 with the biomarkers; 1 biomarkers nonzero at lambda_1se; 1 of 9 fits did not certify")
    prefix = str(tmp_path / "r")
    cli.write_lasso(prefix, genes, [0, 1, 2, 0], res, ["A", "C"], line)
    assert open(prefix + "_lasso.txt").read() == (
        "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tEntry\tBeta_min\tBeta_1se\tFold_entered\tBiomarker\n"
        "A\t0\t1\t0.5\t0.5\t1.000000\t1\n"
        "B\t1\t2\t0\t0\t0.000000\t0\n"
        "C\t2\t-1\t0\t0\t0.500000\t1\n"
        "D\t0\t-1\t0\t0\t0.000000\t0\n" + line + "\n")
    cli.write_lasso_path(prefix, res)
    assert open(prefix + "_lasso_path.txt").read() == (
        "Index\tLambda\tDf\tDev_ratio\tCV_deviance\tCV_SE\tCV_AUC\tMark\n"
        "0\t0.4\t0\t0.000000\t1.400000\t0.100000\t0.500000\t\n"
        "1\t0.2\t1\t0.100000\t1.200000\t0.050000\t0.750000\tmin,1se\n"
        "2\t0.1\t2\t0.250000\t1.300000\t0.200000\t0.650000\t\n")
    assert lasso.fold_top(res, 0, 1, 5).tolist() == [0, 1, 2]
