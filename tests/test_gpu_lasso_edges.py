"""The lasso path on the GPU (DESIGN.md §4.37) where tests/test_gpu_lasso.py does not reach: the numbers the command
line reports from the solutions (held-out deviance, cvm, cvsd, lambda_min, lambda_1se, fit 0's intercept, deviance
ratio and df) against the float64 oracle; more than 64 fits (the second fit tile of g2v_lasso_grad); a gene constant on
some training folds only; alpha below glmnet's 1e-3 floor; KKT-violator rounds; a path capped at 512 genes across
chunkings; and a minority class of exactly F samples.

Tolerances, in terms of the certificate's eps = 1e-7: the device stops Newton when a sweep moves no coordinate by
more than v d^2 < 1e-20 and the oracle at 1e-22, so both solutions are far inside eps, and at G < n (a strictly convex
problem) a solution is determined to well below eps / (smallest curvature).  The held-out eta of two such solutions
agree to 1e-5 (100 eps, as in test_gpu_lasso.py); on well-conditioned cohorts they agree to ~1e-8, and cvm and cvsd
to 1e-9 relative.  Where a fold fit is nearly separable its solution is determined only to eps / (a small curvature)
and cvm is not compared with the oracle's: it is checked in two parts, the device's own held-out eta through the
oracle's deviance and rule (to summation order), and that eta against the oracle's (1e-5).  A held-out deviance moves
by at most 2 |d eta| (its slope is -2 (1 - p) or 2 p, and 0 where p is clamped), so cvm is then within
2 mean |d eta| of the oracle's."""
import numpy as np
import pytest

from tests import lasso_oracle as orc
from tests.test_gpu_lasso import check_fit, cohort, run

pytestmark = pytest.mark.gpu

EPS = 1e-7
FIELDS = ("lambdas", "a0", "beta", "df", "dev_ratio", "cvm", "cvsd", "auc", "auc_mean", "entry", "entry_abs", "n_iter",
          "kkt", "scores", "folds")


def same(a, b, fields=FIELDS):
    for name in fields:
        assert np.array_equal(getattr(a, name), getattr(b, name)), name
    assert (a.n_lambda, a.i_min, a.i_1se, a.converged, a.fits) == (b.n_lambda, b.i_min, b.i_1se, b.converged, b.fits)


def per_fit_bytes(G, n):
    """lasso_cv's per-fit device bytes of a chunk, so that max_chunk_bytes = r per_fit_bytes gives r fits per chunk."""
    from g2vec_b200 import _capi, lasso
    n_pad = -(-n // 32) * 32
    ws = int(_capi.load().g2v_lasso_workspace_bytes(G, n_pad, 1))
    assert ws > 0
    return ws + 10 * G + 24 * lasso.N_LAMBDA


def fold_fit(res, x, lab, k, f):
    """The oracle's path of fold fit (k, f) on its training samples with the device's lambdas, and the test mask."""
    te = res.folds[k] == f
    return orc.path(x[~te], lab[~te].astype(np.float64), res.alpha, lams=res.lambdas), te


def oracle_scores(res, x, lab):
    """The oracle's held-out eta [L, K, n] of every fold fit."""
    K, F = res.auc.shape[1:]
    sc = np.zeros_like(res.scores)
    for k in range(K):
        for f in range(F):
            fit, te = fold_fit(res, x, lab, k, f)
            for li in range(res.n_lambda):
                sc[li, k, te] = orc.predict(fit, x[te], li)
    return sc


def check_pick(res, want, tol):
    """i_min and i_1se equal the oracle's, or, where the oracle's cvm is within tol of a tie that decides them, the
    device's picks satisfy the rule on the device's own cvm and cvsd."""
    cvm, cvsd, i_min, i_1se = want
    near_min = (np.abs(cvm - cvm[i_min]) <= tol).sum() > 1
    if not near_min:
        assert res.i_min == i_min
    assert res.cvm[res.i_min] == res.cvm.min() and (res.cvm[:res.i_min] > res.cvm.min()).all()
    thr = cvm[i_min] + cvsd[i_min]
    if not near_min and not (np.abs(cvm - thr) <= tol).any():
        assert res.i_1se == i_1se
    t = res.cvm[res.i_min] + res.cvsd[res.i_min]
    assert res.cvm[res.i_1se] <= t and (res.cvm[:res.i_1se] > t).all()


def check_cv(res, x, lab, rtol=1e-9):
    """cvm, cvsd, lambda_min and lambda_1se: the device's held-out eta through the oracle's deviance and rule, that
    eta against the oracle's fold paths, and (rtol not None) cvm and cvsd against the oracle's own to rtol relative.
    Returns the oracle's held-out eta."""
    F = res.auc.shape[2]
    y = lab[None, None, :]
    # the device's own held-out eta through the oracle's deviance and rule: the same numbers up to summation order
    own = orc.cv_glmnet(orc.heldout_deviance(res.scores, y), res.folds, F)
    np.testing.assert_allclose(res.cvm, own[0], rtol=1e-13)
    np.testing.assert_allclose(res.cvsd, own[1], rtol=1e-11)
    assert (res.i_min, res.i_1se) == own[2:]
    sc = oracle_scores(res, x, lab)
    np.testing.assert_allclose(res.scores, sc, atol=1e-5)
    want = orc.cv_glmnet(orc.heldout_deviance(sc, y), res.folds, F)
    if rtol is not None:
        np.testing.assert_allclose(res.cvm, want[0], rtol=rtol)
        np.testing.assert_allclose(res.cvsd, want[1], rtol=rtol)
    # a tie closer than the comparison's resolution may go either way
    tol = rtol * np.abs(want[0]).max() if rtol is not None else 2.0 * np.abs(res.scores - sc).max()
    check_pick(res, want, tol)
    return sc


def separable(n=40, G=10, seed=4):
    rs = np.random.RandomState(seed)
    x = rs.randn(n, G)
    lab = (np.arange(n) % 2).astype(np.int64)
    x[:, 0] += 6.0 * lab                               # separable on one gene
    return x, lab


# ------------------------------------------------------------------------------------ 1. cvm, cvsd, the lambda picks
@pytest.mark.parametrize("data,alpha", [("plain", 1.0), ("plain", 0.5), ("separable", 1.0)])
def test_cv_outputs_against_oracle(data, alpha):
    x, lab = cohort(60, 12, 21) if data == "plain" else separable()
    res = run(x, lab, folds=4, repeats=2, alpha=alpha, seed=3)
    assert res.converged == res.fits * res.n_lambda
    sc = check_cv(res, x, lab)
    if data == "separable":
        # the clamp is reached: some held-out p is beyond [1e-5, 1 - 1e-5], on the device and in the oracle
        for s in (res.scores, sc):
            p = 1.0 / (1.0 + np.exp(-s))
            assert ((p < orc.P_MIN) | (p > 1.0 - orc.P_MIN)).any()


# ---------------------------------------------------------------------- 2. fit 0's intercept, deviance ratio and df
@pytest.mark.parametrize("alpha", [1.0, 0.5])
def test_fit0_intercept_dev_ratio_and_df(alpha):
    x, lab = cohort(60, 12, 22)
    res = run(x, lab, folds=3, alpha=alpha, seed=1)
    L = res.n_lambda
    ref = orc.path(x, lab.astype(np.float64), alpha, lams=res.lambdas)
    assert ref["L"] == L
    # |g0| <= eps on both sides and the curvature in b0 is mean p (1 - p) >= ~0.05 here: 1e-6 is 10 eps
    np.testing.assert_allclose(res.a0, ref["b0"][:L], atol=1e-6)
    # the deviance is stationary at the solution: a gradient within eps moves the ratio by O(eps^2)
    np.testing.assert_allclose(res.dev_ratio, ref["dev_ratio"][:L], rtol=0, atol=1e-9)
    nz = res.beta != 0
    assert (res.df == nz.sum(axis=1)).all()
    differ = nz != (ref["beta"][:L] != 0)
    # a gene at the edge of the active set may be zero on one side and within 100 eps of zero on the other
    assert (np.maximum(np.abs(res.beta), np.abs(ref["beta"][:L]))[differ] < 1e-5).all()
    assert (np.abs(res.df - (ref["beta"][:L] != 0).sum(axis=1)) <= differ.sum(axis=1)).all()


# ------------------------------------------------------------------------------------------ 3. more than 64 fits
@pytest.mark.parametrize("F,K", [(9, 7), (8, 8), (10, 10)])
def test_more_than_64_fits_chunked_and_against_oracle(F, K):
    n, G = 72, 10
    x, lab = cohort(n, G, 42)
    res = run(x, lab, folds=F, repeats=K, seed=7)
    assert res.fits == 1 + K * F and res.converged == res.fits * res.n_lambda
    per_fit = per_fit_bytes(G, n)
    for rows in (1, 64, 65):
        same(res, run(x, lab, folds=F, repeats=K, seed=7, max_chunk_bytes=rows * per_fit))
    # every fold fit of the second 64-fit tile, and a few of the first, against the oracle
    for gf in sorted(set(range(64, res.fits)) | {1, 63}):
        k, f = divmod(gf - 1, F)
        fit, te = fold_fit(res, x, lab, k, f)
        for li in range(res.n_lambda):
            np.testing.assert_allclose(res.scores[li, k, te], orc.predict(fit, x[te], li), atol=1e-5,
                                       err_msg="fit %d lambda %d" % (gf, li))
    if K == 10:
        # the folds of repeat k depend on (seed, k) only: K = 1 is a prefix of K = 10
        one = run(x, lab, folds=F, repeats=1, seed=7)
        assert np.array_equal(one.folds[0], res.folds[0])
        for name in ("lambdas", "a0", "beta", "df", "dev_ratio"):
            assert np.array_equal(getattr(one, name), getattr(res, name)), name
        for name in ("entry", "entry_abs", "kkt", "n_iter"):
            assert np.array_equal(getattr(one, name)[:F + 1], getattr(res, name)[:F + 1]), name
        assert np.array_equal(one.scores[:, 0], res.scores[:, 0])


# ------------------------------------------------------------------------ 4. a gene constant on some folds only
@pytest.mark.parametrize("variant", ["fold", "two"])
def test_gene_constant_on_some_training_folds_only(variant):
    n, G, F = 80, 10, 4
    x, lab = cohort(n, G, 41, const=False)
    first = run(x, lab, folds=F, repeats=2, seed=9)
    te = first.folds[0] == 0                           # held out by fit 1: fold 0 of repeat 0
    j = G - 1
    # a floor value off fold 0 of repeat 0, not 0: a sum of copies of 0.3 divided by their count need not give 0.3
    # back, so a kernel that misjudged the gene as varying would get an SD of 0 or of rounding noise, and an isd of
    # inf or ~1e16, instead of quietly multiplying zeros
    x[:, j] = 0.3
    rows = np.nonzero(te)[0]
    if variant == "two":                               # off the floor on two samples of fold 0, one per label
        rows = np.r_[rows[lab[rows] == 1][:1], rows[lab[rows] == 0][:1]]
        x[rows, j] = [2.3, 1.3]
    else:                                              # off the floor on fold 0 of repeat 0, with some label signal
        rs = np.random.RandomState(41)
        x[rows, j] = 1.3 + 0.6 * lab[rows] + 0.5 * rs.randn(rows.size)
    res = run(x, lab, folds=F, repeats=2, seed=9)
    assert np.array_equal(res.folds, first.folds)      # the folds depend on the labels and the seed only
    assert res.converged == res.fits * res.n_lambda
    # constant over fit 1's training samples: it never enters fit 1, and fit 1's held-out eta ignores it
    assert res.entry[1, j] == -1 and res.entry_abs[1, j] == 0.0
    fit, te1 = fold_fit(res, x, lab, 0, 0)
    assert fit["const"][j] and np.array_equal(te1, te)
    assert np.isfinite(res.scores).all()
    for li in range(res.n_lambda):
        np.testing.assert_allclose(res.scores[li, 0, te], orc.predict(fit, x[te], li), atol=1e-5)
    # and it varies, and enters, in the fits that train on those samples
    assert (res.entry[np.r_[0, 2:res.fits], j] >= 0).any()
    check_fit(res, x, lab, 1.0, res.n_lambda)
    varies = 0
    for gf in range(2, res.fits):                      # every other fold fit, constant there or not
        k, f = divmod(gf - 1, F)
        other, te2 = fold_fit(res, x, lab, k, f)
        varies += not other["const"][j]
        if other["const"][j]:
            assert res.entry[gf, j] == -1
        for li in range(res.n_lambda):
            np.testing.assert_allclose(res.scores[li, k, te2], orc.predict(other, x[te2], li), atol=1e-5)
    assert varies > 0


# ------------------------------------------------------------------------------------ 5. alpha below the 1e-3 floor
@pytest.mark.parametrize("alpha", [1e-2, 1e-3, 1e-4])
def test_alpha_below_glmnet_floor(alpha):
    x, lab = cohort(60, 12, 50)
    y = lab.astype(np.float64)
    res = run(x, lab, folds=3, alpha=alpha, seed=2)
    z, mu, sd, const = orc.standardise(x)
    np.testing.assert_allclose(res.lambdas, orc.lambdas(z, y, alpha)[:res.n_lambda], rtol=1e-12)
    ref = check_fit(res, x, lab, alpha, res.n_lambda)
    assert ref["L"] == res.n_lambda
    np.testing.assert_allclose(res.beta, ref["beta"][:res.n_lambda], atol=1e-6)
    np.testing.assert_allclose(res.a0, ref["b0"][:res.n_lambda], atol=1e-6)
    # below the floor lambda_max is no longer the null solution's lambda: the first solution has genes
    assert res.beta[0].any() == (alpha < 1e-3)
    if alpha < 1e-3:
        assert res.df[0] > 0 and (ref["beta"][0] != 0).any()
    assert res.converged == res.fits * res.n_lambda
    # G > n: the certificate on the host and the objective against the oracle's
    x2, lab2 = cohort(30, 40, 51)
    res2 = run(x2, lab2, folds=3, alpha=alpha, seed=2)
    z2, _, _, _ = orc.standardise(x2)
    np.testing.assert_allclose(res2.lambdas, orc.lambdas(z2, lab2.astype(np.float64), alpha)[:res2.n_lambda],
                               rtol=1e-12)
    check_fit(res2, x2, lab2, alpha, res2.n_lambda)
    assert res2.converged == res2.fits * res2.n_lambda
    assert res2.beta[0].any() == (alpha < 1e-3)


# ------------------------------------------------------------------------------------------ 6. KKT-violator rounds
def suppressor(seed, n=60, G=24):
    """Suppressor genes: a = s + 1.5 e is a noisy copy of a signal s, b = e is its noise alone (marginally unrelated to
    the label), and a - 1.5 b = s.  Once a enters, b's gradient can grow faster than lambda falls, which the
    sequential strong rule assumes it does not."""
    rs = np.random.RandomState(seed)
    m = G // 3
    s, e = rs.randn(n, m), rs.randn(n, m)
    x = np.concatenate([s + 1.5 * e, e, rs.randn(n, m)], axis=1)
    eta = 2.0 * s[:, 0] - 1.5 * s[:, 1] + s[:, 2]
    lab = (rs.rand(n) < 1 / (1 + np.exp(-eta))).astype(np.int64)
    lab[:2] = [0, 1]
    return x, lab


def fit0_rounds(monkeypatch):
    """Records (lambda index, round) of every g2v_lasso_cd call on the chunk that starts at fit 0."""
    from g2vec_b200 import _capi
    lib = _capi.load()
    std, cd = lib.g2v_lasso_standardise, lib.g2v_lasso_cd
    chunk, calls = [None], []

    def std_hook(*args):
        chunk[0] = int(args[8])                        # fit0: the chunk's first global fit
        return std(*args)

    def cd_hook(*args):
        if chunk[0] == 0:
            calls.append((int(args[7]), int(args[11])))
        return cd(*args)
    monkeypatch.setattr(lib, "g2v_lasso_standardise", std_hook)
    monkeypatch.setattr(lib, "g2v_lasso_cd", cd_hook)
    return calls


def test_kkt_violator_rounds_certify(monkeypatch):
    x, lab = suppressor(0)
    n, G = x.shape
    calls = fit0_rounds(monkeypatch)
    # one fit per chunk, so the first chunk's calls are fit 0's alone
    res = run(x, lab, folds=2, seed=0, max_chunk_bytes=per_fit_bytes(G, n))
    monkeypatch.undo()
    assert calls and calls[0] == (0, 0)
    late = sorted({k for k, r in calls if r >= 2 and k < res.n_lambda})
    assert late, "fit 0 needed no round after the first KKT-violator round"
    z, mu, sd, const = orc.standardise(x)
    y = lab.astype(np.float64)
    lam = res.lambdas
    b00 = np.log(y.mean() / (1 - y.mean()))
    # replay the sequential strong rule on fit 0's own solutions: a gene that enters although the rule never admitted
    # it up to its entry joined the working set as a KKT violator, at a lambda no later than its entry, and a round
    # that adds a violator is always followed by another
    admitted = np.zeros(G, dtype=bool)
    missed = []
    for k in range(res.n_lambda):
        a0, beta = (b00, np.zeros(G)) if k == 0 else (res.a0[k - 1], res.beta[k - 1])
        g = orc.gradient(z, y, a0, beta, lam[k], 1.0)[1]
        admitted |= np.abs(g) > 2 * lam[k] - lam[max(k - 1, 0)] - 1e-10       # host vs device g: ~1e-14
        missed += [(k, j) for j in np.nonzero((res.entry[0] == k) & ~admitted)[0]]
    assert missed, "every gene of fit 0 was admitted by the strong rule"
    assert any(late[0] <= k for k, j in missed), (missed, late)
    # every fit certified at those lambdas; fit 0's solutions pass the host's certificate, and their objective is
    # no worse than the oracle's own solve at that lambda (from the null model, over every gene)
    assert (res.kkt[:, late] <= EPS).all()
    for k in late:
        assert orc.kkt(z, y, res.a0[k], res.beta[k], lam[k], 1.0, const) <= EPS + 1e-12
        b0, beta = orc.solve(z, y, b00, np.zeros(G), lam[k], 1.0)
        o_dev = orc.objective(z, y, res.a0[k], res.beta[k], lam[k], 1.0)
        o_ref = orc.objective(z, y, b0, beta, lam[k], 1.0)
        assert o_dev <= o_ref + 1e-9 * abs(o_ref), (k, o_dev, o_ref)


# ------------------------------------------------------------------------------ 7. a capped path across chunkings
def test_capped_path_is_the_same_in_every_chunking():
    rs = np.random.RandomState(8)
    n, G = 2000, 1200
    x = rs.randn(n, G)
    eta = x @ (rs.randn(G) * 0.08)
    lab = (rs.rand(n) < 1 / (1 + np.exp(-eta))).astype(np.int64)
    a = run(x, lab, folds=3)
    assert a.n_lambda < 100 and (a.entry[0] >= 0).sum() <= 512
    b = run(x, lab, folds=3, max_chunk_bytes=1)
    same(a, b, ("entry", "entry_abs", "kkt", "n_iter", "scores", "cvm", "auc"))
    # no fit reports an entry at or after the lambda where fit 0 reached the cap
    assert (a.entry < a.n_lambda).all() and (b.entry < b.n_lambda).all()


# ------------------------------------------------------------------------- 8. a minority class of exactly F samples
def test_minority_class_equal_to_folds():
    rs = np.random.RandomState(60)
    n, G, F = 40, 10, 5
    x = rs.randn(n, G) + rs.uniform(-1, 1, G)
    lab = np.zeros(n, dtype=np.int64)
    lab[rs.choice(n, F, replace=False)] = 1
    x[:, :3] += 1.2 * lab[:, None]
    res = run(x, lab, folds=F, repeats=2, seed=4)
    for k in range(2):                                 # every held-out fold has exactly one minority sample
        assert (np.bincount(res.folds[k][lab == 1], minlength=F) == 1).all()
    assert res.converged == res.fits * res.n_lambda
    # four training positives make the fold fits nearly separable at small lambda: the eta-implied bound
    check_cv(res, x, lab, rtol=None)
