"""Host side of the survival CV (g2vec_b200/survival_cv.py, DESIGN.md §4.33) and the NumPy restatement of
tests/survival_cv_oracle.py, without a GPU."""
import math

import numpy as np
import pytest

from g2vec_b200 import cli, survival
from g2vec_b200 import survival_cv as scv
from tests import survival_cv_oracle as oc


def _records(rs, n, ties=True, p_event=0.6):
    t = rs.exponential(10.0, n)
    if ties:
        t = np.round(t / 3.0) * 3.0                    # heavy ties
    e = (rs.uniform(size=n) < p_event).astype(np.int64)
    e[0] = 1
    return t, e


def _setup(seed, n=60, p=4, scale=1.0):
    rs = np.random.RandomState(seed)
    t, e = _records(rs, n)
    order, flags, grp = oc.layout(t, e)
    z = rs.standard_normal((n, p)) * scale
    return z, grp, (flags & 1).astype(bool), rs


def _breslow(z, grp, ev, b):
    """The Breslow ridge objective written directly, in plain float64."""
    eta = z @ b
    L = 0.5 * b @ b - eta[ev].sum()
    for k in np.unique(grp):
        d = int(ev[grp == k].sum())
        if d:
            L += d * np.log(np.exp(eta[grp <= k]).sum())
    return L


def test_loss_gradient_and_hessian_are_the_derivatives_of_the_breslow_objective_with_ties():
    z, grp, ev, rs = _setup(1)
    b = 0.4 * rs.standard_normal(4)
    L, g, H = oc.objective(z, grp, ev, b)
    assert abs(L - _breslow(z, grp, ev, b)) <= 1e-12 * abs(L)
    h = 1e-5
    I = np.eye(4)
    gn = np.array([(_breslow(z, grp, ev, b + h * I[j]) - _breslow(z, grp, ev, b - h * I[j])) / (2 * h) for j in range(4)])
    Hn = np.array([(oc.objective(z, grp, ev, b + h * I[j])[1] - oc.objective(z, grp, ev, b - h * I[j])[1]) / (2 * h)
                   for j in range(4)])
    assert np.abs(g - gn).max() <= 1e-7 * max(1.0, np.abs(g).max())
    assert np.abs(H - Hn).max() <= 1e-7 * max(1.0, np.abs(H).max())


def test_two_gram_hessian_equals_the_direct_form():
    z, grp, ev, rs = _setup(2)
    b = 0.3 * rs.standard_normal(4)
    H = oc.objective(z, grp, ev, b)[2]
    eta = z @ b
    D = np.eye(4)
    for k in np.unique(grp):
        d = int(ev[grp == k].sum())
        if d:
            R = grp <= k
            w = np.exp(eta[R])
            m = (w[:, None] * z[R]).sum(0) / w.sum()
            D += d / w.sum() * ((w[:, None] * (z[R] - m)).T @ (z[R] - m))
    assert np.abs(H - D).max() <= 1e-12 * np.abs(D).max()


def test_oracle_minimiser_agrees_with_scipy():
    from scipy.optimize import minimize
    z, grp, ev, _ = _setup(3)
    b, it, ok = oc.fit(z, grp, ev)
    r = minimize(lambda v: _breslow(z, grp, ev, v), np.zeros(4), method="BFGS", options={"gtol": 1e-10})
    assert ok and np.abs(b - r.x).max() <= 1e-6


def test_scaled_recurrences_stay_finite_and_match_mpmath_at_large_eta():
    import mpmath
    mpmath.mp.dps = 50
    z, grp, ev, rs = _setup(4, n=40, p=2)
    b = np.array([300.0, -200.0])                      # |eta| in the hundreds
    sc = {}
    L, g, H = oc.objective(z, grp, ev, b, scratch=sc)
    assert np.isfinite(L) and np.isfinite(g).all() and np.isfinite(H).all() and np.isfinite(sc["omega"]).all()
    eta = [mpmath.mpf(float(v)) for v in z @ b]
    for lk, d, a, _ in sc["groups"]:
        S0 = mpmath.fsum(mpmath.exp(eta[i]) for i in range(len(eta)) if grp[i] <= grp[a])
        assert abs(float(mpmath.log(S0)) - lk) <= 1e-12 * max(1.0, abs(lk))
    for i in range(len(eta)):
        om = mpmath.exp(eta[i]) * mpmath.fsum(
            int(ev[grp == k].sum()) / mpmath.fsum(mpmath.exp(eta[j]) for j in range(len(eta)) if grp[j] <= k)
            for k in np.unique(grp) if k >= grp[i])          # the risk sets that hold i
        assert abs(float(om) - sc["omega"][i]) <= 1e-10 * max(1.0, float(om))
    assert 0.0 <= sc["omega"].min() and sc["omega"].max() <= ev.sum()


def test_concordance_counts_against_a_double_loop_with_ties():
    rs = np.random.RandomState(5)
    n = 50
    t, e = _records(rs, n)
    eta = np.round(rs.standard_normal(n), 1)           # ties in eta
    cmp = con = tie = 0
    for i in range(n):
        for j in range(n):
            if t[i] < t[j] and e[i]:
                cmp += 1; con += eta[i] > eta[j]; tie += eta[i] == eta[j]
    order, flags, grp = oc.layout(t, e)
    assert oc.conc_counts(eta[order], grp, e[order].astype(bool)) == (cmp, con, tie)
    c = scv.concordance(np.array([[cmp, con, tie], [0, 0, 0]]))
    assert c[0] == (2.0 * con + tie) / (2.0 * cmp) and math.isnan(c[1])


def test_folds_are_stratified_by_event_and_every_test_fold_has_one():
    rs = np.random.RandomState(6)
    t, e = _records(rs, 97, p_event=0.2)
    _, flags, _ = oc.layout(t, e)
    F = 5
    fold = oc.folds(flags, 3, F, 9)
    ev = (flags & 1).astype(bool)
    for k in range(3):
        per = np.bincount(fold[k][ev], minlength=F)
        assert per.min() >= 1 and per.max() - per.min() <= 1
        cen = np.bincount(fold[k][~ev], minlength=F)
        assert cen.max() - cen.min() <= 1


def test_log_rank_z_and_hazard_ratio():
    from scipy.stats import logrank
    from scipy.optimize import minimize_scalar
    rs = np.random.RandomState(7)
    n = 80
    t = rs.exponential(10.0, n)                        # no tied times
    e = (rs.uniform(size=n) < 0.7).astype(np.int64)
    scores = rs.standard_normal((3, n)) + (t < 8.0)
    risk, group, z, p, hr, lo, hi = scv.risk_groups(scores, t, e)
    assert np.array_equal(risk, scores.mean(0)) and (group == (risk > np.median(risk))).all()
    from scipy.stats import CensoredData
    hi_d = CensoredData(uncensored=t[(group == 1) & (e == 1)], right=t[(group == 1) & (e == 0)])
    lo_d = CensoredData(uncensored=t[(group == 0) & (e == 1)], right=t[(group == 0) & (e == 0)])
    want = logrank(hi_d, lo_d).statistic
    assert abs(abs(z) - abs(want)) <= 1e-10 and abs(p - math.erfc(abs(z) / math.sqrt(2))) <= 1e-15

    def nll(b):
        return oc.loss(group[np.argsort(-t, kind="stable")][:, None].astype(float),
                       np.arange(n), e[np.argsort(-t, kind="stable")].astype(bool), np.array([b])) - 0.5 * b * b
    r = minimize_scalar(nll, bracket=(-2, 2), tol=1e-12)
    assert abs(math.log(hr) - r.x) <= 1e-6 and lo < hr < hi
    e2 = e.copy(); e2[group == 0] = 0                  # no event in the low group
    assert math.isnan(scv.risk_groups(scores, t, e2)[4])


def test_summaries():
    c = np.array([[[0.7, 0.8]], [[0.6, np.nan]], [[0.5, 0.5]], [[0.65, 0.65]], [[0.9, 0.9]], [[np.nan, np.nan]]])
    c = np.concatenate([c, c], axis=1)                 # K = 2
    c_mean, c_sd, p_random = scv.summarise(c, 3, 3)
    assert np.allclose(c_mean[:5], [0.75, 0.6, 0.5, 0.65, 0.9]) and math.isnan(c_mean[5])
    assert c_sd[0] == 0.0 and math.isnan(scv.summarise(c[:, :1], 3, 3)[1][0])
    assert list(p_random) == [2 / 4, 3 / 4, 3 / 4]     # NaN never counts as >=


def _inputs(n=40, G=30):
    rs = np.random.RandomState(8)
    x = rs.standard_normal((n, G))
    t, e = _records(rs, n)
    return x, t, e, rs.randint(0, 2, n)


@pytest.mark.parametrize("case", ["R0", "F1", "K0", "K101", "Fevents", "Fhalf", "fits", "p0", "p129", "nan_x",
                                  "no_event", "label"])
def test_check_inputs_refuses(case):
    x, t, e, lab = _inputs()
    kw = dict(p=5, n_random=10, folds=3, repeats=2)
    if case == "R0": kw["n_random"] = 0
    if case == "F1": kw["folds"] = 1
    if case == "K0": kw["repeats"] = 0
    if case == "K101": kw["repeats"] = 101
    if case == "Fevents": e[:] = 0; e[:2] = 1
    if case == "Fhalf": t[3:] = np.nan; kw["folds"] = 2; e[:3] = 1
    if case == "fits": kw.update(n_random=65536, folds=20, repeats=100)
    if case == "p0": kw["p"] = 0
    if case == "p129": kw["p"] = 31
    if case == "nan_x": x[0, 0] = np.nan
    if case == "no_event": e[:] = 0
    if case == "label": lab[:] = 0
    with pytest.raises(ValueError):
        scv.check_inputs(x, t, e, lab, **kw)


def test_survival_cv_refuses_before_any_upload_and_without_a_device(monkeypatch):
    import torch
    x, t, e, lab = _inputs()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(ValueError):
        scv.survival_cv(x, t, e, lab, np.array([1, 1, 2]), 5)
    with pytest.raises(RuntimeError):
        scv.survival_cv(x, t, e, lab, np.array([1, 2, 3]), 5, folds=3, repeats=2)


def test_option_parsing(capsys):
    base = ["E", "C", "N", "R"]
    a = cli.parse_arguments(base)
    assert a.survival_cv == 0 and a.survival_cv_folds == 5 and a.survival_cv_repeats == 10
    for bad in (["--survival-cv", "3"], ["--survival", "S", "--survival-cv", "65537"],
                ["--survival", "S", "--survival-cv", "-1"], ["--survival-cv-folds", "1"],
                ["--survival-cv-folds", "101"], ["--survival-cv-repeats", "0"], ["--survival-cv-repeats", "101"],
                ["--survival", "S", "--survival-cv", "3", "-n", "65"]):
        with pytest.raises(SystemExit):
            cli.parse_arguments(base + bad)
    assert "--survival-cv needs --survival FILE" in capsys.readouterr().err


def test_step_2_refusals(tmp_path, capsys):
    from tests import helpers
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    samples = open(ef).readline().rstrip("\n").split("\t")[1:]
    sf = tmp_path / "s.tsv"
    with open(sf, "w") as f:
        f.write("SAMPLE\tTIME\tEVENT\n")
        f.writelines("%s\t%d\t%d\n" % (s, i, int(i < 3)) for i, s in enumerate(samples))   # 3 events
    for extra, msg in ((["--survival-cv-folds", "4"], "F = 4 folds need at least F events, got 3"),
                       (["--survival-cv", "65536", "--survival-cv-folds", "3", "--survival-cv-repeats", "100"],
                        "fits, at most 2^24")):
        with pytest.raises(SystemExit) as ex:
            cli.main([ef, cf, nf, str(tmp_path / "r"), "--survival", str(sf), "--survival-cv", "5"] + extra)
        assert ex.value.code == 1
        out = capsys.readouterr().out
        assert "ERROR: --survival-cv: " in out and msg in out


def _fake_result():
    S, K, F, p, n = 5, 2, 3, 4, 6
    c = np.full((S, K, F), 0.6)
    c_mean, c_sd, p_random = scv.summarise(c, 3, 2)
    return scv.SurvivalCVResult(
        names=["biomarkers", "top_t", "top_z", "random_1", "random_2"], genes=np.arange(S * p).reshape(S, p) % 7,
        folds=np.zeros((K, n), np.int8), counts=np.zeros((S, K, F, 3), np.int64), c=c,
        n_iter=np.ones((S, K, F), np.int32), converged=S * K * F - 2, beta=np.zeros((3, K, F, p)),
        scores=np.zeros((3, K, n)), c_mean=c_mean, c_sd=c_sd, p_random=p_random,
        risk=np.tile(np.linspace(-1, 1, n), (3, 1)), group=np.tile(np.array([0, 0, 0, 1, 1, 1], np.int8), (3, 1)),
        logrank_z=np.array([2.5, 1.0, 0.5]), logrank_p=np.array([0.0124, 0.3, 0.6]), hr=np.array([2.0, 1.2, np.nan]),
        hr_low=np.array([1.1, 0.8, np.nan]), hr_high=np.array([3.6, 1.8, np.nan]))


def test_writers_and_summary_format(tmp_path):
    r = _fake_result()
    genes = ["G%d" % i for i in range(7)]
    prefix = str(tmp_path / "res")
    cli.write_survival_cv(prefix, genes, r, ["G0", "G1"])
    rows = open(prefix + "_survival_cv.txt").read().splitlines()
    assert rows[0] == "Signature\tSize\tC\tC_SD\tP_random\tLogRank_Z\tLogRank_P\tHR\tHR_Low\tHR_High\tBiomarkers"
    assert rows[1] == "biomarkers\t4\t0.600000\t0.000000\t1\t2.500000\t0.0124\t2\t1.1\t3.6\t2"
    assert rows[3].split("\t")[7:10] == ["nan"] * 3
    assert rows[4].split("\t")[4:10] == ["nan"] * 6 and len(rows) == 6
    cli.write_risk(prefix, ["S%d" % i for i in range(6)], np.arange(6) * 1.5, [1, 0, 1, 0, 1, 1], r)
    risk = open(prefix + "_risk.txt").read().splitlines()
    assert risk[0] == "SAMPLE\tTIME\tEVENT\tRISK\tGROUP" and risk[2] == "S1\t1.5\t0\t-0.600000\t0"
    line = scv.summary(r)
    assert line.startswith("survival CV: 3-fold x 2 repeats, 4 genes: C 0.600 (biomarkers), 0.600 (top |t|), 0.600 "
                           "(top |Z|), random mean 0.600 [0.600, 0.600]; P_random 1 / 1 / 1; biomarker risk groups: "
                           "log-rank Z = 2.5000, P = 0.0124, HR 2.000 (1.100, 3.600)")
    assert line.endswith("; 2 of 30 fits did not converge")

