"""The survival CV on the H100 (csrc/g2v_cox.cu, g2vec_b200/survival_cv.py; DESIGN.md §4.33) against the NumPy
restatement of tests/survival_cv_oracle.py.  Concordance counts are compared exactly; coefficients and scores within
1e-8 max(1, |beta|), since exp and log are CUDA's."""
import os

import numpy as np
import pytest

from g2vec_b200 import signature, survival, survival_cv as scv
from tests import signature_oracle as so, survival_cv_oracle as oc

pytestmark = pytest.mark.gpu


def _lib():
    from g2vec_b200 import _capi
    return _capi, _capi.load()


def _st():
    import torch
    return torch.cuda.current_stream().cuda_stream


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gpu_fit(xs, flags, grp, genes, fold, cap=None):
    """xs [n, G] in position order -> scores [S, K, n], n_iter, converged [S, K, F], beta [S, K, F, p],
    counts [S, K, F, 3]."""
    import torch
    capi, lib = _lib()
    n, G = xs.shape
    S, p = genes.shape
    K = fold.shape[0]
    F = int(fold.max()) + 1
    n_pad = -(-n // 32) * 32
    Xt = np.zeros((G, n_pad)); Xt[:, :n] = xs.T
    Xd, fl, gr, fd, gd = _dev(Xt), _dev(flags.astype(np.uint8)), _dev(grp.astype(np.int32)), _dev(fold), \
        _dev(genes.astype(np.int32))
    sc = torch.full((S, K, n), np.nan, dtype=torch.float64, device="cuda")
    ell = torch.empty((S * K * F, n), dtype=torch.float64, device="cuda")
    it = torch.empty((S, K, F), dtype=torch.int32, device="cuda")
    cv = torch.empty((S, K, F), dtype=torch.uint8, device="cuda")
    be = torch.empty((S, K, F, p), dtype=torch.float64, device="cuda")
    capi.check(lib.g2v_cox_fit(Xd.data_ptr(), G, n, n_pad, fl.data_ptr(), fd.data_ptr(), K, F, gd.data_ptr(), S, p,
                               ell.data_ptr(), sc.data_ptr(), it.data_ptr(), cv.data_ptr(), be.data_ptr(), S, _st()),
               "g2v_cox_fit")
    if cap is None:
        cap = min(scv.MAX_STAGED, max(int((fold[k] == f).sum()) for k in range(K) for f in range(F)))
    cnt = torch.empty((S, K, F, 3), dtype=torch.int64, device="cuda")
    capi.check(lib.g2v_cox_concordance(sc.data_ptr(), fl.data_ptr(), gr.data_ptr(), fd.data_ptr(), n, K, F, S, cap,
                                       cnt.data_ptr(), _st()), "g2v_cox_concordance")
    return sc.cpu().numpy(), it.cpu().numpy(), cv.cpu().numpy(), be.cpu().numpy(), cnt.cpu().numpy()


def _data(n, G, seed, p_event=0.7, ties=False):
    rs = np.random.RandomState(seed)
    x = rs.standard_normal((n, G)) * rs.uniform(0.5, 3.0, G) + rs.uniform(-5, 5, G)
    haz = np.exp(0.5 * (x[:, 0] - x[:, 0].mean()) / x[:, 0].std())
    t = rs.exponential(1.0 / haz)
    if ties:
        t = np.round(t * 4) / 4
    e = (rs.uniform(size=n) < p_event).astype(np.int64)
    e[rs.randint(n)] = 1
    return x, t, e


def _check(x, t, e, genes, K, F, seed=1, cap=None):
    order, flags, grp = oc.layout(t, e)
    xs = x[order]
    fold = oc.folds(flags, K, F, seed)
    sc, it, cv, be, cnt = gpu_fit(xs, flags, grp, genes, fold, cap)
    want = oc.cv(xs, flags, grp, genes, fold)
    assert cv.all() and (it >= 1).all() and (it <= 100).all()
    scale = np.abs(want["beta"]).max(axis=-1, keepdims=True)
    assert np.all(np.abs(be - want["beta"]) <= 1e-8 * np.maximum(1.0, scale))
    tol = 1e-8 * max(1.0, float(scale.max()))
    assert np.all(np.abs(sc - want["scores"]) <= tol * np.maximum(1.0, np.abs(want["scores"])))
    ev = (flags & 1).astype(bool)
    for s in range(genes.shape[0]):
        for k in range(K):
            for f in range(F):
                te = fold[k] == f
                assert tuple(cnt[s, k, f]) == oc.conc_counts(sc[s, k, te], grp[te], ev[te])
    return sc, be, cnt, fold, want


@pytest.mark.parametrize("p", [1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 100, 127, 128])
def test_fits_equal_the_oracle_at_every_signature_size(p):
    x, t, e = _data(135, 200, p, ties=p % 2 == 0)
    rs = np.random.RandomState(p)
    genes = np.stack([np.sort(rs.choice(200, p, replace=False)) for _ in range(2)])
    _check(x, t, e, genes, 2, 5)


@pytest.mark.parametrize("n,F", [(4, 2), (10, 5), (135, 5), (1000, 5), (4097, 3)])
def test_fits_equal_the_oracle_at_every_sample_count(n, F):
    x, t, e = _data(n, 40, n, p_event=0.9 if n < 20 else 0.7)
    genes = np.array([np.arange(0, 40, 2), np.arange(1, 40, 2)])[:, : min(20, n)]
    _check(x, t, e, genes, 2, F)


def test_fits_at_the_largest_cohort_staged_and_from_global_memory():
    x, t, e = _data(32768, 6, 4, ties=True)
    genes = np.array([[0, 1, 2, 3, 4, 5]])
    sc, be, cnt, fold, _ = _check(x, t, e, genes, 1, 2)
    order, flags, grp = oc.layout(t, e)
    _, _, _, _, cnt2 = gpu_fit(x[order], flags, grp, genes, fold, cap=0)     # every fold read from global memory
    assert (cnt2 == cnt).all()


def test_fits_on_hard_data():
    rs = np.random.RandomState(9)
    n = 60
    x, t, e = _data(n, 12, 9)
    order, flags, grp = oc.layout(t, e)
    fold = oc.folds(flags, 2, 3, 1)
    xs = x[order]
    xs[:, 4] = 1.0
    xs[fold[0] == 1, 4] = 2.0                         # constant over the training rows of fold (0, 1) only
    xs[:, 5] = -np.arange(n) + 0.01 * rs.standard_normal(n)   # orders the times perfectly
    xs[:, 6] = xs[:, 7]                               # duplicated columns
    xs[:, 8] *= 2.0 ** 40
    xs[:, 9] *= 2.0 ** -40
    xs[:, 10] = 7.5                                   # constant everywhere
    genes = np.array([[4, 5, 6, 7, 8, 9, 10, 11]])
    sc, it, cv, be, cnt = gpu_fit(xs, flags, grp, genes, fold)
    want = oc.cv(xs, flags, grp, genes, fold)
    assert cv.all() and np.isfinite(be).all()
    assert np.all(np.abs(be - want["beta"]) <= 1e-8 * np.maximum(1.0, np.abs(want["beta"]).max()))
    assert (be[..., 6] == 0).all()                    # the constant gene's coefficient is exactly 0
    assert be[0, 0, 1, 0] == 0                        # gene 4 is constant on the training rows of fold (0, 1)


@pytest.mark.parametrize("case", ["all_events", "few_events", "one_time"])
def test_fits_on_hard_records(case):
    x, t, e = _data(80, 10, 5)
    if case == "all_events":
        e[:] = 1
    elif case == "few_events":
        e[:] = 0
        e[[3, 40, 77]] = 1
    else:
        t[:] = 2.5                                    # every sample tied in time
    _check(x, t, e, np.array([np.arange(10)]), 2, 3)


def test_fits_with_a_two_valued_feature():
    x, t, e = _data(200, 4, 7)
    x[:, 0] = np.where(np.arange(200) % 3 == 0, 60.0, -60.0) + np.random.RandomState(1).standard_normal(200)
    _check(x, t, e, np.array([[0, 1, 2, 3]]), 1, 4)


# --------------------------------------------------------------------------------------------------- the API
def _cohort(n=135, G=700, seed=3, effect=0.0):
    rs = np.random.RandomState(seed)
    x = rs.standard_normal((n, G))
    haz = np.exp(effect * x[:, :10].sum(axis=1) / np.sqrt(10))
    t = rs.exponential(1.0 / haz)
    e = (rs.uniform(size=n) < 0.75).astype(np.int64)
    t[rs.choice(n, 5, replace=False)] = np.nan        # samples without a record
    lab = rs.randint(0, 2, n)
    return x, t, e, lab


def _same(a, b):
    for f in a._fields:
        u, v = getattr(a, f), getattr(b, f)
        if isinstance(u, np.ndarray):
            assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v, equal_nan=u.dtype.kind == "f"), f
        else:
            assert u == v, f


def test_survival_cv_is_deterministic_chunking_invariant_and_paired():
    x, t, e, lab = _cohort()
    sig = np.arange(0, 700, 35)
    a = scv.survival_cv(x, t, e, lab, sig, 9, folds=4, repeats=2, seed=6)
    _same(a, scv.survival_cv(x, t, e, lab, sig, 9, folds=4, repeats=2, seed=6))
    n = int(np.isfinite(t).sum())
    per = 8 * 2 * n + 8 * 2 * 4 * n + 4 * len(sig) + 29 * 2 * 4
    for max_bytes in (1, per * 2, per * 5):
        _same(a, scv.survival_cv(x, t, e, lab, sig, 9, folds=4, repeats=2, seed=6, max_chunk_bytes=max_bytes))
    used = np.isfinite(t)
    assert a.names[:4] == ["biomarkers", "top_t", "top_z", "random_1"] and a.genes.shape == (12, 20)
    assert (a.genes[1] == np.sort(signature.top_t(x, lab, 20))).all()
    res = survival.survival_test(x[used], t[used], e[used], 1)
    assert (a.genes[2] == np.sort(res.order[:20])).all()
    sig_res = signature.signature_cv(x, lab, sig, 9, folds=4, repeats=2, seed=6)
    assert (a.genes[3:] == sig_res.genes[2:]).all()
    # named rows against the oracle
    order, flags, grp = oc.layout(t[used], e[used])
    fold_pos = oc.folds(flags, 2, 4, 6)
    assert (a.folds[:, order] == fold_pos).all()
    want = oc.cv(x[used][order], flags, grp, a.genes[:3], fold_pos)
    assert np.all(np.abs(a.beta - want["beta"]) <= 1e-8 * np.maximum(1.0, np.abs(want["beta"]).max()))
    assert a.converged == 12 * 8 and np.isfinite(a.c).all()
    for s in range(3):
        rg = scv.risk_groups(a.scores[s], t[used], e[used])
        assert np.array_equal(rg[0], a.risk[s]) and rg[2] == a.logrank_z[s]


def test_planted_effect_gives_high_c_and_a_null_cohort_one_half():
    x, t, e, lab = _cohort(n=300, G=2000, seed=11, effect=1.5)
    R = 40
    r = scv.survival_cv(x, t, e, lab, np.arange(10), R, folds=5, repeats=2, seed=1)
    assert r.c_mean[0] > 0.7 and r.p_random[0] == 1.0 / (R + 1) and r.logrank_p[0] < 1e-4 and r.hr[0] > 1.5
    x, t, e, lab = _cohort(n=300, G=2000, seed=12)
    r = scv.survival_cv(x, t, e, lab, np.arange(10), 200, folds=5, repeats=1, seed=3)
    assert abs(r.c_mean[3:].mean() - 0.5) < 0.03


def test_entry_points_refuse_bad_sizes_and_launch_nothing():
    capi, lib = _lib()
    import torch
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p, st = buf.data_ptr(), _st()
    before = capi.launch_count()
    fit = lambda n=100, K=2, F=5, S=1, pp=10, G=50, n_pad=128, rows=0, ell=p: lib.g2v_cox_fit(
        p, G, n, n_pad, p, p, K, F, p, S, pp, ell, p, p, p, p, rows, st)
    conc = lambda n=100, K=2, F=5, S=1, cap=20: lib.g2v_cox_concordance(p, p, p, p, n, K, F, S, cap, p, st)
    bad = [fit(n=2), fit(n=32769, n_pad=32800), fit(K=0), fit(K=101), fit(F=1), fit(F=101), fit(n=10, F=6), fit(S=0),
           fit(pp=0), fit(pp=129, G=200), fit(pp=51), fit(n_pad=99), fit(rows=2), fit(ell=None),
           fit(S=(1 << 24) // 10 + 1, K=2, F=5),
           conc(cap=-1), conc(cap=101), conc(n=2), conc(S=0), conc(F=1), conc(n=20000, cap=18433)]
    assert all(rc != 0 for rc in bad)
    assert int(lib.g2v_cox_fit_smem_bytes(0)) == 0 and int(lib.g2v_cox_fit_smem_bytes(129)) == 0
    assert capi.launch_count() == before and len(lib.g2v_last_error()) > 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------- CLI
def test_command_line_writes_the_two_files_and_leaves_the_other_files_alone(tmp_path, capsys):
    from g2vec_b200 import cli
    from tests import helpers
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    samples = open(ef).readline().rstrip("\n").split("\t")[1:]
    rs = np.random.RandomState(5)
    sf = tmp_path / "surv.tsv"
    with open(sf, "w") as f:
        f.write("SAMPLE\tTIME\tEVENT\n")
        for i, s in enumerate(samples):
            f.write("%s\t%s\t%s\n" % ((s, "NA", "NA") if i % 17 == 3 else (s, "%.1f" % rs.exponential(30.0),
                                                                          int(rs.uniform() < 0.6))))
    base = ["-r", "2", "-e", "5", "-n", "20", "--seed", "3", "--deterministic", "--survival", str(sf),
            "--survival-permutations", "10"]
    a, b = str(tmp_path / "plain"), str(tmp_path / "scv")
    cli.main([ef, cf, nf, a] + base)
    log_a = capsys.readouterr().out
    cli.main([ef, cf, nf, b] + base + ["--survival-cv", "20", "--survival-cv-repeats", "2"])
    log_b = capsys.readouterr().out
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt", "_survival.txt"):
        assert open(a + suffix).read() == open(b + suffix).read(), suffix
    assert not os.path.exists(a + "_survival_cv.txt") and not os.path.exists(a + "_risk.txt")
    import re
    untimed = lambda log, prefix: [re.sub(r" \([0-9.]+ sec\)$", "", l).replace(prefix, "RES")
                                   for l in log.splitlines()]
    extra = [l for l in untimed(log_b, b) if l not in untimed(log_a, a)]
    assert len(extra) == 4 and extra[0].startswith("Namespace(") and "survival_cv=20" in extra[0]
    assert extra[1].startswith("    survival CV: 5-fold x 2 repeats, ")
    assert extra[2:] == ["    RES_survival_cv.txt", "    RES_risk.txt"]
    rows = open(b + "_survival_cv.txt").read().splitlines()
    assert rows[0].split("\t") == ["Signature", "Size", "C", "C_SD", "P_random", "LogRank_Z", "LogRank_P", "HR",
                                   "HR_Low", "HR_High", "Biomarkers"] and len(rows) == 24
    assert rows[4].startswith("random_1\t") and rows[4].split("\t")[4:10] == ["nan"] * 6
    risk = open(b + "_risk.txt").read().splitlines()
    assert risk[0] == "SAMPLE\tTIME\tEVENT\tRISK\tGROUP"
    assert [r.split("\t")[0] for r in risk[1:]] == [s for i, s in enumerate(samples) if i % 17 != 3]
