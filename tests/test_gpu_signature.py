"""The signature test on the H100 (csrc/g2v_sig.cu, g2vec_b200/signature.py; DESIGN.md §4.29) against the NumPy
restatement of tests/signature_oracle.py.  Folds, draws, AUC and accuracy are compared exactly; coefficients and
scores within 1e-8 max(1, |beta|), since exp and log1p are CUDA's."""
import os

import numpy as np
import pytest

from g2vec_b200 import signature
from g2vec_b200.signature import signature_cv
from tests import signature_oracle as so

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


def gpu_folds(y, K, F, seed):
    import torch
    capi, lib = _lib()
    out = torch.full((K, len(y)), -1, dtype=torch.int8, device="cuda")
    yd = _dev(np.asarray(y, np.uint8))
    capi.check(lib.g2v_sig_folds(yd.data_ptr(), len(y), K, F, seed, out.data_ptr(), _st()), "g2v_sig_folds")
    return out.cpu().numpy()


def gpu_draw(G, p, seed, r_begin, count):
    import torch
    capi, lib = _lib()
    out = torch.full((count, p), -1, dtype=torch.int32, device="cuda")
    capi.check(lib.g2v_sig_draw(G, p, seed, r_begin, count, out.data_ptr(), _st()), "g2v_sig_draw")
    return out.cpu().numpy()


def gpu_fit(x, y, genes, fold, beta_rows=None):
    """scores [S, K, n], n_iter, converged [S, K, F], beta [beta_rows, K, F, p + 1], auc, acc [S, K, F]."""
    import torch
    capi, lib = _lib()
    n, G = x.shape
    S, p = genes.shape
    K = fold.shape[0]
    F = int(fold.max()) + 1
    beta_rows = S if beta_rows is None else beta_rows
    n_pad = -(-n // 32) * 32
    Xt = np.zeros((G, n_pad)); Xt[:, :n] = x.T
    Xd, yd, fd, gd = _dev(Xt), _dev(np.asarray(y, np.uint8)), _dev(fold), _dev(genes.astype(np.int32))
    sc = torch.full((S, K, n), np.nan, dtype=torch.float64, device="cuda")
    it = torch.empty((S, K, F), dtype=torch.int32, device="cuda")
    cv = torch.empty((S, K, F), dtype=torch.uint8, device="cuda")
    be = torch.empty((max(beta_rows, 1), K, F, p + 1), dtype=torch.float64, device="cuda")
    capi.check(lib.g2v_sig_fit(Xd.data_ptr(), G, n, n_pad, yd.data_ptr(), fd.data_ptr(), K, F, gd.data_ptr(), S, p,
                               sc.data_ptr(), it.data_ptr(), cv.data_ptr(), be.data_ptr(), beta_rows, _st()),
               "g2v_sig_fit")
    cap = max(int((fold[k] == f).sum()) for k in range(K) for f in range(F))
    auc, acc = (torch.empty((S, K, F), dtype=torch.float64, device="cuda") for _ in range(2))
    capi.check(lib.g2v_sig_auc(sc.data_ptr(), yd.data_ptr(), fd.data_ptr(), n, K, F, S, cap, auc.data_ptr(),
                               acc.data_ptr(), _st()), "g2v_sig_auc")
    return (sc.cpu().numpy(), it.cpu().numpy(), cv.cpu().numpy(), be.cpu().numpy()[:beta_rows], auc.cpu().numpy(),
            acc.cpu().numpy())


def _close(got, want, tol=1e-8):
    return np.all(np.abs(got - want) <= tol * np.maximum(1.0, np.abs(want)))


# ------------------------------------------------------------------------------------------------ folds, draws
@pytest.mark.parametrize("F", [2, 3, 5, 10, 100])
def test_folds_equal_the_oracle_bit_for_bit(F):
    for extra in (0, 1, F - 1, 5000 - F):
        m0, m1 = F + extra, F + (extra * 7) % (F + 1)
        y = np.array([0] * m0 + [1] * m1, np.uint8)
        np.random.RandomState(F + extra).shuffle(y)
        got = gpu_folds(y, 3, F, 77)
        assert (got == so.folds(y, 3, F, 77)).all()


@pytest.mark.parametrize("G,p", [(1, 1), (128, 128), (129, 128), (7523, 100), (1 << 20, 128)])
def test_draws_equal_floyd_bit_for_bit(G, p):
    got = gpu_draw(G, p, 5, 3, 40)
    for q in range(40):
        assert (got[q] == so.floyd(G, p, 5, 3 + q)).all()
    last = gpu_draw(G, p, 5, signature.MAX_RANDOM, 1)
    assert (last[0] == so.floyd(G, p, 5, signature.MAX_RANDOM)).all()


# -------------------------------------------------------------------------------------------------------- fits
def _data(n, G, seed, n0=None):
    rs = np.random.RandomState(seed)
    y = np.zeros(n, np.int64)
    y[: n - (n // 2 if n0 is None else n0)] = 1
    rs.shuffle(y)
    x = rs.standard_normal((n, G)) * rs.uniform(0.5, 3.0, G) + rs.uniform(-5, 5, G)
    x[:, :3] += 0.7 * y[:, None]
    return x, y


def _check_fits(x, y, genes, K, F, seed=1):
    fold = so.folds(y, K, F, seed)
    sc, it, cv, be, auc, acc = gpu_fit(x, y, genes, fold)
    want = so.cv(x, y, genes, fold)
    assert cv.all() and (it >= 1).all() and (it <= 100).all()
    scale = np.abs(want["beta"]).max(axis=-1, keepdims=True)
    assert np.all(np.abs(be - want["beta"]) <= 1e-8 * np.maximum(1.0, scale))
    assert _close(sc, want["scores"], 1e-8 * max(1.0, float(scale.max())))
    return sc, auc, acc, fold, want


@pytest.mark.parametrize("p", [1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 100, 127, 128])
def test_fits_equal_the_oracle_at_every_signature_size(p):
    x, y = _data(135, 200, p)
    rs = np.random.RandomState(p)
    genes = np.stack([np.sort(rs.choice(200, p, replace=False)) for _ in range(2)])
    _check_fits(x, y, genes, 2, 5)


@pytest.mark.parametrize("n,F", [(10, 5), (4, 2), (135, 5), (1000, 5), (4097, 3)])
def test_fits_equal_the_oracle_at_every_sample_count(n, F):
    x, y = _data(n, 40, n)
    genes = np.array([np.arange(0, 40, 2), np.arange(1, 40, 2)])
    _check_fits(x, y, genes, 2, F)


def test_fits_at_the_largest_cohort():
    x, y = _data(32768, 6, 4)
    _check_fits(x, y, np.array([[0, 1, 2, 3, 4, 5]]), 1, 2)


def test_fits_on_hard_data():
    rs = np.random.RandomState(9)
    n = 60
    x, y = _data(n, 12, 9)
    fold = so.folds(y, 2, 3, 1)
    x[:, 4] = 1.0
    x[fold[0] == 1, 4] = 2.0                          # constant over the training rows of fold (0, 0) only
    x[:, 5] = np.where(y == 1, 3.0, -3.0) + 0.01 * rs.standard_normal(n)   # separates the labels perfectly
    x[:, 6] = x[:, 7]                                 # duplicated columns
    x[:, 8] *= 2.0 ** 40
    x[:, 9] *= 2.0 ** -40
    x[:, 10] = 7.5                                    # constant everywhere
    genes = np.array([[4, 5, 6, 7, 8, 9, 10, 11]])
    sc, it, cv, be, auc, acc = gpu_fit(x, y, genes, fold)
    want = so.cv(x, y, genes, fold)
    assert cv.all() and np.isfinite(be).all()
    assert np.all(np.abs(be - want["beta"]) <= 1e-8 * np.maximum(1.0, np.abs(want["beta"]).max()))
    assert (be[..., 7] == 0).all()                    # the constant gene's coefficient is exactly 0


def test_auc_and_accuracy_are_exact_counts_of_the_device_scores():
    x, y = _data(301, 50, 3)
    fold = so.folds(y, 3, 7, 2)
    genes = np.array([np.arange(10), np.arange(10, 20), np.arange(5, 15)])
    sc, it, cv, be, auc, acc = gpu_fit(x, y, genes, fold)
    want = so.cv(x, y, genes, fold)
    for s in range(3):
        for k in range(3):
            for f in range(7):
                te = fold[k] == f
                assert auc[s, k, f] == so.auc_counts(sc[s, k, te], y[te])
                assert acc[s, k, f] == so.accuracy(sc[s, k, te], y[te])
    assert (auc == want["auc"]).all() and (acc == want["acc"]).all()


def test_auc_counts_ties():
    """Scores of a constant gene are all the intercept: every pair ties, AUC = 1/2 exactly."""
    x, y = _data(50, 3, 1)
    x[:, 0] = 2.0
    sc, it, cv, be, auc, acc = gpu_fit(x, y, np.array([[0]]), so.folds(y, 2, 5, 3))
    assert (auc == 0.5).all()


# --------------------------------------------------------------------------------------------------- the API
def _ex():
    from tests.helpers import GOLDEN
    e = np.load(os.path.join(GOLDEN, "ex_expr.npz"))
    return e["expr"], np.load(os.path.join(GOLDEN, "ex_graph.npz"))["label"]


def _same(a, b):
    for f in a._fields:
        u, v = getattr(a, f), getattr(b, f)
        if isinstance(u, np.ndarray):
            assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v, equal_nan=u.dtype.kind == "f"), f
        else:
            assert u == v, f


def test_signature_cv_is_deterministic_and_chunking_invariant():
    x, lab = _ex()
    sig = np.arange(0, 7000, 140)
    a = signature_cv(x, lab, sig, 9, folds=4, repeats=2, seed=6)
    _same(a, signature_cv(x, lab, sig, 9, folds=4, repeats=2, seed=6))
    per = 8 * 2 * x.shape[0] + 4 * len(sig) + 21 * 2 * 4           # one signature's chunk buffers
    for max_bytes in (1, per * 2, per * 5):
        _same(a, signature_cv(x, lab, sig, 9, folds=4, repeats=2, seed=6, max_chunk_bytes=max_bytes))
    assert a.names[:3] == ["biomarkers", "top_t", "random_1"] and a.genes.shape == (11, 50)
    assert (a.genes[0] == sig).all() and (a.genes[1] == np.sort(signature.top_t(x, lab, 50))).all()
    for r in range(1, 10):
        assert (a.genes[r + 1] == so.floyd(x.shape[1], 50, 6, r)).all()
    used = (lab == 0) | (lab == 1)
    assert (a.folds == so.folds(lab[used], 2, 4, 6)).all()
    want = so.cv(x[used], lab[used], a.genes[:3], a.folds)
    assert (a.auc[:3] == want["auc"]).all() and (a.acc[:3] == want["acc"]).all()
    assert np.all(np.abs(a.beta - want["beta"][:2]) <= 1e-8 * np.maximum(1.0, np.abs(want["beta"][:2]).max()))
    assert (a.p_random == so.p_random(a.auc_mean, 9)).all() and a.converged == 11 * 8


def test_planted_signal_beats_random_signatures_and_top_t_only_where_it_should():
    rs = np.random.RandomState(11)
    n, G = 120, 3000
    x = rs.standard_normal((n, G))
    y = np.array([0] * 60 + [1] * 60)
    rs.shuffle(y)
    x[:, 100:120] += 1.0 * y[:, None]
    R = 50
    r = signature_cv(x, y, np.arange(100, 120), R, folds=5, repeats=3, seed=1)
    assert r.auc_mean[0] > 0.9 and r.p_random[0] == 1.0 / (R + 1) and r.converged == (R + 2) * 15
    assert abs(r.auc_mean[0] - r.auc_mean[1]) < 0.05   # top_t finds the same planted genes
    weak = signature_cv(x, y, np.arange(110, 130), R, folds=5, repeats=3, seed=1)   # half of it is noise
    assert weak.auc_mean[0] < r.auc_mean[1] and weak.p_random[0] == 1.0 / (R + 1)


def test_null_cohort_random_signatures_average_one_half():
    rs = np.random.RandomState(12)
    x = rs.standard_normal((100, 2000))
    y = rs.randint(0, 2, 100)
    r = signature_cv(x, y, np.arange(20), 200, folds=5, repeats=2, seed=3)
    assert abs(r.auc_mean[2:].mean() - 0.5) < 0.05


def test_entry_points_refuse_bad_sizes_and_launch_nothing():
    capi, lib = _lib()
    import torch
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p, st = buf.data_ptr(), _st()
    before = capi.launch_count()
    fit = lambda n=100, K=2, F=5, S=1, pp=10, G=50, n_pad=128, rows=0: lib.g2v_sig_fit(
        p, G, n, n_pad, p, p, K, F, p, S, pp, p, p, p, p, rows, st)
    auc = lambda n=100, K=2, F=5, S=1, cap=20: lib.g2v_sig_auc(p, p, p, n, K, F, S, cap, p, p, st)
    bad = [lib.g2v_sig_folds(p, 2, 1, 2, 0, p, st), lib.g2v_sig_folds(p, 100, 0, 2, 0, p, st),
           lib.g2v_sig_folds(p, 100, 101, 2, 0, p, st), lib.g2v_sig_folds(p, 100, 1, 1, 0, p, st),
           lib.g2v_sig_folds(p, 100, 1, 51, 0, p, st), lib.g2v_sig_folds(p, 32769, 1, 2, 0, p, st),
           lib.g2v_sig_draw(10, 0, 0, 1, 1, p, st), lib.g2v_sig_draw(10, 11, 0, 1, 1, p, st),
           lib.g2v_sig_draw(200, 129, 0, 1, 1, p, st), lib.g2v_sig_draw(10, 5, 0, 0, 1, p, st),
           lib.g2v_sig_draw(10, 5, 0, 65536, 2, p, st), lib.g2v_sig_draw(10, 5, 0, 1, 0, p, st),
           fit(n=2), fit(K=0), fit(K=101), fit(F=1), fit(F=101), fit(S=0), fit(pp=0), fit(pp=129, G=200),
           fit(pp=51), fit(n_pad=99), fit(rows=2), fit(S=(1 << 24) // 10 + 1, K=2, F=5),
           lib.g2v_sig_fit(None, 50, 100, 128, p, p, 2, 5, p, 1, 10, p, p, p, p, 0, st),
           lib.g2v_sig_fit(p, 50, 100, 128, p, p, 2, 5, p, 1, 10, p, p, p, None, 1, st),
           auc(cap=1), auc(cap=101), auc(n=2), auc(S=0), auc(F=1)]
    assert all(rc != 0 for rc in bad)
    assert int(lib.g2v_sig_fit_smem_bytes(0)) == 0 and int(lib.g2v_sig_fit_smem_bytes(129)) == 0
    assert capi.launch_count() == before and len(lib.g2v_last_error()) > 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------- CLI
def test_command_line_writes_the_signature_file_and_leaves_the_other_files_alone(tmp_path, capsys):
    from g2vec_b200 import cli
    from tests import helpers
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    base = ["-r", "2", "-e", "5", "-n", "20", "--seed", "3", "--deterministic"]
    a, b = str(tmp_path / "plain"), str(tmp_path / "sig")
    cli.main([ef, cf, nf, a] + base)
    log_a = capsys.readouterr().out
    cli.main([ef, cf, nf, b] + base + ["--signature-cv", "20", "--signature-repeats", "2"])
    log_b = capsys.readouterr().out
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt"):
        assert open(a + suffix).read() == open(b + suffix).read(), suffix
    assert not os.path.exists(a + "_signature.txt")
    import re
    untimed = lambda log, prefix: [re.sub(r" \([0-9.]+ sec\)$", "", l).replace(prefix, "RES")
                                   for l in log.splitlines()]
    extra = [l for l in untimed(log_b, b) if l not in untimed(log_a, a)]
    assert len(extra) == 3 and extra[0].startswith("Namespace(") and "signature_cv=20" in extra[0]
    assert extra[1].startswith("    signature CV: 5-fold x 2 repeats, ") and extra[2] == "    RES_signature.txt"
    data = cli.load_data(ef)
    data["label"] = cli.match_labels(cli.load_clinical(cf), data["sample"])
    data, _ = cli.restrict(data, cli.load_network(nf))
    bm = open(b + "_biomarkers.txt").read().split()[1:]
    g = list(data["gene"])
    r = signature_cv(data["expr"], data["label"], np.array([g.index(x) for x in bm]), 20, folds=5, repeats=2, seed=3)
    assert extra[1] == "    " + signature.summary(r)
    rows = open(b + "_signature.txt").read().splitlines()
    assert rows[0] == "Signature\tSize\tAUC\tAUC_SD\tAccuracy\tP_random\tBiomarkers" and len(rows) == 23
    assert rows[1] == "biomarkers\t%d\t%.6f\t%.6f\t%.6f\t%.6g\t%d" % (len(bm), r.auc_mean[0], r.auc_sd[0], r.acc_mean[0],
                                                                     r.p_random[0], len(bm))
    assert rows[3].startswith("random_1\t%d\t" % len(bm)) and rows[3].split("\t")[5] == "nan"
