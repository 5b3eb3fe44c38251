"""CPU checks of the exact t-SNE map (DESIGN.md §4.27): the oracle of tests/tsne_oracle.py against plain Python float
arithmetic and against scikit-learn (_binary_search_perplexity, _kl_divergence's gradient, PCA); the stage switch at
iteration 250; the PCA initialisation and its fallback; every refusal of tsne_map, affinities and optimize (raised
before the library is loaded), the --tsne option and the _tsne.txt writer."""
import numpy as np
import pytest

from g2vec_b200 import cli, tsne
from tests import tsne_oracle


def _python_dist(x, y):
    acc = 0.0
    for a, b in zip(x, y):
        t = float(a) - float(b)
        acc = acc + t * t
    return acc


@pytest.mark.parametrize("m,D,seed", [(2, 1, 0), (5, 7, 1), (9, 40, 2)])
def test_distance_chain_equals_python_floats(m, D, seed):
    rs = np.random.RandomState(seed)
    X = (rs.standard_normal((m, D)) * np.exp2(rs.randint(-20, 20, size=(m, 1)))).astype(np.float32).astype(np.float64)
    d = tsne_oracle.dist(X)
    for i in range(m):
        for j in range(m):
            assert d[i, j] == _python_dist(X[i], X[j])
    assert (d.view(np.int64) == d.T.view(np.int64)).all() and (np.diag(d) == 0).all()


def _python_iteration_parts(P, Y):
    """Per row: the chains of w, p w t_c and w^2 t_c over j != i in blocks of BLOCK columns, the block partials
    chained; Z = the chain of Z_i in blocks of BLOCK rows, then over the blocks."""
    m = len(Y)
    B = tsne.BLOCK
    rows = []
    for i in range(m):
        tot = [0.0] * 5
        for b0 in range(0, m, B):
            part = [0.0] * 5
            for j in range(b0, min(m, b0 + B)):
                if j == i:
                    continue
                t0 = float(Y[i][0]) - float(Y[j][0])
                t1 = float(Y[i][1]) - float(Y[j][1])
                w = 1.0 / (1.0 + (t0 * t0 + t1 * t1))
                a = float(P[i][j]) * w
                r = w * w
                part = [part[0] + w, part[1] + a * t0, part[2] + a * t1, part[3] + r * t0, part[4] + r * t1]
            tot = [x + y for x, y in zip(tot, part)]
        rows.append(tot)
    Z = 0.0
    for b0 in range(0, m, B):
        zb = 0.0
        for i in range(b0, min(m, b0 + B)):
            zb = zb + rows[i][0]
        Z = Z + zb
    return rows, Z


def _random_P(m, rs):
    c = rs.random_sample((m, m))
    np.fill_diagonal(c, 0.0)
    c /= c.sum(axis=1, keepdims=True)
    return tsne_oracle.joint(c)


@pytest.mark.parametrize("m", [2, 3, 17, tsne.BLOCK + 3])
def test_iteration_chains_equal_python_floats(m):
    rs = np.random.RandomState(m)
    P = _random_P(m, rs)
    Y = rs.standard_normal((m, 2)) * 3.0
    rows, Z = _python_iteration_parts(P, Y)
    for alpha in (12.0, 1.0):
        g, Zo = tsne_oracle.gradient(P, Y, alpha)
        assert Zo == Z
        for i in range(m):
            for c in range(2):
                want = 4.0 * ((alpha * rows[i][1 + c]) - (rows[i][3 + c] / Z))
                assert g[i, c] == want, (i, c)
    u = rs.standard_normal((m, 2))
    gains = rs.random_sample((m, 2)) * 2
    gains[0, 0] = 0.011                                       # * 0.8 falls below the 0.01 floor
    g, _ = tsne_oracle.gradient(P, Y, 1.0)
    u[0, 0] = g[0, 0]                                         # same sign: the gain shrinks
    Y1, u1, gains1 = tsne_oracle.step(g, Y, u, gains, 400, 55.5)
    for i in range(m):
        for c in range(2):
            gi, ui, gain = float(g[i, c]), float(u[i, c]), float(gains[i, c])
            gain = gain + 0.2 if ui * gi < 0.0 else gain * 0.8
            gain = max(gain, 0.01)
            gi = gi * gain
            ui = 0.8 * ui - 55.5 * gi
            assert gains1[i, c] == gain and u1[i, c] == ui and Y1[i, c] == float(Y[i, c]) + ui
    assert gains1[0, 0] == 0.01


# --------------------------------------------------------------------------------- against scikit-learn
@pytest.mark.parametrize("seed,m,D,perplexity", [(0, 60, 5, 5.0), (1, 200, 16, 30.0), (2, 300, 3, 2.5),
                                                 (3, 40, 8, 10.0)])
def test_conditional_affinities_equal_scikit_learn(seed, m, D, perplexity):
    """On distances exact in float32 and perplexities exact in float32 (scikit-learn takes both as float32); no row of
    these seeded inputs has an entropy within rounding of the tolerance.  scikit-learn does not return beta: it is
    recovered from its P, where any other beta the bisection could reach would move P far beyond 1e-12."""
    from sklearn.manifold import _utils
    rs = np.random.RandomState(seed)
    X = rs.standard_normal((m, D)).astype(np.float32).astype(np.float64)
    d = tsne_oracle.dist(X).astype(np.float32).astype(np.float64)
    c, beta, steps = tsne_oracle.conditional(d, perplexity)
    sk = _utils._binary_search_perplexity(d.astype(np.float32), np.float32(perplexity), 0)
    assert (steps < tsne.MAX_STEPS).all()
    np.testing.assert_allclose(c, sk, rtol=1e-12, atol=0)
    for i in range(m):
        j = [k for k in np.argsort(d[i]) if k != i and sk[i, k] > 1e-300]      # normal, not underflowed
        lo, hi = j[0], j[-1]
        est = np.log(sk[i, lo] / sk[i, hi]) / (d[i, hi] - d[i, lo])
        assert abs(est / beta[i] - 1.0) < 1e-9
        assert abs(tsne_oracle.entropy(d, beta)[i] - np.log(perplexity)) <= tsne.TOLERANCE


def test_unconverged_rows_report_100_steps_and_their_last_beta():
    d = np.full((4, 4), 1e60)                                 # every exp underflows: the sum is floored, beta halves
    np.fill_diagonal(d, 0.0)
    c, beta, steps = tsne_oracle.conditional(d, 2.0)
    assert (steps == tsne.MAX_STEPS).all() and (beta == 2.0 ** -99).all() and (c == 0).all()


def test_joint_affinities_are_symmetric_and_sum_to_one():
    rs = np.random.RandomState(4)
    X = rs.standard_normal((50, 6))
    c, _, _ = tsne_oracle.conditional(tsne_oracle.dist(X), 10.0)
    P = tsne_oracle.joint(c)
    assert (P.view(np.int64) == P.T.view(np.int64)).all() and (np.diag(P) == 0).all()
    assert abs(P.sum() - 1.0) < 1e-12


@pytest.mark.parametrize("m", [5, 40, 300])
def test_gradient_equals_scikit_learn_kl_divergence(m):
    """scikit-learn's gradient is 4 sum_j (p_ij - q_ij) w_ij (y_i - y_j) with P multiplied by the exaggeration and Q
    clamped at eps; the two differ by rounding only."""
    from scipy.spatial.distance import squareform
    from sklearn.manifold._t_sne import _kl_divergence
    rs = np.random.RandomState(m)
    X = rs.standard_normal((m, 4))
    c, _, _ = tsne_oracle.conditional(tsne_oracle.dist(X), min(30.0, m / 3.0))
    P = tsne_oracle.joint(c)
    Y = rs.standard_normal((m, 2)) * 0.5
    for alpha in (12.0, 1.0):
        g, _ = tsne_oracle.gradient(P, Y, alpha)
        kl, sk = _kl_divergence(Y.ravel().copy(), squareform(P * alpha, checks=False), 1, m, 2)
        sk = sk.reshape(m, 2)
        assert np.abs(g - sk).max() <= 1e-10 * np.abs(sk).max()
        if alpha == 1.0:
            assert abs(tsne_oracle.kl(P, Y) - kl) <= 1e-10 * abs(kl)


def test_stage_switch_at_250_resets_u_and_the_gains():
    rs = np.random.RandomState(5)
    m = 7
    g, Y = rs.standard_normal((m, 2)), rs.standard_normal((m, 2))
    u, gains = rs.standard_normal((m, 2)), rs.random_sample((m, 2)) + 0.5
    assert tsne_oracle.stage(0) == (12.0, 0.5, True) and tsne_oracle.stage(249) == (12.0, 0.5, False)
    assert tsne_oracle.stage(250) == (1.0, 0.8, True) and tsne_oracle.stage(251) == (1.0, 0.8, False)
    fresh = tsne_oracle.step(g, Y, np.zeros((m, 2)), np.ones((m, 2)), 251, 50.0)
    reset = tsne_oracle.step(g, Y, u, gains, 250, 50.0)
    for a, b in zip(fresh, reset):
        assert (a == b).all()
    kept = tsne_oracle.step(g, Y, u, gains, 249, 50.0)
    assert (kept[1] == 0.5 * u - 50.0 * (g * kept[2])).all()
    # the whole run: 251 iterations = 250 exaggerated ones, then one from u = 0 and gains = 1 with alpha = 1
    P = _random_P(m, rs)
    Y250, _ = tsne_oracle.optimize(P, Y, 250)
    Y251, _ = tsne_oracle.optimize(P, Y, 251)
    g250, _ = tsne_oracle.gradient(P, Y250, 1.0)
    want = tsne_oracle.step(g250, Y250, None, None, 250, tsne.learning_rate(m))[0]
    assert (Y251 == want).all()


def test_learning_rate_is_scikit_learn_auto():
    """TSNE._fit's learning_rate="auto": X.shape[0] / self.early_exaggeration / 4, then np.maximum(..., 50)."""
    for m in (2, 600, 601, 3769, 20000, 32768):
        assert tsne.learning_rate(m) == float(np.maximum(m / 12.0 / 4, 50))
    assert tsne.learning_rate(600) == 50.0 and tsne.learning_rate(3769) == 3769 / 48.0


# ---------------------------------------------------------------------------------------------- PCA init
def test_pca_init_equals_scikit_learn_pca():
    from sklearn.decomposition import PCA
    rs = np.random.RandomState(6)
    W = (rs.standard_normal((300, 12)) * np.arange(1, 13)).astype(np.float32)
    Y0 = tsne.pca_init(W)
    X = W.astype(np.float64)
    sk = PCA(n_components=2, svd_solver="full").fit_transform(X)
    sk = sk / np.std(sk[:, 0]) * 1e-4
    np.testing.assert_allclose(Y0, sk, rtol=1e-8, atol=1e-16)
    assert Y0.dtype == np.float64 and abs(np.std(Y0[:, 0]) - 1e-4) < 1e-18
    V = np.linalg.svd(X - X.mean(axis=0), full_matrices=False)[2][:2]
    for k in range(2):
        comp = np.linalg.lstsq(X - X.mean(axis=0), Y0[:, k], rcond=None)[0]
        assert comp[np.argmax(np.abs(comp))] > 0 and abs(abs(comp @ V[k]) / np.linalg.norm(comp) - 1) < 1e-9
    assert (tsne.pca_init(W, seed=3) == Y0).all()


def test_pca_init_falls_back_to_the_seeded_random_init():
    for W in (np.tile(np.float32([[1.5, -2.0, 3.0]]), (10, 1)), np.arange(8, dtype=np.float32)[:, None]):
        want = np.random.default_rng(7).standard_normal((W.shape[0], 2)) * 1e-4
        assert (tsne.pca_init(W, seed=7) == want).all()


# ---------------------------------------------------------------------------------------------- refusals
def _no_library(monkeypatch):
    from g2vec_b200 import _capi

    def boom():
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(_capi, "load", boom)


@pytest.mark.parametrize("case", ["1d", "3d", "m1", "m_max", "D0", "nan", "inf", "f32_overflow", "perp_lt1",
                                  "perp_eq_m", "perp_nan", "perp_inf", "perp_str", "perp_bool", "iter0", "iter_float",
                                  "init_str", "init_shape", "init_nan"])
def test_refusals_raise_before_the_library_is_loaded(case, monkeypatch):
    _no_library(monkeypatch)
    W = np.random.RandomState(0).standard_normal((20, 8)).astype(np.float32)
    kw = {"perplexity": 5.0}
    if case == "1d":
        W = W[0]
    elif case == "3d":
        W = W.reshape(4, 5, 8)
    elif case == "m1":
        W = W[:1]
        kw["perplexity"] = 1.0
    elif case == "m_max":
        W = np.zeros((tsne.MAX_GENES + 1, 1), np.float32)
    elif case == "D0":
        W = W[:, :0]
    elif case == "nan":
        W[3, 2] = np.nan
    elif case == "inf":
        W[3, 2] = -np.inf
    elif case == "f32_overflow":
        W = W.astype(np.float64); W[0, 0] = 1e300
    elif case == "perp_lt1":
        kw["perplexity"] = 0.999
    elif case == "perp_eq_m":
        kw["perplexity"] = 20
    elif case == "perp_nan":
        kw["perplexity"] = float("nan")
    elif case == "perp_inf":
        kw["perplexity"] = float("inf")
    elif case == "perp_str":
        kw["perplexity"] = "5"
    elif case == "perp_bool":
        kw["perplexity"] = True
    elif case == "iter0":
        kw["n_iter"] = 0
    elif case == "iter_float":
        kw["n_iter"] = 10.0
    elif case == "init_str":
        kw["init"] = "random"
    elif case == "init_shape":
        kw["init"] = np.zeros((20, 3))
    else:
        kw["init"] = np.full((20, 2), np.nan)
    with pytest.raises(ValueError):
        tsne.tsne_map(W, **kw)
    if "init" not in kw and "n_iter" not in kw:
        with pytest.raises(ValueError):
            tsne.affinities(W, kw["perplexity"])


@pytest.mark.parametrize("case", ["not_square", "too_small", "nan", "y0_shape", "y0_inf", "iter0"])
def test_optimize_refusals_raise_before_the_library_is_loaded(case, monkeypatch):
    _no_library(monkeypatch)
    P, Y0, n = np.full((4, 4), 1 / 12.0), np.zeros((4, 2)), 3
    if case == "not_square":
        P = P[:3]
    elif case == "too_small":
        P, Y0 = P[:1, :1], Y0[:1]
    elif case == "nan":
        P[1, 2] = np.nan
    elif case == "y0_shape":
        Y0 = Y0[:3]
    elif case == "y0_inf":
        Y0[0, 1] = np.inf
    else:
        n = 0
    with pytest.raises(ValueError):
        tsne.optimize(P, Y0, n)


def test_admitted_inputs():
    W, init = tsne.check_inputs(np.ones((2, 1)), 1.0)
    assert W.dtype == np.float32 and W.shape == (2, 1) and init == "pca"
    tsne.check_inputs(np.zeros((3, 2), np.float32), np.float32(2.5), np.int64(1), np.zeros((3, 2), np.float32))
    tsne.check_inputs(np.zeros((tsne.MAX_GENES, 1), np.float32), 30)


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        tsne.tsne_map(np.random.RandomState(0).standard_normal((6, 2)).astype(np.float32), 2.0, n_iter=1)


# ----------------------------------------------------------------------------------------- command line
def test_tsne_option():
    a = cli.parse_arguments(["E", "C", "N", "R"])
    assert a.tsne == 0 and "tsne=0" in repr(a)
    assert cli.parse_arguments(["E", "C", "N", "R", "--tsne", "30"]).tsne == 30.0
    assert cli.parse_arguments(["E", "C", "N", "R", "--tsne", "1"]).tsne == 1.0
    assert cli.parse_arguments(["E", "C", "N", "R", "--tsne", "1000"]).tsne == 1000.0
    assert cli.parse_arguments(["E", "C", "N", "R", "--tsne", "7.5"]).tsne == 7.5
    for bad in ("-1", "0.5", "1000.5", "nan", "inf", "x"):
        with pytest.raises(SystemExit):
            cli.parse_arguments(["E", "C", "N", "R", "--tsne", bad])


def test_tsne_writer_format(tmp_path):
    p = str(tmp_path / "res")
    genes = np.array(["A1CF", "AAK1", "ABL1", "ACTB"])
    lgroup = np.array([1, 2, 2, 0], np.int32)
    Y = np.array([[1.0, -2.5], [3.1234567, 0.0], [-1e-7, 12345.6789]])
    cli.write_tsne(p, genes, lgroup, np.array([0, 1, 3]), Y)
    assert open(p + "_tsne.txt").read() == (
        "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tX\tY\n"
        "A1CF\t1\t1.000000\t-2.500000\n"
        "AAK1\t2\t3.123457\t0.000000\n"
        "ACTB\t0\t-0.000000\t12345.678900\n")


def test_summary_line():
    assert tsne.summary(3769, 30.0, 1000, 1.23456789) == \
        "t-SNE: 2-D map of 3769 genes in paths, perplexity 30, 1000 iterations: KL divergence 1.234568"
