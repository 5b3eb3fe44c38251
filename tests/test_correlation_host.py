"""CPU side of the Spearman / bicor edge weights (DESIGN.md §4.22): the NumPy host path (graph.corr_transform,
graph.edge_abs_corr, graph.group_csr) against the float64 oracle on random cohorts and gadgets, `pearson` as today's
path, and which values --correlation, --min-corr and the expression data are accepted with."""
import os

import numpy as np
import pytest
from scipy import stats

from g2vec_b200 import cli, graph
from tests import corr_oracle as co

METHODS = ("spearman", "bicor")


def _z_ok(got, want, method):
    if method == "spearman":                 # every sum of the rank transform is exact: the same bits
        assert (got == want.astype(np.float32)).all()
    else:
        assert np.abs(got.astype(np.float64) - want).max() <= 4 * co.U * max(1.0, np.abs(want).max())


def _pairs(V):
    a, b = np.triu_indices(V, 1)
    return a.astype(np.int32), b.astype(np.int32)


def cohort(S, V, seed, kind="normal"):
    rs = np.random.RandomState(seed)
    if kind == "normal":
        X = rs.randn(S, V)
    elif kind == "heavy":                    # heavy tails and many ties, as in expression data
        X = np.round(rs.standard_t(2, size=(S, V)) * 4) / 4
    else:                                    # correlated pairs so that some edges pass a cutoff
        base = rs.randn(S, (V + 1) // 2)
        X = np.repeat(base, 2, axis=1)[:, :V] + 0.6 * rs.randn(S, V)
    return X.astype(np.float32)


def gadgets():
    """Named [S, V] blocks that hit the transforms' special cases."""
    out = {}
    rs = np.random.RandomState(7)
    for S in (1, 2, 3, 4, 5, 8):
        out["small%d" % S] = rs.randn(S, 4).astype(np.float32)
    c = np.zeros((9, 4), np.float32)
    c[:, 0] = 3.0                                          # constant gene: weight 0
    c[:, 1] = [0, 1, 0, 1, 0, 1, 0, 1, 1]                  # two-valued
    c[:, 2] = [2, 2, 2, 2, 5, 2, 2, 7, 2]                  # mad = 0 with spread: bicor's Pearson fallback
    c[:, 3] = np.arange(9)
    out["ties"] = c
    z = np.array([[-0.0, 0.0, 1.0, -1.0, -0.0, 2.0, 0.0, 3.0]], np.float32).T
    plus = np.where(z == 0, np.float32(0.0), z)            # the same values with every zero +0.0
    assert np.signbit(z).sum() > np.signbit(plus).sum()
    out["signed_zero"] = np.concatenate([z, plus, rs.randn(8, 1).astype(np.float32)], axis=1)
    o = rs.randn(12, 3).astype(np.float32)
    o[0, 0] = 1e4                                          # far beyond 9 mad: a_i = 0
    m = co.mad(o[:, 1]); med = np.median(o[:, 1].astype(np.float64))
    o[1, 1] = np.float32(med + 9.0 * m)                    # at about 9 mad
    out["outliers"] = o
    h = np.zeros((10, 3), np.float32)
    h[:6, 0] = 1.0; h[6:, 0] = [4, 5, 6, 7]                # more than half equal, S even
    h[:, 1] = [1, 1, 1, 1, 1, 2, 2, 2, 2, 2]               # exactly half: mad > 0
    h[:, 2] = rs.randn(10)
    out["halves"] = h
    return out


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("S,V,seed,kind", [(7, 12, 0, "normal"), (40, 30, 1, "heavy"), (61, 24, 2, "pairs"),
                                           (128, 16, 3, "heavy"), (33, 10, 4, "normal")])
def test_host_transform_and_weights_match_oracle(method, S, V, seed, kind):
    X = cohort(S, V, seed, kind)
    Z = graph.corr_transform(X, method)
    _z_ok(Z, co.transform(X, method), method)
    a, b = _pairs(V)
    w = graph.edge_abs_corr(X, a, b, method)
    assert np.abs(w - co.weights(X, a, b, method)).max() <= co.EDGE_TOL


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name", sorted(gadgets()))
def test_host_gadgets(method, name):
    X = gadgets()[name]
    Z = graph.corr_transform(X, method)
    _z_ok(Z, co.transform(X, method), method)
    a, b = _pairs(X.shape[1])
    w = graph.edge_abs_corr(X, a, b, method)
    want = co.weights(X, a, b, method)
    assert np.abs(w - want).max() <= co.EDGE_TOL
    for v in range(X.shape[1]):
        if np.all(X[:, v] == X[0, v]):                     # constant gene: z = 0, every weight 0
            assert (Z[:, v] == 0).all()
            assert (w[(a == v) | (b == v)] == 0).all()


def test_oracle_spearman_is_scipy():
    X = cohort(50, 6, 11, "heavy")
    Z = co.transform(X, "spearman")
    for a in range(6):
        for b in range(a + 1, 6):
            rho = stats.spearmanr(X[:, a], X[:, b]).correlation
            assert abs(co.edge_weights(Z, [a], [b])[0] - abs(rho)) < 1e-12


def test_signed_zero_ties():
    X = gadgets()["signed_zero"]
    Z = graph.corr_transform(X, "spearman")
    assert (Z[:, 0] == Z[:, 1]).all()                      # -0.0 and +0.0 are one value
    assert graph.edge_abs_corr(X, [0], [1], "spearman")[0] == np.float32(1.0)


def test_bicor_fallback_and_rejection():
    X = gadgets()["ties"]
    assert co.mad(X[:, 2]) == 0 and co.mad(X[:, 3]) > 0
    Z = graph.corr_transform(X, "bicor")
    assert np.abs(Z[:, 2] - co.pearson_z(X[:, 2])).max() < 1e-6
    o = gadgets()["outliers"]
    Zo = graph.corr_transform(o, "bicor")
    assert Zo[0, 0] == 0                                   # beyond 9 mad: weight 0 in the biweight
    for Zg in (Z, Zo):
        ok = np.abs(Zg).sum(axis=0) > 0
        assert np.allclose((Zg[:, ok].astype(np.float64) ** 2).mean(axis=0), 1.0, atol=1e-6)


@pytest.mark.parametrize("method", METHODS)
def test_invariances_host(method):
    rs = np.random.RandomState(5)
    X = cohort(45, 8, 6, "heavy")
    a, b = _pairs(8)
    w = graph.edge_abs_corr(X, a, b, method)
    assert (graph.edge_abs_corr(-X, a, b, method) == w).all()
    if method == "bicor":
        assert (graph.edge_abs_corr(X * np.float32(8), a, b, method) == w).all()
    else:
        Y = X.copy()
        for v in range(8):                                 # order-preserving relabelling per gene
            u, inv = np.unique(Y[:, v], return_inverse=True)
            Y[:, v] = np.sort(rs.uniform(-1e3, 1e3, size=len(u))).astype(np.float32)[inv.ravel()]
            assert len(np.unique(Y[:, v])) == len(u)
        assert (graph.edge_abs_corr(Y, a, b, method) == w).all()


def test_pearson_is_todays_path(golden_dir):
    for name in ("pcc_small.npz", "ex_expr.npz"):
        z = np.load(os.path.join(golden_dir, name))
        if name == "ex_expr.npz":
            label = np.load(os.path.join(golden_dir, "ex_graph.npz"))["label"]
        else:
            label = z["label"]
        src, dst = z["src"].astype(np.int32), z["dst"].astype(np.int32)
        for g in (0, 1):
            X = z["expr"][label == g]
            assert (graph.edge_abs_corr(X, src, dst) == graph.edge_abs_pcc(X, src, dst)).all()
            old = graph.group_csr(z["expr"], label, g, src, dst)
            new = graph.group_csr(z["expr"], label, g, src, dst, threshold=0.5, method="pearson")
            for u, v in zip(old, new):
                assert u.dtype == v.dtype and (u == v).all()


@pytest.mark.parametrize("T", [0.0, 0.3, 0.5, 0.9])
@pytest.mark.parametrize("method", METHODS)
def test_host_csr_against_oracle(method, T):
    X = cohort(60, 40, 9, "pairs")
    label = np.zeros(60, np.int64)
    a, b = _pairs(40)
    rp, col, w = graph.group_csr(X, label, 0, a, b, threshold=T, method=method)
    want = co.weights(X, a, b, method)
    got = {(int(s), int(d)) for s, d in zip(np.repeat(np.arange(40), np.diff(rp)), col)}
    ref = {(int(s), int(d)) for s, d, x in zip(a, b, want) if x > T}
    for k in got ^ ref:
        assert abs(want[(a == k[0]) & (b == k[1])][0] - T) <= co.EDGE_TOL
    assert (w > T).all()


def test_graph_refusals():
    X = cohort(10, 4, 0)
    label = np.zeros(10, np.int64)
    a, b = _pairs(4)
    for bad in ("kendall", "Pearson", None):
        with pytest.raises(ValueError):
            graph.group_csr(X, label, 0, a, b, method=bad)
        with pytest.raises(ValueError):
            graph.group_csr_gpu(X, label, 0, a, b, method=bad)
    for T in (-0.1, 1.0, 1.5, float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError):
            graph.group_csr(X, label, 0, a, b, threshold=T)
        with pytest.raises(ValueError):
            graph.group_csr_gpu(X, label, 0, a, b, threshold=T, method="spearman")
    for v in (np.nan, np.inf, -np.inf):
        Y = X.copy(); Y[3, 2] = v
        for m in METHODS:
            with pytest.raises(ValueError, match="finite"):
                graph.group_csr(Y, label, 0, a, b, method=m)
            with pytest.raises(ValueError, match="finite"):            # before anything is uploaded
                graph.group_csr_gpu(Y, label, 0, a, b, method=m)
    big = np.zeros((graph.CORR_MAX_SAMPLES + 1, 2), np.float32)
    with pytest.raises(ValueError, match="at most"):
        graph.group_csr_gpu(big, np.zeros(len(big)), 0, [0], [1], method="bicor")


def _args(*extra):
    return cli.parse_arguments(["E", "C", "N", "R"] + list(extra))


def test_cli_accepts():
    a = _args()
    assert a.correlation == "pearson" and a.min_corr == 0.5
    for m in ("pearson", "spearman", "bicor"):
        assert _args("--correlation", m).correlation == m
    for t in ("0", "0.3", "0.999", "0.5"):
        assert _args("--min-corr", t).min_corr == float(t)


@pytest.mark.parametrize("extra", [["--correlation", "kendall"], ["--correlation", "Pearson"], ["--min-corr", "-0.1"],
                                   ["--min-corr", "1"], ["--min-corr", "nan"], ["--min-corr", "inf"],
                                   ["--min-corr", "-inf"], ["--min-corr", "x"]])
def test_cli_refuses(extra, capsys):
    with pytest.raises(SystemExit) as e:
        _args(*extra)
    assert e.value.code == 2
    err = capsys.readouterr().err
    assert ("--min-corr" in err) or ("--correlation" in err)
