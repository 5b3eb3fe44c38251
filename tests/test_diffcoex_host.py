"""Host side of the differential co-expression test (g2vec_b200/diffcoex.py, DESIGN.md §4.30) and its NumPy
restatement (tests/diffcoex_oracle.py): no GPU needed."""
import os

import numpy as np
import pytest

from g2vec_b200 import diffcoex, perm
from tests import diffcoex_oracle
from tests.test_perm_host import cohort


def _obs(x, lab, pairs):
    prep = diffcoex.prepare(x, lab, pairs)
    return prep, diffcoex.observed(prep, *diffcoex_oracle.observed_sums(prep))


def _random_pairs(rs, G, E):
    return diffcoex.pairs_from_edges(rs.randint(0, G, E), rs.randint(0, G, E))


# ------------------------------------------------------------------------------------------------ statistics
def test_oracle_r_matches_corrcoef_and_z_the_fisher_formula():
    rs = np.random.RandomState(1)
    x, lab = cohort(135, 60, 2, 77)
    x[:, 5] = x[:, 6] * 2.0 + 0.1 * rs.standard_normal(135)
    pairs = _random_pairs(rs, 60, 400)
    prep, (rg, rp, D) = _obs(x, lab, pairs)
    for grp, r in ((0, rg), (1, rp)):
        c = np.corrcoef(x[lab == grp].T)
        assert np.abs(r - c[pairs[:, 0], pairs[:, 1]]).max() < 1e-4
    res = diffcoex.finish(prep, rg, rp, D, np.argsort(-D, kind="stable"), np.zeros(len(D)), np.zeros(len(D)), 1)
    z = (np.arctanh(rp) - np.arctanh(rg)) / np.sqrt(1.0 / (77 - 3) + 1.0 / (58 - 3))
    assert np.allclose(res.Z, z, rtol=1e-12, atol=0)
    # D orders the pairs exactly as |Z| does
    assert (np.argsort(-D, kind="stable") == np.argsort(-np.abs(res.Z), kind="stable")).all()
    assert np.allclose(D, np.tanh(np.abs(np.arctanh(rp) - np.arctanh(rg))), rtol=1e-12, atol=1e-15)


def test_constant_genes_and_perfect_correlation_rules():
    x, lab = cohort(32, 8, 3, 16)                       # integer values over 32 samples: every mean is dyadic, so
    rs = np.random.RandomState(3)                       # the quantisation of these genes is exact and affine
    x[:, 2:6] = rs.randint(-50, 51, size=(32, 4))
    x[:, 1] = 5.0                                       # constant: r = 0 in both groups
    x[:, 2] = 3.0 * x[:, 3] - 1.0                       # r = 1 in both groups: D = 0, Z = 0
    x[:, 4] = np.where(lab == 0, x[:, 5], -x[:, 5])     # r = 1 in the good samples, -1 in the poor: D = 1
    x[lab == 1, 6] = 7.0                                # constant in the poor group only
    pairs = np.array([[0, 1], [2, 3], [4, 5], [6, 7]], np.int32)
    prep, (rg, rp, D) = _obs(x, lab, pairs)
    assert rg[0] == rp[0] == 0.0 and D[0] == 0.0
    assert rg[1] == rp[1] == 1.0 and D[1] == 0.0
    assert rg[2] == 1.0 and rp[2] == -1.0 and D[2] == 1.0
    assert rp[3] == 0.0 and D[3] == abs(rg[3])
    z = diffcoex.z_of(rg, rp, 16, 16)
    assert z[0] == 0.0 and z[1] == 0.0 and z[2] == -np.inf
    assert ((-1.0 <= rg) & (rg <= 1.0)).all() and ((0.0 <= D) & (D <= 1.0)).all()


def test_int64_bounds_hold_at_the_extremes():
    """|q| = 2^16 at n = 32768: C, V and every product of them equal Python's integers (no wrap)."""
    n, v = 32768, 1 << 16
    rs = np.random.RandomState(4)
    for k in (4, n // 2, n - 4, n):
        qi = np.where(rs.rand(n) < 0.5, v, -v).astype(np.int64)
        qj = np.full(n, -v, np.int64)
        for a, b in ((qi, qj), (qj, qj), (np.full(n, v, np.int64), qj)):
            s = slice(0, k)
            P, Ai, Aj, Bi, Bj = (int((a[s] * b[s]).sum()), int(a[s].sum()), int(b[s].sum()), int((a[s] ** 2).sum()),
                                 int((b[s] ** 2).sum()))
            C, Vi, Vj = k * P - Ai * Aj, k * Bi - Ai * Ai, k * Bj - Aj * Aj
            assert max(abs(k * P), abs(Ai * Aj), abs(C), Vi, Vj, k * Bi) <= 1 << 62
            assert abs(P) <= 1 << 47 and Bi <= 1 << 47
            want = 0.0 if Vi == 0 or Vj == 0 else max(-1.0, min(1.0, float(C) / np.sqrt(float(Vi) * float(Vj))))
            got = diffcoex.corr_of(k, np.array([P]), np.array([Ai]), np.array([Aj]), np.array([Bi]), np.array([Bj]))
            assert got[0] == want
    M = np.ones((1, n), np.uint8)
    q = np.full((n, 2), v, np.int64); q[:, 1] = -v
    assert diffcoex_oracle.sums(M, q, np.array([0]), np.array([1]))[0, 0] == -n * v * v == -(1 << 47)


def test_quantise_default_is_unchanged_and_bits_sets_the_bound():
    x, _ = cohort(100, 50, 5)
    q22 = perm.quantise(x)
    assert (q22 == perm.quantise(x, bits=22)).all()
    m = np.abs(q22).max(axis=0)
    assert ((m >= 1 << 21) & (m <= 1 << 22)).all()
    q16 = perm.quantise(x, bits=diffcoex.Q_BITS)
    m = np.abs(q16).max(axis=0)
    assert ((m >= 1 << 15) & (m <= 1 << 16)).all()


# ------------------------------------------------------------------------------------------------------ counts
def test_fast_step_down_equals_the_naive_one():
    rs = np.random.RandomState(6)
    E, B = 40, 25
    D_obs = rs.rand(E); D_obs[3] = D_obs[7] = D_obs[11]            # ties
    Dp = rs.rand(B, E) * 1.2
    Dp[2, 5] = D_obs[5]                                 # D_b = D_obs counts
    o = np.argsort(-D_obs, kind="stable")
    c, cm = diffcoex_oracle.tally(Dp[:, o], D_obs[o])
    assert (cm == diffcoex_oracle.maxt_counts_naive(Dp, D_obs)).all()
    assert (c == (Dp[:, o] >= D_obs[o][None, :]).sum(axis=0)).all()


def test_oracle_in_any_chunking_and_a_planted_pair():
    x, lab = cohort(30, 12, 7, 14)
    rs = np.random.RandomState(8)
    x[lab == 1, 3] = x[lab == 1, 4] * 2.0 + 0.01 * rs.standard_normal(16)     # correlated in the poor group only
    pairs = diffcoex.pairs_from_edges(*np.triu_indices(12, 1))
    a = diffcoex_oracle.diffcoex_test(x, lab, pairs, 60, seed=2)
    b = diffcoex_oracle.diffcoex_test(x, lab, pairs, 60, seed=2, chunk=7)
    for f in ("count", "count_maxt", "P", "P_maxT", "Q", "D", "Z"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    e = int(np.nonzero((pairs[:, 0] == 3) & (pairs[:, 1] == 4))[0][0])
    assert a.order[0] == e and a.P[e] == 1.0 / 61 and a.R_poor[e] > 0.99
    assert (a.P_maxT >= a.P).all() and (np.diff(a.P_maxT[a.order]) >= 0).all()


# ------------------------------------------------------------------------------------------------------- pairs
def test_pairs_from_the_example_network():
    from tests.helpers import GOLDEN
    e = np.load(os.path.join(GOLDEN, "ex_expr.npz"))
    p = diffcoex.pairs_from_edges(e["src"], e["dst"])
    assert len(e["src"]) == 216540 and p.shape == (140902, 2) and p.dtype == np.int32
    assert (p[:, 0] < p[:, 1]).all()
    key = p[:, 0].astype(np.int64) * 7523 + p[:, 1]
    assert (np.diff(key) > 0).all()


def test_pairs_collapse_duplicates_reversed_edges_and_self_loops():
    p = diffcoex.pairs_from_edges([3, 1, 2, 1, 5, 0, 2], [1, 3, 2, 3, 0, 5, 4])
    assert p.tolist() == [[0, 5], [1, 3], [2, 4]]
    assert diffcoex.pairs_from_edges([1], [1]).shape == (0, 2)


def test_graph_pairs_reads_either_direction():
    pairs = np.array([[0, 1], [0, 3], [1, 2], [2, 3]], np.int32)
    rowptr = np.array([0, 1, 1, 2, 3])                  # 0->1, 2->1, 3->0
    col = np.array([1, 1, 0])
    assert diffcoex.graph_pairs(pairs, 4, rowptr, col).tolist() == [1, 1, 1, 0]


# ---------------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("case", ["shape", "B0", "Bbig", "Bfloat", "n0", "n1", "nan", "nopairs", "pair_oob", "pair_rev",
                                  "pair_dup", "pair_unsorted", "pair_shape", "too_many_samples"])
def test_check_inputs_refuses(case):
    x, lab = cohort(20, 6, 9, 10)
    pairs, B = np.array([[0, 1], [2, 5]], np.int32), 10
    if case == "shape":
        lab = lab[:-1]
    elif case == "B0":
        B = 0
    elif case == "Bbig":
        B = (1 << 20) + 1
    elif case == "Bfloat":
        B = 2.5
    elif case == "n0":
        lab = np.array([1] * 17 + [0] * 3)
    elif case == "n1":
        lab = np.array([0] * 17 + [1] * 3)
    elif case == "nan":
        x[4, 2] = np.nan
    elif case == "nopairs":
        pairs = np.zeros((0, 2), np.int32)
    elif case == "pair_oob":
        pairs = np.array([[0, 6]])
    elif case == "pair_rev":
        pairs = np.array([[2, 1]])
    elif case == "pair_dup":
        pairs = np.array([[0, 1], [0, 1]])
    elif case == "pair_unsorted":
        pairs = np.array([[2, 3], [0, 1]])
    elif case == "pair_shape":
        pairs = np.array([0, 1])
    elif case == "too_many_samples":
        x, lab = np.zeros((32769, 2)), np.arange(32769) % 2
        pairs = np.array([[0, 1]])
    with pytest.raises(ValueError):
        diffcoex.check_inputs(x, lab, pairs, B)


def test_check_inputs_leaves_out_other_labels():
    x, lab = cohort(20, 6, 9, 10)
    lab[0] = 2
    x[0, 0] = np.nan                                    # in a left-out sample: ignored
    xx, ll, pp = diffcoex.check_inputs(x, lab, [[0, 1]], 5)
    assert xx.shape == (19, 6) and (ll != 2).all() and pp.dtype == np.int32
    with pytest.raises(ValueError):
        diffcoex.check_inputs(x, lab, [[0, 1]], 1 << 21)


# ---------------------------------------------------------------------------------------------- command line
def test_option_parsing():
    from g2vec_b200 import cli
    pos = ["E", "C", "N", "R"]
    assert cli.parse_arguments(pos).diff_coexpression == 0
    assert cli.parse_arguments(pos + ["--diff-coexpression", "200"]).diff_coexpression == 200
    assert cli.parse_arguments(pos + ["--diff-coexpression", str(1 << 20)]).diff_coexpression == 1 << 20
    for bad in ("-1", str((1 << 20) + 1), "1.5", "x"):
        with pytest.raises(SystemExit):
            cli.parse_arguments(pos + ["--diff-coexpression", bad])


def test_writer_format(tmp_path):
    from g2vec_b200 import cli
    genes = np.array(["A", "B", "C"])
    res = diffcoex.DiffCoexResult(pairs=np.array([[0, 1], [1, 2]], np.int32), R_good=np.array([0.5, -1.0]),
                                  R_poor=np.array([0.25, 1.0]), Z=np.array([-1.234567891, np.inf]), D=np.zeros(2),
                                  P=np.array([0.001, 1.0]), P_maxT=np.array([0.0123456789, 1.0]),
                                  Q=np.array([0.002, 1.0]), count=np.zeros(2), count_maxt=np.zeros(2),
                                  order=np.arange(2), n_perm=999)
    prefix = str(tmp_path / "out")
    cli.write_diffcoex(prefix, genes, res, np.array([1, 0]), np.array([0, 0]), np.array([2, 0]))
    assert open(prefix + "_diffcoex.txt").read().splitlines() == [
        "Gene1\tGene2\tR_good\tR_poor\tZ\tP\tP_maxT\tQ\tInGood\tInPoor\tBiomarkers",
        "A\tB\t0.500000\t0.250000\t-1.234568\t0.001\t0.0123457\t0.002\t1\t0\t2",
        "B\tC\t-1.000000\t1.000000\tinf\t1\t1\t1\t0\t0\t0"]
    line = diffcoex.summary(res, np.array([1, 0]), np.array([0, 0]), np.array([2, 0]))
    assert line == ("differential co-expression: 999 label permutations of 2 gene pairs: 1 with Q <= 0.05, 1 with "
                    "P_maxT <= 0.05; 1 of them in one group's graph only, 1 touching a biomarker")
