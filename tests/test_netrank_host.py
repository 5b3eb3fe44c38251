"""CPU checks of the NetRank test (DESIGN.md §4.35): the iteration count, the CSR, the oracle against a direct sparse
solve, d = 0, invariance to power-of-two scaling, every refusal (raised before the library is loaded), the options and
the exact formats of the writer and the summary line."""
import os

import numpy as np
import pytest

from g2vec_b200 import cli, diffcoex, netrank, perm
from tests import netrank_oracle
from tests.test_perm_host import _no_library, cohort


def _ex():
    from tests.helpers import GOLDEN
    e = np.load(os.path.join(GOLDEN, "ex_expr.npz"))
    return e["expr"], np.load(os.path.join(GOLDEN, "ex_graph.npz"))["label"], diffcoex.pairs_from_edges(e["src"],
                                                                                                     e["dst"])


# ------------------------------------------------------------------------------------------- iteration count
def test_iteration_count():
    assert [netrank.n_iterations(d) for d in (0.0, 0.3, 0.5, 0.95)] == [0, 23, 40, 539]
    for d in (0.3, 0.5, 0.9, 0.95, 1e-13):
        T = netrank.n_iterations(d)
        prod = 1.0
        for _ in range(T - 1):
            prod *= d
        assert prod > 1e-12 and prod * d <= 1e-12, d
    assert netrank.n_iterations(1e-13) == 1


# ------------------------------------------------------------------------------------------------------ CSR
def test_csr_collapses_duplicates_reversed_edges_and_self_loops_and_keeps_isolated_genes():
    pairs = diffcoex.pairs_from_edges([3, 0, 1, 0, 2, 4, 4], [0, 3, 1, 1, 0, 4, 0])
    assert pairs.tolist() == [[0, 1], [0, 2], [0, 3], [0, 4]]
    rowptr, col, deg, w = netrank.csr(pairs, 6)
    assert rowptr.tolist() == [0, 4, 5, 6, 7, 8, 8] and col.tolist() == [1, 2, 3, 4, 0, 0, 0, 0]
    assert deg.tolist() == [4, 1, 1, 1, 1, 0] and w.tolist() == [0.25, 1.0, 1.0, 1.0, 1.0, 0.0]
    assert rowptr.dtype == np.int32 and col.dtype == np.int32
    assert netrank.row_order(deg).tolist() == [0, 1, 2, 3, 4, 5]
    rs = np.random.RandomState(1)
    pairs = diffcoex.pairs_from_edges(rs.randint(0, 50, 400), rs.randint(0, 50, 400))
    rowptr, col, deg, w = netrank.csr(pairs, 60)
    for j in range(60):
        nb = col[rowptr[j]:rowptr[j + 1]]
        assert (np.diff(nb) > 0).all()
        want = sorted(set(pairs[pairs[:, 0] == j, 1]) | set(pairs[pairs[:, 1] == j, 0]))
        assert nb.tolist() == want and deg[j] == len(want)
    assert (deg[50:] == 0).all()


# --------------------------------------------------------------------------------------------------- oracle
def _direct(S, pairs, d):
    import scipy.sparse as sp
    import scipy.sparse.linalg as spl
    G = S.shape[0]
    rowptr, col, deg, w = netrank.csr(pairs, G)
    A = sp.csr_matrix((np.ones(col.shape[0]), col, rowptr.astype(np.int64)), shape=(G, G))
    M = (sp.identity(G) - d * (A.T @ sp.diags(w))).tocsc()
    return np.stack([spl.spsolve(M, (1.0 - d) * S[:, b]) for b in range(S.shape[1])], axis=1)


@pytest.mark.parametrize("d", [0.3, 0.5, 0.9, 0.95])
def test_oracle_equals_a_direct_solve(d):
    rs = np.random.RandomState(int(d * 100))
    G = 300
    pairs = diffcoex.pairs_from_edges(rs.randint(0, 250, 1500), rs.randint(0, 250, 1500))   # 50 isolated genes
    pairs = np.unique(np.vstack([pairs, np.stack([np.zeros(40, int), np.arange(1, 41)], 1)]), axis=0).astype(np.int32)
    S = rs.uniform(size=(G, 3))
    S[7] = 0.0
    got, want = netrank_oracle.propagate(S, pairs, d), _direct(S, pairs, d)
    assert (np.abs(got - want).sum(axis=0) <= 1e-10 * np.abs(want).sum(axis=0)).all()
    assert np.array_equal(got[250:], (1.0 - d) * S[250:])                                     # no neighbours


def test_oracle_equals_a_direct_solve_on_the_example_network():
    x, lab, pairs = _ex()
    S = np.sqrt(perm.prepare(x, lab)["rho_obs"])[:, None]
    got, want = netrank_oracle.propagate(S, pairs, 0.5), _direct(S, pairs, 0.5)
    assert np.abs(got - want).sum() <= 1e-10 * np.abs(want).sum()


def test_zero_damping_gives_the_seeds_bit_for_bit():
    x, lab = cohort(40, 30, 3, 17)
    x[:, 4] = 1.5                                       # constant gene: S = 0
    pairs = diffcoex.pairs_from_edges(*np.triu_indices(20, 1))
    r = netrank_oracle.netrank_test(x, lab, pairs, 25, damping=0.0, seed=2)
    rho = perm.prepare(x, lab)["rho_obs"]
    assert r.n_iter == 0 and np.array_equal(r.S, np.sqrt(rho)) and np.array_equal(r.score, r.S) and r.S[4] == 0.0


def test_zero_damping_counts_equal_the_permutation_tests_counts():
    from tests import perm_oracle
    x, lab = cohort(33, 12, 8, 15)
    pairs = diffcoex.pairs_from_edges([0, 1, 2], [1, 2, 3])
    r = netrank_oracle.netrank_test(x, lab, pairs, 40, damping=0.0, seed=5)
    p = perm_oracle.perm_test(x, lab, 40, seed=5)
    assert (r.count == p.count).all()


def test_scores_are_invariant_to_scaling_a_gene_by_a_power_of_two():
    x, lab = cohort(30, 25, 4, 14)
    pairs = diffcoex.pairs_from_edges(np.arange(24), np.arange(1, 25))
    a = netrank_oracle.netrank_test(x, lab, pairs, 20, damping=0.9, seed=1)
    y = x.copy()
    y[:, 3] *= 2.0 ** 20
    y[:, 11] *= 2.0 ** -30
    b = netrank_oracle.netrank_test(y, lab, pairs, 20, damping=0.9, seed=1)
    for f in ("S", "score", "P", "Q"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    assert (a.order == b.order).all() and (a.count == b.count).all()


# -------------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("case", ["shape", "B0", "Bbig", "Bfloat", "Bstr", "d_neg", "d_big", "d_nan", "d_inf", "d_str",
                                  "n0", "n1", "n_small", "n_large", "nan", "inf", "nopairs", "pair_oob", "pair_neg",
                                  "pair_rev", "pair_self", "pair_dup", "pair_unsorted", "pair_shape", "pair_float"])
def test_refusals_raise_before_the_library_is_loaded(case, monkeypatch):
    _no_library(monkeypatch)
    x, lab = cohort(20, 6, 9, 10)
    pairs, B, d = np.array([[0, 1], [2, 5]], np.int32), 10, 0.5
    if case == "shape":
        lab = lab[:-1]
    elif case == "B0":
        B = 0
    elif case == "Bbig":
        B = (1 << 20) + 1
    elif case == "Bfloat":
        B = 2.5
    elif case == "Bstr":
        B = "x"
    elif case == "d_neg":
        d = -1e-300
    elif case == "d_big":
        d = 0.9500001
    elif case == "d_nan":
        d = float("nan")
    elif case == "d_inf":
        d = float("inf")
    elif case == "d_str":
        d = "x"
    elif case == "n0":
        lab = np.ones(20, int)
    elif case == "n1":
        lab = np.zeros(20, int); lab[:3] = 2
    elif case == "n_small":
        lab = np.full(20, 2); lab[0], lab[1] = 0, 1
    elif case == "n_large":
        x, lab = np.zeros((32769, 6)), np.arange(32769) % 2
    elif case == "nan":
        x[4, 2] = np.nan
    elif case == "inf":
        x[4, 2] = -np.inf
    elif case == "nopairs":
        pairs = np.zeros((0, 2), np.int32)
    elif case == "pair_oob":
        pairs = np.array([[0, 6]])
    elif case == "pair_neg":
        pairs = np.array([[-1, 2]])
    elif case == "pair_rev":
        pairs = np.array([[2, 1]])
    elif case == "pair_self":
        pairs = np.array([[2, 2]])
    elif case == "pair_dup":
        pairs = np.array([[0, 1], [0, 1]])
    elif case == "pair_unsorted":
        pairs = np.array([[2, 3], [0, 1]])
    elif case == "pair_shape":
        pairs = np.array([0, 1])
    elif case == "pair_float":
        pairs = np.array([[0.0, 1.0]])
    with pytest.raises(ValueError, match="netrank"):
        netrank.netrank_test(x, lab, pairs, B, damping=d)


def test_admitted_extremes_and_left_out_samples():
    x, lab = cohort(20, 6, 9, 10)
    lab[0] = 2
    x[0, 0] = np.nan                                    # in a left-out sample: ignored
    xx, ll, pp = netrank.check_inputs(x, lab, [[0, 1]], 1 << 20, 0.95)
    assert xx.shape == (19, 6) and (ll != 2).all() and pp.dtype == np.int32
    netrank.check_inputs(x, lab, [[0, 5]], 1, 0.0)


# ----------------------------------------------------------------------------------------------- command line
def test_options():
    pos = ["E", "C", "N", "R"]
    a = cli.parse_arguments(pos)
    assert a.netrank == 0 and a.netrank_damping == 0.5 and "netrank=0, netrank_damping=0.5" in repr(a)
    a = cli.parse_arguments(pos + ["--netrank", str(1 << 20), "--netrank-damping", "0.95"])
    assert a.netrank == 1 << 20 and a.netrank_damping == 0.95
    assert cli.parse_arguments(pos + ["--netrank-damping", "0"]).netrank_damping == 0.0
    for bad in (["--netrank", "-1"], ["--netrank", str((1 << 20) + 1)], ["--netrank", "1.5"],
                ["--netrank-damping", "-0.1"], ["--netrank-damping", "0.96"], ["--netrank-damping", "nan"],
                ["--netrank-damping", "inf"], ["--netrank-damping", "x"]):
        with pytest.raises(SystemExit):
            cli.parse_arguments(pos + bad)


def test_cli_refuses_bad_inputs_before_step_3(tmp_path, capsys, monkeypatch):
    _no_library(monkeypatch)
    ef, cf, nf = (str(tmp_path / f) for f in ("E.txt", "C.txt", "N.txt"))
    with open(ef, "w") as f:
        f.write("G\tS1\tS2\tS3\tS4\nA\t1\t2\t3\t4\nB\t4\t3\t2\t2\nC\t1\t1\t1\t2\n")
    with open(cf, "w") as f:
        f.write("P\tLABEL\nS1\t0\nS2\t1\nS3\t0\nS4\t1\n")
    with open(nf, "w") as f:
        f.write("src\tdest\nA\tA\nC\tC\n")                # self-loops only: no pairs
    with pytest.raises(SystemExit) as e:
        cli.main([ef, cf, nf, str(tmp_path / "res"), "--netrank", "10"])
    out = capsys.readouterr().out
    assert e.value.code == 1 and "ERROR: --netrank: netrank: 0 gene pairs" in out and ">>> 3." not in out
    with open(cf, "w") as f:
        f.write("P\tLABEL\nS1\t0\nS2\t0\nS3\t0\nS4\t0\n")
    with open(nf, "w") as f:
        f.write("src\tdest\nA\tB\n")
    with pytest.raises(SystemExit):
        cli.main([ef, cf, nf, str(tmp_path / "res"), "--netrank", "10"])
    out = capsys.readouterr().out
    assert "ERROR: --netrank: netrank: needs samples of both labels" in out and ">>> 3." not in out


def _result():
    return netrank.NetRankResult(degree=np.array([2, 0, 1]), S=np.array([0.5, 0.125, 1.0]),
                                 score=np.array([0.3125, 0.0625, 0.40625]), order=np.array([2, 0, 1]),
                                 P=np.array([0.001, 1.0, 0.0123456789]), Q=np.array([0.003, 1.0, 0.0185185]),
                                 count=np.array([0, 998, 11]), n_iter=40, n_perm=999)


def test_summary_and_writer_formats(tmp_path):
    res = _result()
    line = netrank.summary(res, 0.5, 2, np.array([True, False, False]))
    assert line == ("netrank: 999 label permutations, d = 0.5 (40 iterations), 3 genes, 2 pairs: 2 genes with Q <= "
                    "0.05 (1 of the biomarkers); top_netrank (1 genes) Jaccard 0.000 with the biomarkers")
    line2 = netrank.summary(res, 0.95, 2, np.array([False, True, True]), auc=(0.8125, 0.71875))
    assert line2 == ("netrank: 999 label permutations, d = 0.95 (40 iterations), 3 genes, 2 pairs: 2 genes with Q <= "
                     "0.05 (1 of the biomarkers); top_netrank (2 genes) Jaccard 0.333 with the biomarkers; CV AUC 0.812 "
                     "(top_netrank), 0.719 (biomarkers)")
    prefix = str(tmp_path / "out")
    cli.write_netrank(prefix, np.array(["A", "B", "C"]), np.array([0, 2, 1]), res, ["A"], line)
    assert open(prefix + "_netrank.txt").read().splitlines() == [
        "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tDegree\tS\tScore\tRank\tP\tQ\tBiomarker",
        "A\t0\t2\t0.500000\t0.312500\t2\t0.001\t0.003\t1",
        "B\t2\t0\t0.125000\t0.062500\t3\t1\t1\t0",
        "C\t1\t1\t1.000000\t0.406250\t1\t0.0123457\t0.0185185\t0",
        line]
    assert netrank.top_netrank(res, 2).tolist() == [0, 2] and netrank.jaccard([0, 2], [2, 1]) == 1 / 3.0
