"""CPU checks of the label-permutation test (DESIGN.md §4.24): the quantisation, the statistic against cli.tscore,
the oracle's permutations, tally and step-down maxT against their definitions, Benjamini-Hochberg against scipy,
every refusal (raised before the library is loaded) and the --permutations option."""
import numpy as np
import pytest

from g2vec_b200 import cli, perm
from tests import perm_oracle


def cohort(n, G, seed, n0=None):
    rs = np.random.RandomState(seed)
    x = rs.standard_normal((n, G)) * rs.uniform(0.1, 10.0, G) + rs.uniform(-50, 50, G)
    n0 = n // 2 if n0 is None else n0
    lab = np.array([0] * n0 + [1] * (n - n0))
    rs.shuffle(lab)
    return x, lab


# ---------------------------------------------------------------------------------------------- quantisation
def test_quantisation_range_and_constant_genes():
    x, _ = cohort(200, 300, 0)
    x[:, 7] = 3.25                                      # constant gene
    x[:, 8] = 0.0
    x[:, 9] = 1e-300 * np.arange(200)                   # tiny spread
    x[:, 10] = 1e300 * (np.arange(200) % 3)             # huge spread
    q = perm.quantise(x)
    m = np.abs(q).max(axis=0)
    assert (m <= 1 << perm.Q_BITS).all()
    nz = np.ones(300, bool); nz[[7, 8]] = False
    assert (q[:, ~nz] == 0).all() and (m[nz] >= 1 << 21).all()


def test_quantisation_invariant_to_power_of_two_scaling_and_shifts():
    rs = np.random.RandomState(1)
    x = rs.randint(-1000, 1000, size=(64, 50)).astype(np.float64) / 8.0      # dyadic: every step below is exact
    q = perm.quantise(x)
    for kexp in (-30, -1, 1, 7, 40):
        assert (perm.quantise(np.ldexp(x, kexp)) == q).all()
    assert (perm.quantise(x + rs.randint(-100, 100, size=50)) == q).all()
    assert (perm.quantise(x * -1.0) == -q).all()


# --------------------------------------------------------------------------------------------- the statistic
@pytest.mark.parametrize("n,n0,seed", [(4, 2, 0), (10, 4, 1), (135, 77, 2), (400, 250, 3), (1001, 500, 4)])
def test_T_is_the_pooled_t_of_cli_tscore(n, n0, seed):
    x, lab = cohort(n, 60, seed, n0)
    prep = perm.prepare(x, lab)
    T = perm.t_of(prep["rho_obs"], n)
    q = prep["q"].astype(np.float64)                    # the identity itself: t of the quantised values
    want = np.array([cli.tscore(q[lab == 0, g], q[lab == 1, g]) for g in range(60)])
    assert np.allclose(T, want, rtol=1e-5, atol=0)
    raw = np.array([cli.tscore(x[lab == 0, g], x[lab == 1, g]) for g in range(60)])   # and of the data, to 2^-21
    assert np.allclose(T, raw, rtol=1e-5, atol=1e-4)


def test_selected_group_and_statistic_do_not_depend_on_which_label_is_selected():
    x, lab = cohort(40, 30, 5, 20)
    a = perm.prepare(x, lab)
    b = perm.prepare(x, 1 - lab)                        # tie in size: label 1 is selected, now the other samples
    assert a["k"] == b["k"] == 20 and (a["obs"] + b["obs"] == 1).all()
    assert (a["rho_obs"] == b["rho_obs"]).all() and (np.abs(a["N_obs"]) == np.abs(b["N_obs"])).all()
    c = perm.prepare(x[:35], lab[:35])
    assert c["k"] == min((lab[:35] == 0).sum(), (lab[:35] == 1).sum())


def test_other_labels_are_left_out():
    x, lab = cohort(50, 20, 6)
    lab2 = lab.copy(); lab2[:5] = 2
    a = perm.prepare(x, lab2)
    b = perm.prepare(x[5:], lab[5:])
    assert a["n"] == 45 and (a["rho_obs"] == b["rho_obs"]).all() and (a["order"] == b["order"]).all()


def test_perfect_separation_gives_rho_one_and_infinite_T():
    x, lab = cohort(30, 3, 7)
    x[:, 1] = lab * 5.0 + 1.0
    prep = perm.prepare(x, lab)
    assert prep["rho_obs"][1] == 1.0 and np.isinf(perm.t_of(prep["rho_obs"], 30)[1])
    assert cli.tscore(x[lab == 0, 1], x[lab == 1, 1]) == 0.0          # where step 6's t-score says 0
    assert prep["order"][0] == 1


# ------------------------------------------------------------------------------------------------ the oracle
def _scalar_fisher_yates(obs, seed, b):
    """One permutation straight from the rule, with Python integers for the 64-bit draws."""
    from oracle import philox4x32_10
    row = list(obs)
    n = len(row)
    sub = (1 << 63) + b
    for i in range(n - 1, 0, -1):
        s = n - 1 - i
        w = philox4x32_10((s >> 1, 0, sub & 0xFFFFFFFF, sub >> 32), (seed & 0xFFFFFFFF, seed >> 32))
        d = (w[3] << 32 | w[2]) if s & 1 else (w[1] << 32 | w[0])
        j = (d * (i + 1)) >> 64
        row[i], row[j] = row[j], row[i]
    return row


@pytest.mark.parametrize("n,k", [(3, 1), (33, 16), (135, 58), (200, 199)])
def test_oracle_labels_follow_the_rule(n, k):
    obs = np.zeros(n, np.uint8); obs[np.random.RandomState(n).choice(n, k, replace=False)] = 1
    S_pad = -(-n // 32) * 32
    M = perm_oracle.labels(obs, S_pad, 12345, 6, 5)
    assert M.shape == (5, S_pad) and (M[:, n:] == 0).all() and (M.sum(axis=1) == k).all()
    for r in range(5):
        assert list(M[r, :n]) == _scalar_fisher_yates(obs, 12345, 7 + r)
    assert (perm_oracle.labels(obs, S_pad, 12345, 8, 2) == M[2:4]).all()


def test_mulhi64():
    rs = np.random.RandomState(0)
    a = rs.randint(0, 2**63, size=200, dtype=np.int64).astype(np.uint64) * np.uint64(2) + np.uint64(1)
    b = rs.randint(0, 2**63, size=200, dtype=np.int64).astype(np.uint64)
    got = perm_oracle.mulhi64(a, b)
    assert all(int(g) == (int(x) * int(y)) >> 64 for g, x, y in zip(got, a, b))


@pytest.mark.parametrize("seed", range(4))
def test_step_down_maxT_fast_form_equals_the_definition(seed):
    G, Bn, n = 7, 13, 12
    x, lab = cohort(n, G, seed, 5)
    x[:, 2] = x[:, 5]                                   # ties in rho_obs: by gene index
    x[:, 6] = 1.0                                       # constant gene
    prep = perm.prepare(x, lab)
    o = prep["order"]
    M = perm_oracle.labels(prep["obs"], 32, seed, 0, Bn)
    A = perm_oracle.sums(M, prep["q"][:, o])
    c, cm = perm_oracle.tally(A, n, prep["k"], prep["Q"][o], prep["W"][o], np.abs(prep["N_obs"][o]),
                              prep["rho_obs"][o])
    Agene = perm_oracle.sums(M, prep["q"])
    N = n * Agene - prep["k"] * prep["Q"]
    rho = perm.rho_of(N, prep["W"][None, :])
    assert (cm == perm_oracle.maxt_counts_naive(rho, prep["rho_obs"])).all()
    assert (c == (np.abs(N) >= np.abs(prep["N_obs"])).sum(axis=0)[o]).all()
    res = perm.finish(prep, c, cm, Bn)
    assert res.count[6] == Bn and res.P[6] == 1.0 and res.P_maxT[6] == 1.0
    assert (res.P_maxT >= res.P - 1e-15).all() and (np.diff(res.P_maxT[o]) >= 0).all()


def test_bh_matches_scipy():
    from scipy import stats
    rs = np.random.RandomState(3)
    for m in (1, 2, 10, 1000):
        p = rs.uniform(size=m) ** 3
        p[: m // 3] = p[0]                              # ties
        assert np.allclose(perm.bh(p), stats.false_discovery_control(p, method="bh"), rtol=1e-12, atol=0)


# ---------------------------------------------------------------------------------------------- refusals
def _no_library(monkeypatch):
    from g2vec_b200 import _capi

    def boom():
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(_capi, "load", boom)


@pytest.mark.parametrize("case", ["n0", "n1", "n_small", "n_large", "B0", "B_large", "B_float", "nan", "inf", "shape"])
def test_refusals_raise_before_the_library_is_loaded(case, monkeypatch):
    _no_library(monkeypatch)
    x, lab = cohort(20, 5, 0)
    B = 10
    if case == "n0":
        lab = np.ones(20, int)
    elif case == "n1":
        lab = np.zeros(20, int); lab[:3] = 2
    elif case == "n_small":
        lab = np.full(20, 2); lab[0], lab[1] = 0, 1
    elif case == "n_large":
        x = np.zeros((32769, 1)); lab = np.arange(32769) % 2
    elif case == "B0":
        B = 0
    elif case == "B_large":
        B = (1 << 24) + 1
    elif case == "B_float":
        B = 2.5
    elif case == "nan":
        x[3, 2] = np.nan
    elif case == "inf":
        x[3, 2] = -np.inf
    else:
        lab = lab[:-1]
    with pytest.raises(ValueError):
        perm.perm_test(x, lab, B)


def test_non_finite_values_of_left_out_samples_are_ignored(monkeypatch):
    x, lab = cohort(20, 5, 0)
    x[0, 0] = np.nan; lab[0] = 2
    xs, ls = perm.check_inputs(x, lab, 1 << 24)
    assert xs.shape == (19, 5) and np.isfinite(xs).all()
    x2 = np.zeros((32768, 1)); x2[::2] = 1.0
    perm.check_inputs(x2, np.arange(32768) % 2, 1)      # the largest n and the smallest B are admitted


# ----------------------------------------------------------------------------------------- command line
def test_permutations_option():
    a = cli.parse_arguments(["E", "C", "N", "R"])
    assert a.permutations == 0 and "permutations=0" in repr(a)
    assert cli.parse_arguments(["E", "C", "N", "R", "--permutations", "1000"]).permutations == 1000
    assert cli.parse_arguments(["E", "C", "N", "R", "--permutations", str(1 << 24)]).permutations == 1 << 24
    for bad in ("-1", str((1 << 24) + 1), "1.5", "x"):
        with pytest.raises(SystemExit):
            cli.parse_arguments(["E", "C", "N", "R", "--permutations", bad])


def test_cli_refuses_bad_inputs_before_step_3(tmp_path, capsys, monkeypatch):
    """A cohort with one label only fails right after step 2, without touching the GPU modules."""
    _no_library(monkeypatch)
    ef, cf, nf = (str(tmp_path / f) for f in ("E.txt", "C.txt", "N.txt"))
    with open(ef, "w") as f:
        f.write("G\tS1\tS2\tS3\tS4\nA\t1\t2\t3\t4\nB\t4\t3\t2\t2\n")
    with open(cf, "w") as f:
        f.write("P\tLABEL\nS1\t0\nS2\t0\nS3\t0\nS4\t0\n")
    with open(nf, "w") as f:
        f.write("src\tdest\nA\tB\n")
    with pytest.raises(SystemExit):
        cli.main([ef, cf, nf, str(tmp_path / "res"), "--permutations", "10"])
    out = capsys.readouterr().out
    assert "ERROR: permutation test: needs samples of both labels" in out and ">>> 3." not in out


def test_pvalues_writer_format(tmp_path):
    p = str(tmp_path / "res")
    res = perm.PermResult(T=np.array([1.5, np.inf]), P=np.array([0.5, 1 / 3.0]), P_maxT=np.array([0.75, 1 / 3.0]),
                          Q=np.array([0.5, 2 / 3.0]), count=None, count_maxt=None, order=None, n_perm=2)
    cli.write_pvalues(p, np.array(["A1CF", "AAK1"]), np.array([1, 2]), res, ["AAK1"])
    assert open(p + "_pvalues.txt").read() == (
        "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tT\tP\tP_maxT\tQ\tBiomarker\n"
        "A1CF\t1\t1.500000\t0.5\t0.75\t0.5\t0\nAAK1\t2\tinf\t0.333333\t0.333333\t0.666667\t1\n")
