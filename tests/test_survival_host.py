"""Host side of the permutation Cox score test (g2vec_b200/survival.py, DESIGN.md §4.31) and its NumPy restatement
(tests/survival_oracle.py): no GPU needed."""
import numpy as np
import pytest

from g2vec_b200 import survival
from tests import perm_oracle, survival_oracle


def _times(rs, n, ties=False, p_event=0.7):
    t = rs.exponential(10.0, n)
    if ties:
        t = np.round(t)                                 # many tied times, events and censorings among them
    return t, (rs.rand(n) < p_event).astype(np.int64)


def _loglik(beta, x, t, e):
    """Breslow log partial likelihood sum_k [beta E1_k - d_k log sum_{time >= t_k} exp(beta x)]."""
    out = 0.0
    for tk in np.unique(t[e == 1]):
        ev = (t == tk) & (e == 1)
        out += beta * x[ev].sum() - ev.sum() * np.log(np.exp(beta * x[t >= tk]).sum())
    return out


# ------------------------------------------------------------------------------------------------ statistic
def test_oracle_u_and_v_are_the_derivatives_of_the_breslow_likelihood_with_ties():
    rs = np.random.RandomState(1)
    n = 60
    t, e = _times(rs, n, ties=True)
    q = rs.randint(-20, 21, size=(n, 4)).astype(np.int64)
    order, _, flags, a, c = survival.time_groups(t, e)
    assert (np.diff(np.unique(t, return_counts=True)[1]) != 0).any()
    _, U, V = survival_oracle.scan(q, order[None, :], flags, a, c)
    for g in range(4):
        x = q[:, g].astype(np.float64)
        h = 1e-4
        du = (_loglik(h, x, t, e) - _loglik(-h, x, t, e)) / (2 * h)
        h = 1e-3
        dv = -(_loglik(h, x, t, e) - 2 * _loglik(0.0, x, t, e) + _loglik(-h, x, t, e)) / (h * h)
        assert abs(U[0, g] - du) <= 1e-6 * max(1.0, abs(du))
        assert abs(V[0, g] - dv) <= 1e-4 * max(1.0, abs(dv))
        z, u, v = survival.cox_score(x, t, e)
        assert abs(u - U[0, g]) <= 1e-9 * max(1.0, abs(u)) and abs(v - V[0, g]) <= 1e-9 * v


def test_z_is_the_signed_log_rank_statistic_without_ties():
    from scipy import stats
    rs = np.random.RandomState(2)
    for n in (10, 57, 300):
        t, e = _times(rs, n)
        x = (rs.rand(n) < 0.4).astype(np.float64)
        z = survival.cox_score(x, t, e)[0]
        g1, g0 = x == 1, x == 0
        r = stats.logrank(stats.CensoredData(uncensored=t[g1 & (e == 1)], right=t[g1 & (e == 0)]),
                          stats.CensoredData(uncensored=t[g0 & (e == 1)], right=t[g0 & (e == 0)]))
        assert abs(z - r.statistic) <= 1e-12 * max(1.0, abs(z))
        assert abs(survival.p_score([z])[0] - r.pvalue) <= 1e-12


def test_z_from_q_is_z_from_x_and_scaling_a_gene_changes_nothing():
    rs = np.random.RandomState(3)
    n, G = 135, 50
    x = rs.standard_normal((n, G)) * rs.uniform(0.1, 10.0, G) + rs.uniform(-50, 50, G)
    t, e = _times(rs, n, ties=True)
    prep = survival.prepare(x, t, e)
    _, U, V = survival_oracle.observed(prep)
    zq = survival.z_of(U, V)
    zx = survival.cox_score(x, t, e)[0]
    assert (np.abs(zq - zx) <= 1e-3 * np.maximum(1.0, np.abs(zx))).all()
    x2 = x.copy(); x2[:, 7] *= 4.0; x2[:, 9] *= -1.0 / 1024
    T2, U2, V2 = survival_oracle.observed(survival.prepare(x2, t, e))
    T1 = survival_oracle.observed(prep)[0]
    assert T2[7] == T1[7] and U2[7] == U[7] and V2[7] == V[7]
    assert T2[9] == T1[9] and U2[9] == -U[9]


def test_int64_bounds_hold_at_the_extremes():
    """|q| = 2^16 at n = 32768: num_u and num_v equal Python's integers (no wrap) and stay within 2^47 and 2^62."""
    n, v = 32768, 1 << 16
    rs = np.random.RandomState(4)
    cases = [np.full(n, v), np.full(n, -v), np.where(np.arange(n) < n // 2, v, -v), np.where(rs.rand(n) < 0.5, v, -v)]
    for q in cases:
        for S0 in (1, n // 2, n):
            s = q[:S0].astype(object)
            S1, S2 = sum(s), sum(x * x for x in s)
            for d in (1, S0):
                E1 = sum(s[S0 - d:]) if d < S0 else S1
                num_u, num_v = S0 * E1 - d * S1, S0 * S2 - S1 * S1
                assert abs(num_u) <= 1 << 47 and 0 <= num_v <= 1 << 62 and S0 * S2 <= 1 << 62
                assert abs(S1) <= 1 << 31 and S2 <= 1 << 47
                qi = np.array(q[:S0], np.int64)
                S1i, S2i = qi.sum(), (qi * qi).sum()
                assert int(np.int64(S0) * S2i - S1i * S1i) == num_v
                assert int(np.int64(S0) * qi[S0 - d:].sum() - np.int64(d) * S1i) == num_u
    # every sample at one time with every one an event: S0 S2 = 2^62 exactly
    q = np.full((n, 1), v, np.int64)
    order, _, flags, a, c = survival.time_groups(np.zeros(n), np.ones(n, np.int64))
    T, U, V = survival_oracle.scan(q, order[None, :], flags, a, c)
    assert U[0, 0] == 0.0 and V[0, 0] == 0.0 and T[0, 0] == 0.0


def test_v_zero_rule():
    rs = np.random.RandomState(5)
    n = 20
    t, e = _times(rs, n)
    x = rs.standard_normal((n, 3))
    x[:, 1] = 2.5                                       # constant gene: q = 0, U = V = T = 0
    e[:] = 0; e[np.argmax(t)] = 1                      # one event, at the latest time: its risk set is itself
    prep = survival.prepare(x, t, e)
    T, U, V = survival_oracle.observed(prep)
    assert (V == 0).all() and (U == 0).all() and (T == 0).all()
    res = survival.finish(prep, T, U, V, np.arange(3), np.zeros(3), np.zeros(3), 1)
    assert (res.Z == 0).all() and (res.P_score == 1.0).all()


def test_layout_of_the_time_groups():
    t = np.array([5.0, 2.0, 5.0, 7.0, 2.0, 1.0])
    e = np.array([1, 0, 0, 1, 1, 0])
    order, slot, flags, a, c = survival.time_groups(t, e)
    assert order.tolist() == [3, 0, 2, 1, 4, 5] and (slot[order] == np.arange(6)).all()
    assert flags.tolist() == [3, 1, 2, 0, 3, 2]
    assert a.tolist() == [1.0, 0.0, 1 / 3, 0.0, 1 / 5, 1 / 6]
    assert c.tolist() == [1.0, 0.0, 1 / 9, 0.0, 1 / 25, 0.0]


# ------------------------------------------------------------------------------------------------------ rows
def test_rows_carry_the_permutation_tests_draws():
    rs = np.random.RandomState(6)
    for n in (3, 31, 200):
        t, e = _times(rs, n, ties=True)
        order, slot, _, _, _ = survival.time_groups(t, e)
        pi = survival_oracle.perms(n, 11, 4, 9)
        obs = (rs.rand(n) < 0.5).astype(np.uint8)
        assert (obs[pi] == perm_oracle.labels(obs, -(-n // 32) * 32, 11, 4, 9)[:, :n]).all()
        idx = survival_oracle.rows(slot, 11, 4, 9)
        assert (order[np.argsort(idx, axis=1)] == pi).all()
        assert (np.sort(idx, axis=1) == np.arange(n)).all()


# ------------------------------------------------------------------------------------------------------ counts
def test_fast_step_down_equals_the_naive_one():
    rs = np.random.RandomState(7)
    G, B = 30, 20
    T_obs = rs.rand(G); T_obs[2] = T_obs[9] = T_obs[4]
    Tp = rs.rand(B, G) * 1.2
    Tp[3, 5] = T_obs[5]
    o = np.argsort(-T_obs, kind="stable")
    c, cm = survival_oracle.tally(Tp[:, o], T_obs[o])
    assert (cm == perm_oracle.maxt_counts_naive(Tp, T_obs)).all()
    assert (c == (Tp[:, o] >= T_obs[o][None, :]).sum(axis=0)).all()


def test_oracle_in_any_chunking_and_a_planted_gene():
    rs = np.random.RandomState(8)
    n, G = 40, 12
    x = rs.standard_normal((n, G))
    t, e = _times(rs, n)
    x[:, 5] = -np.log(t) + 0.05 * rs.standard_normal(n)   # high expression, short time: Z > 0
    a = survival_oracle.survival_test(x, t, e, 60, seed=2)
    b = survival_oracle.survival_test(x, t, e, 60, seed=2, chunk=7)
    for f in ("count", "count_maxt", "P", "P_maxT", "Q", "T", "Z"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    assert a.order[0] == 5 and a.P[5] == 1.0 / 61 and a.Z[5] > 3
    assert (a.P_maxT >= a.P).all() and (np.diff(a.P_maxT[a.order]) >= 0).all()


# ---------------------------------------------------------------------------------------------------- parser
def _write(tmp_path, text):
    p = tmp_path / "S.txt"
    p.write_text(text)
    return str(p)


def test_reader_and_matcher(tmp_path):
    path = _write(tmp_path, "SAMPLE\tTIME\tEVENT\tSTAGE\nA\t10.5\t1\tII\nB\tNA\t0\nC\t3\t\nD\t0\t0\tIV\nX\t4\t1\n")
    rec = survival.read_survival(path)
    assert rec == {"A": (10.5, 1), "B": (None, None), "C": (None, None), "D": (0.0, 0), "X": (4.0, 1)}
    time, event, used = survival.match_survival(rec, ["D", "B", "A", "C"])
    assert used.tolist() == [True, False, True, False] and event.tolist() == [0, 0, 1, 0]
    assert time[0] == 0.0 and time[2] == 10.5 and np.isnan(time[1])
    with pytest.raises(ValueError, match="no row"):
        survival.match_survival(rec, ["A", "Q"])


@pytest.mark.parametrize("body", ["A\t1\t1\nA\t2\t0\n", "A\tx\t1\n", "A\t-1\t1\n", "A\tinf\t1\n", "A\t1\t2\n",
                                  "A\t1\t0.5\n", "A\t1\n"])
def test_reader_refuses(tmp_path, body):
    with pytest.raises(ValueError):
        survival.read_survival(_write(tmp_path, "SAMPLE\tTIME\tEVENT\n" + body))


@pytest.mark.parametrize("case", ["shape", "B0", "Bbig", "Bfloat", "few", "many", "no_events", "nan_x", "neg_t",
                                  "bad_event"])
def test_check_inputs_refuses(case):
    rs = np.random.RandomState(9)
    x = rs.standard_normal((10, 4))
    t, e = _times(rs, 10)
    e[0] = 1
    B = 10
    if case == "shape":
        t = t[:-1]
    elif case == "B0":
        B = 0
    elif case == "Bbig":
        B = (1 << 20) + 1
    elif case == "Bfloat":
        B = 2.5
    elif case == "few":
        x, t, e = x[:2], t[:2], e[:2]
    elif case == "many":
        x, t, e = np.zeros((32769, 1)), np.ones(32769), np.ones(32769, np.int64)
    elif case == "no_events":
        e[:] = 0
    elif case == "nan_x":
        x[3, 1] = np.nan
    elif case == "neg_t":
        t[2] = -1.0
    elif case == "bad_event":
        e[2] = 2
    with pytest.raises(ValueError):
        survival.check_inputs(x, t, e, B)


# ---------------------------------------------------------------------------------------------- command line
def test_option_parsing():
    from g2vec_b200 import cli
    pos = ["E", "C", "N", "R"]
    a = cli.parse_arguments(pos)
    assert a.survival is None and a.survival_permutations == 1000
    a = cli.parse_arguments(pos + ["--survival", "S.txt", "--survival-permutations", str(1 << 20)])
    assert a.survival == "S.txt" and a.survival_permutations == 1 << 20
    for bad in ("0", "-1", str((1 << 20) + 1), "1.5", "x"):
        with pytest.raises(SystemExit):
            cli.parse_arguments(pos + ["--survival-permutations", bad])


def test_writer_and_summary_format(tmp_path):
    from g2vec_b200 import cli
    genes = np.array(["A", "B", "C"])
    res = survival.SurvivalResult(Z=np.array([2.5, -1.234567891, 0.0]), T=np.array([6.25, 1.5, 0.0]),
                                  P_score=np.array([0.0124193, 0.217, 1.0]), P=np.array([0.001, 0.2, 1.0]),
                                  P_maxT=np.array([0.0123456789, 0.5, 1.0]), Q=np.array([0.003, 0.3, 1.0]),
                                  count=np.zeros(3), count_maxt=np.zeros(3), order=np.arange(3), n_perm=999, n=130,
                                  n_events=41)
    prefix = str(tmp_path / "out")
    cli.write_survival(prefix, genes, np.array([0, 2, 1]), res, ["B", "A"])
    assert open(prefix + "_survival.txt").read().splitlines() == [
        "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tZ\tP_score\tP\tP_maxT\tQ\tBiomarker",
        "A\t0\t2.500000\t0.0124193\t0.001\t0.0123457\t0.003\t1",
        "B\t2\t-1.234568\t0.217\t0.2\t0.5\t0.3\t1",
        "C\t1\t0.000000\t1\t1\t1\t1\t0"]
    line = survival.summary(res, np.array([1, 1, 0]), 1.5, 0.1336)
    assert line == ("survival: 999 permutations of 130 samples (41 events): 1 genes with P_maxT <= 0.05 (1 of the "
                    "biomarkers), 1 with Q <= 0.05; Cox score test of the good / poor label: Z = 1.5000, "
                    "P_score = 0.1336")


def test_label_score_is_cox_score_of_the_label():
    rs = np.random.RandomState(10)
    t, e = _times(rs, 50)
    lab = rs.randint(0, 2, 50); lab[3] = 2
    z, p = survival.label_score(lab, t, e)
    keep = lab != 2
    assert z == survival.cox_score(lab[keep].astype(float), t[keep], e[keep])[0]
    assert p == survival.p_score([z])[0]
    assert survival.label_score(np.zeros(50, int), t, e) == (0.0, 1.0)
