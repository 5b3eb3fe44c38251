"""CPU checks of the gene-set enrichment test (DESIGN.md §4.28): GMT parsing and the size filter, the oracle's ES
against the running sum over all G positions, exact cases, the metric's sign against scipy, NES / P / FDR / FWER
against loops over their definitions, every refusal (raised before the library is loaded), the options and the
writer."""
import numpy as np
import pytest

from g2vec_b200 import cli, perm
from g2vec_b200.gsea import (GseaResult, MAX_SET_SIZE, check_inputs, finish, leading_edge, read_gmt, restrict_sets,
                             sign_of, summary)
from tests import gsea_oracle as go
from tests.test_perm_host import cohort


def _gmt(tmp_path, text, name="s.gmt"):
    p = tmp_path / name
    p.write_text(text)
    return str(p)


# ------------------------------------------------------------------------------------------------------------ GMT
def test_read_gmt_parses_lines_and_counts_duplicates_once(tmp_path):
    path = _gmt(tmp_path, "A\tdesc a\tG1\tG2\tG1\t\tG3\n\n   \nB\thttp://x\r\nC\t\tG4\n")
    assert read_gmt(path) == [("A", "desc a", ["G1", "G2", "G3"]), ("B", "http://x", []), ("C", "", ["G4"])]


@pytest.mark.parametrize("text,what", [("A\tx\tG1\nlonely\n", "line 2"), ("A\tx\tG1\nB\ty\nA\tz\tG2\n", "line 3")])
def test_read_gmt_refuses_short_lines_and_duplicate_names(tmp_path, text, what):
    with pytest.raises(ValueError, match=what):
        read_gmt(_gmt(tmp_path, text))


def test_restrict_sets_drops_outside_genes_and_filters_sizes():
    genes = ["a", "b", "c", "d", "e"]
    sets = [("s1", "", ["a", "zz", "c"]), ("s2", "", ["e", "d", "c", "b"]), ("s3", "", ["zz"]),
            ("s4", "", ["a", "b", "c", "d", "e"]), ("s5", "", ["b"])]
    ptr, idx, names = restrict_sets(sets, genes, 1, 4)
    assert names == ["s1", "s2", "s5"] and ptr.tolist() == [0, 2, 6, 7] and idx.tolist() == [0, 2, 1, 2, 3, 4, 1]
    ptr, idx, names = restrict_sets(sets, genes, 2, 5)
    assert names == ["s1", "s2"]                        # s4 has k = G: no gene is left to miss
    assert restrict_sets([("x", [0, 3, 3])], range(4), 1, 4)[1].tolist() == [0, 3]


# ------------------------------------------------------------------------------------------------------------- ES
def test_es_equals_the_running_sum_over_all_positions():
    rs = np.random.RandomState(1)
    worst = 0.0
    for _ in range(400):
        G = int(rs.randint(4, 300))
        r = rs.uniform(-1, 1, G)
        r[rs.rand(G) < 0.1] = 0.0
        if rs.rand() < 0.3:
            r[rs.randint(G, size=G // 4)] = r[0]          # ties, broken by the gene index
        rq = np.rint(r * 2.0 ** 32).astype(np.int64)
        k = int(rs.randint(1, G))
        mem = np.sort(rs.choice(G, k, replace=False))
        key = (((1 << 32) - rq) << 20) | np.arange(G)
        pos = go.rank(key[None, :])[0]
        got = go.es_one(pos, np.abs(rq), mem, G)
        assert got == go.es_brute(rq, mem)                # the same three float64 operations at every hit
        worst = max(worst, abs(got - go.es_brute(r, mem)))
    assert worst <= 1e-9


def test_es_of_the_top_and_bottom_genes_and_of_weightless_sets():
    G, k = 100, 10
    rq = np.rint(np.linspace(1, -1, G) * 2.0 ** 32).astype(np.int64)   # gene g has rank g
    pos, u = np.arange(G, dtype=np.int32), np.abs(rq)
    assert go.es_one(pos, u, np.arange(k), G) == 1.0
    assert go.es_one(pos, u, np.arange(G - k, G), G) == -1.0
    assert go.es_one(pos, np.zeros(G, np.int64), np.arange(5, 20), G) == 0.0
    assert np.copysign(1.0, go.es_one(pos, np.zeros(G, np.int64), np.arange(5, 20), G)) == 1.0


@pytest.mark.parametrize("smaller", [0, 1])
def test_metric_sign_follows_scipy_pointbiserialr(smaller):
    from scipy import stats
    x, lab = cohort(41, 30, 5, 13 if smaller == 0 else 28)
    prep = perm.prepare(x, lab)
    assert sign_of(prep) == (1 if smaller == 1 else -1)
    S_pad = 64
    M = np.zeros((1, S_pad), np.uint8); M[0, :41] = prep["obs"]
    from tests import perm_oracle
    rq, u, _ = go.keys(perm_oracle.sums(M, prep["q"]), prep["n"], prep["k"], sign_of(prep), prep["Q"], prep["W"])
    want = np.array([stats.pointbiserialr(lab, prep["q"][:, g]).statistic for g in range(30)])
    assert np.allclose(rq[0] / 2.0 ** 32, want, atol=1e-9, rtol=0)
    assert (u == np.abs(rq)).all() and np.abs(rq).max() <= 1 << 32


def test_keys_order_by_rq_descending_then_gene():
    rq = np.array([[5, -3, 5, 1 << 32, -(1 << 32), 0]])
    key = (((1 << 32) - rq) << 20) | np.arange(6)
    assert go.rank(key).tolist() == [[1, 4, 2, 0, 5, 3]]


# ------------------------------------------------------------------------------------ normalisation and counts
def _naive(es_null, es_obs):
    """NES, P, FDR, FWER straight from their definitions with Python loops."""
    B, S = es_null.shape
    mp, mn, nes_obs = np.full(S, np.nan), np.full(S, np.nan), np.full(S, np.nan)
    for s in range(S):
        p = [e for e in es_null[:, s] if e >= 0]
        n = [-e for e in es_null[:, s] if e < 0]
        t = 0.0
        for e in p:
            t += e
        mp[s] = t / len(p) if p else np.nan
        t = 0.0
        for e in n:
            t += e
        mn[s] = t / len(n) if n else np.nan
        nes_obs[s] = es_obs[s] / (mp[s] if es_obs[s] >= 0 else mn[s])
    valid = [s for s in range(S) if not np.isnan(nes_obs[s])]
    nes = [[es_null[b, s] / (mp[s] if es_null[b, s] >= 0 else mn[s]) for s in valid] for b in range(B)]
    P, FDR, FW = np.ones(S), np.full(S, np.nan), np.full(S, np.nan)
    for s in valid:
        x, e = nes_obs[s], es_obs[s]
        col = es_null[:, s]
        if e >= 0:
            P[s] = (1 + sum(c >= e for c in col)) / (1 + sum(c >= 0 for c in col))
            a = sum(v >= x for row in nes for v in row) / sum(v >= 0 for row in nes for v in row)
            c = sum(nes_obs[t] >= x for t in valid) / sum(nes_obs[t] >= 0 for t in valid)
            FW[s] = (1 + sum(1 for row in nes if any(v >= 0 for v in row) and max(v for v in row if v >= 0) >= x)) / (B + 1)
        else:
            P[s] = (1 + sum(c <= e for c in col)) / (1 + sum(c < 0 for c in col))
            a = sum(v <= x for row in nes for v in row) / sum(v < 0 for row in nes for v in row)
            c = sum(nes_obs[t] <= x for t in valid) / sum(nes_obs[t] < 0 for t in valid)
            FW[s] = (1 + sum(1 for row in nes if any(v < 0 for v in row) and min(v for v in row if v < 0) <= x)) / (B + 1)
        FDR[s] = min(1.0, a / c)
    return nes_obs, P, FDR, FW


def test_nes_p_fdr_fwer_equal_their_definitions():
    rs = np.random.RandomState(3)
    B, S = 37, 9
    es_null = np.round(rs.uniform(-1, 1, (B, S)), 2)    # ties between permutations and sets
    es_null[:, 4] = np.abs(es_null[:, 4])               # no negative null: a negative ES gets NaN
    es_null[:5, 6] = 0.0
    es_obs = np.round(rs.uniform(-1, 1, S), 2)
    es_obs[4] = -0.3
    es_obs[6] = es_null[7, 6]                           # a tie with the null
    nes, mp, mn, nes_obs, counts = go.norm(es_null, es_obs)
    res = finish(["s%d" % i for i in range(S)], np.arange(S + 1), np.arange(S), es_obs, nes_obs, counts,
                 go.null_counts(nes, nes_obs), mp, mn, B)
    want = _naive(es_null, es_obs)
    assert np.isnan(res.NES[4]) and res.P[4] == 1.0 and np.isnan(res.FDR[4]) and np.isnan(res.FWER[4])
    for got, w in zip((res.NES, res.P, res.FDR, res.FWER), want):
        assert np.array_equal(got, w, equal_nan=True)
    assert (nes[:, 4] != nes[:, 4]).all()               # the NaN set's null column is left out


def test_leading_edge_takes_the_members_up_to_the_peak():
    G = 20
    pos = np.arange(G, dtype=np.int32)
    u = np.full(G, 1 << 30, dtype=np.uint64)
    assert leading_edge(pos, u, [0, 1, 15, 2], G).tolist() == [0, 1, 2]
    assert leading_edge(pos, u, [19, 18, 3], G).tolist() == [18, 19]
    assert leading_edge(pos, np.zeros(G, np.uint64), [0, 1], G).tolist() == []


# ------------------------------------------------------------------------------------------------ refusals
def test_check_inputs_refuses_before_anything_is_uploaded():
    x, lab = cohort(20, 10, 0)
    check_inputs(x, lab, 10, 3, 1, 4)
    bad = [dict(n_perm=0), dict(n_perm=(1 << 20) + 1), dict(n_perm=2.5), dict(n_sets=0),
           dict(n_perm=1 << 18, n_sets=(1 << 10) + 1), dict(min_size=0), dict(min_size=5, max_size=4),
           dict(max_size=MAX_SET_SIZE + 1)]
    for b in bad:
        kw = dict(n_perm=10, n_sets=3, min_size=1, max_size=4)
        kw.update(b)
        with pytest.raises(ValueError):
            check_inputs(x, lab, **kw)
    with pytest.raises(ValueError):
        check_inputs(x, np.zeros(20, int), 10, 3, 1, 4)
    with pytest.raises(ValueError):
        check_inputs(np.zeros((20, (1 << 20) + 1), np.float32), lab, 10, 3, 1, 4)


def test_gsea_refuses_without_touching_the_device(monkeypatch):
    from g2vec_b200 import _capi
    from g2vec_b200.gsea import gsea
    monkeypatch.setattr(_capi, "load", lambda: (_ for _ in ()).throw(AssertionError("loaded")))
    x, lab = cohort(20, 10, 0)
    with pytest.raises(ValueError):
        gsea(x, lab, [("a", [0, 1])], 10, min_size=3, max_size=4)          # no set kept
    with pytest.raises(ValueError):
        gsea(x, lab, [("a", [0, 1, 2])], 0, min_size=1, max_size=4)


# ---------------------------------------------------------------------------------------- options and writer
def test_gene_set_options():
    a = cli.parse_arguments(["e", "c", "n", "r"])
    assert a.gene_sets is None and a.gene_set_permutations == 1000 and a.gene_set_size == (15, 500)
    a = cli.parse_arguments(["e", "c", "n", "r", "--gene-sets", "x.gmt", "--gene-set-permutations", "77",
                             "--gene-set-size", "3,4096"])
    assert a.gene_sets == "x.gmt" and a.gene_set_permutations == 77 and a.gene_set_size == (3, 4096)
    for bad in (["--gene-set-permutations", "0"], ["--gene-set-permutations", str((1 << 20) + 1)],
                ["--gene-set-size", "0,5"], ["--gene-set-size", "6,5"], ["--gene-set-size", "1,4097"],
                ["--gene-set-size", "5"], ["--gene-set-size", "a,b"]):
        with pytest.raises(SystemExit):
            cli.parse_arguments(["e", "c", "n", "r"] + bad)


def test_writer_and_summary(tmp_path):
    genes = np.array(["g0", "g1", "g2", "g3"])
    res = GseaResult(name=["up", "odd"], size=np.array([2, 1]), members=[np.array([0, 2]), np.array([3])],
                     ES=np.array([0.5, -0.25]), NES=np.array([1.5, np.nan]), P=np.array([0.01, 1.0]),
                     FDR=np.array([0.2, np.nan]), FWER=np.array([0.03, np.nan]),
                     leading_edge=[np.array([2, 0]), np.array([], np.int64)], count_pos=None, count_neg=None,
                     count_extreme=None, count_null=None, count_null_side=None, count_obs=None, count_obs_side=None,
                     count_fwer=None, mean_pos=None, mean_neg=None, n_perm=99)
    cli.write_gsea(str(tmp_path / "R"), genes, res, ["g2", "g3"])
    assert (tmp_path / "R_gsea.txt").read_text().splitlines() == [
        "GeneSet\tSize\tES\tNES\tP\tFDR_Q\tFWER_P\tBiomarkers\tLeadingEdge",
        "up\t2\t0.500000\t1.500000\t0.01\t0.2\t0.03\t1\tg2,g0",
        "odd\t1\t-0.250000\tnan\t1\tnan\tnan\t1\t"]
    assert summary(res) == "gene-set test: 99 label permutations: 1 of 2 sets with FDR q <= 0.25 (1 up in poor, 0 up in good)"


def test_oracle_gsea_is_the_same_in_any_chunking():
    x, lab = cohort(30, 60, 4, 12)
    sets = [("s%d" % i, np.random.RandomState(i).choice(60, 5 + i, replace=False)) for i in range(6)]
    a = go.gsea(x, lab, sets, 23, seed=5, min_size=5, max_size=50)
    b = go.gsea(x, lab, sets, 23, seed=5, min_size=5, max_size=50, chunk=7)
    for f in ("ES", "NES", "P", "FDR", "FWER"):
        assert np.array_equal(getattr(a, f), getattr(b, f), equal_nan=True)
