"""The differential co-expression test on the H100 (csrc/g2v_dcx.cu, g2vec_b200/diffcoex.py; DESIGN.md §4.30) against
the NumPy restatement of tests/diffcoex_oracle.py.  Every comparison is bit for bit."""
import os

import numpy as np
import pytest

from g2vec_b200 import diffcoex, perm
from tests import diffcoex_oracle, perm_oracle
from tests.test_perm_host import cohort

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


def _qt(q, S_pad):
    qt = np.zeros((q.shape[1], S_pad), np.int32)
    qt[:, :q.shape[0]] = q.T
    return qt


# The device copies are held in locals until the result is back.
def gpu_sums(M, q, pi, pj):
    import torch
    capi, lib = _lib()
    n_b, S_pad = M.shape
    E = len(pi)
    P = torch.empty((n_b, E), dtype=torch.int64, device="cuda")
    d = [_dev(a) for a in (M, _qt(q, S_pad), np.asarray(pi, np.int32), np.asarray(pj, np.int32))]
    capi.check(lib.g2v_dcx_sums(d[0].data_ptr(), n_b, S_pad, d[1].data_ptr(), q.shape[1], d[2].data_ptr(),
                                d[3].data_ptr(), E, 0, 0, None, None, None, None, None, P.data_ptr(), None, _st()),
               "g2v_dcx_sums")
    return P.cpu().numpy()


def gpu_stats(M, q, pi, pj, n, k, A, Bq, At, Bt, Pt):
    import torch
    capi, lib = _lib()
    n_b, S_pad = M.shape
    E = len(pi)
    D = torch.full((n_b, E), np.nan, dtype=torch.float64, device="cuda")
    d = [_dev(a) for a in (M, _qt(q, S_pad), np.asarray(pi, np.int32), np.asarray(pj, np.int32), A, Bq, At, Bt, Pt)]
    capi.check(lib.g2v_dcx_sums(d[0].data_ptr(), n_b, S_pad, d[1].data_ptr(), q.shape[1], d[2].data_ptr(),
                                d[3].data_ptr(), E, n, k, d[4].data_ptr(), d[5].data_ptr(), d[6].data_ptr(),
                                d[7].data_ptr(), d[8].data_ptr(), None, D.data_ptr(), _st()), "g2v_dcx_sums")
    return D.cpu().numpy()


def gpu_tally(D, D_obs):
    import torch
    capi, lib = _lib()
    n_b, E = D.shape
    c = torch.zeros(E, dtype=torch.int64, device="cuda")
    cm = torch.zeros(E, dtype=torch.int64, device="cuda")
    d = [_dev(a) for a in (D, D_obs)]
    capi.check(lib.g2v_dcx_tally(d[0].data_ptr(), n_b, E, d[1].data_ptr(), c.data_ptr(), cm.data_ptr(), _st()),
               "g2v_dcx_tally")
    return c.cpu().numpy(), cm.cpu().numpy()


# ------------------------------------------------------------------------------------------------------ sums
# rows around the 128-row and 8-row tiles, pairs around the 64-pair and 8-pair tiles, samples around the 32-slab
SUM_SHAPES = [(nb, E, n) for n in (3, 31, 32, 33, 135) for nb in (1, 7, 8, 127, 128, 129) for E in (1, 63, 64, 65, 200)]
SUM_SHAPES += [(2, 5, 32768), (129, 65, 1000), (300, 130, 64)]


def test_sums_equal_the_int64_oracle_at_every_tile_edge():
    rs = np.random.RandomState(0)
    for nb, E, n in SUM_SHAPES:
        G = 40
        q = rs.randint(-(1 << 16), (1 << 16) + 1, size=(n, G)).astype(np.int64)
        S_pad = -(-n // 32) * 32
        M = np.zeros((nb, S_pad), np.uint8); M[:, :n] = rs.randint(0, 2, size=(nb, n))
        pi, pj = rs.randint(0, G, E), rs.randint(0, G, E)
        assert (gpu_sums(M, q, pi, pj) == diffcoex_oracle.sums(M, q, pi, pj)).all(), (nb, E, n)


def test_sums_are_exact_at_the_magnitude_bound():
    n, G, v = 32768, 4, 1 << 16
    q = np.full((n, G), v, np.int64); q[:, 1] = -v; q[:, 2] = v - 1
    M = np.ones((3, n), np.uint8); M[1, ::2] = 0
    pi, pj = np.array([0, 0, 1, 2, 3]), np.array([0, 1, 1, 2, 0])
    got = gpu_sums(M, q, pi, pj)
    assert (got == diffcoex_oracle.sums(M, q, pi, pj)).all()
    assert got[0, 0] == 1 << 47 and got[0, 1] == -(1 << 47)


def _stat_case(rs, n, G, E, nb, k):
    x, lab = cohort(n, G, int(rs.randint(1 << 30)), n - k)
    x[:, 1] = 2.0                                       # constant gene: r = 0
    x[:, 2] = x[:, 3]                                   # r = 1 in every group
    obs = (lab == 1).astype(np.uint8)
    q = perm.quantise(x, bits=16)
    S_pad = -(-n // 32) * 32
    M = perm_oracle.labels(obs, S_pad, 5, 0, nb)
    pairs = diffcoex.pairs_from_edges(np.r_[rs.randint(0, G, E), 1, 2], np.r_[rs.randint(0, G, E), 4, 3])
    pi, pj = pairs[:, 0], pairs[:, 1]
    A, Bq = perm_oracle.sums(M, q), diffcoex_oracle.sums(M, q, np.arange(G), np.arange(G))
    At, Bt = q.sum(axis=0), (q * q).sum(axis=0)
    Pt = (q[:, pi] * q[:, pj]).sum(axis=0)
    return M, q, pi, pj, n, k, A, Bq, At, Bt, Pt


@pytest.mark.parametrize("n,G,E,nb,k", [(8, 6, 10, 1, 4), (33, 20, 63, 129, 10), (135, 300, 700, 130, 58),
                                        (1000, 200, 65, 9, 500), (40, 30, 200, 260, 36)])
def test_statistic_equals_the_oracle(n, G, E, nb, k):
    args = _stat_case(np.random.RandomState(n + E), n, G, E, nb, k)
    got = gpu_stats(*args)
    M, q, pi, pj, n, k, A, Bq, At, Bt, Pt = args
    want = diffcoex_oracle.stats(n, k, A, Bq, diffcoex_oracle.sums(M, q, pi, pj), At, Bt, Pt, pi, pj)
    assert np.array_equal(got, want)
    assert (want == 0.0).any() and (want > 0.0).any()


@pytest.mark.parametrize("E,nb", [(1, 1), (127, 9), (128, 64), (129, 300), (1000, 1000), (3000, 2500)])
def test_tally_equals_the_oracle(E, nb):
    rs = np.random.RandomState(E + nb)
    D_obs = np.sort(rs.rand(E))[::-1].copy()
    D = rs.rand(nb, E) * 1.1
    D[nb // 2, ::3] = D_obs[::3]                        # ties D_b = D_obs
    D_obs[1::5] = D_obs[0]                              # ties in D_obs
    got, want = gpu_tally(D, D_obs), diffcoex_oracle.tally(D, D_obs)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()


def test_entry_points_refuse_bad_sizes_and_launch_nothing():
    capi, lib = _lib()
    import torch
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p, st = buf.data_ptr(), _st()
    N = None
    before = capi.launch_count()
    bad = [lib.g2v_dcx_sums(p, 1, 32, p, 1, p, p, 1, 0, 0, N, N, N, N, N, N, N, st),       # neither P nor D
           lib.g2v_dcx_sums(p, 1, 32, p, 1, p, p, 1, 0, 0, N, N, N, N, N, p, p, st),       # both
           lib.g2v_dcx_sums(p, 0, 32, p, 1, p, p, 1, 0, 0, N, N, N, N, N, p, N, st),
           lib.g2v_dcx_sums(p, (1 << 20) + 1, 32, p, 1, p, p, 1, 0, 0, N, N, N, N, N, p, N, st),
           lib.g2v_dcx_sums(p, 1, 48, p, 1, p, p, 1, 0, 0, N, N, N, N, N, p, N, st),
           lib.g2v_dcx_sums(p, 1, 32800, p, 1, p, p, 1, 0, 0, N, N, N, N, N, p, N, st),
           lib.g2v_dcx_sums(p, 1, 32, p, 0, p, p, 1, 0, 0, N, N, N, N, N, p, N, st),
           lib.g2v_dcx_sums(p, 1, 32, p, 1, p, p, 0, 0, 0, N, N, N, N, N, p, N, st),
           lib.g2v_dcx_sums(p, 1, 32, p, 1, p, p, (1 << 26) + 1, 0, 0, N, N, N, N, N, p, N, st),
           lib.g2v_dcx_sums(p, 1, 32, p, 1, p, p, 1, 20, 10, p, p, p, p, N, N, p, st),     # P_tot missing
           lib.g2v_dcx_sums(p, 1, 32, p, 1, p, p, 1, 20, 3, p, p, p, p, p, N, p, st),      # k < 4
           lib.g2v_dcx_sums(p, 1, 32, p, 1, p, p, 1, 20, 17, p, p, p, p, p, N, p, st),     # n - k < 4
           lib.g2v_dcx_sums(p, 1, 32, p, 1, p, p, 1, 33, 10, p, p, p, p, p, N, p, st),     # n > S_pad
           lib.g2v_dcx_tally(p, 0, 1, p, p, p, st), lib.g2v_dcx_tally(p, 1, 0, p, p, p, st),
           lib.g2v_dcx_tally(p, 1, (1 << 26) + 1, p, p, p, st), lib.g2v_dcx_tally(N, 1, 1, p, p, p, st)]
    assert all(rc != 0 for rc in bad)
    assert capi.launch_count() == before and len(lib.g2v_last_error()) > 0
    torch.cuda.synchronize()


# -------------------------------------------------------------------------------------------- diffcoex_test
def _ex():
    from tests.helpers import GOLDEN
    e = np.load(os.path.join(GOLDEN, "ex_expr.npz"))
    return e["expr"], np.load(os.path.join(GOLDEN, "ex_graph.npz"))["label"], diffcoex.pairs_from_edges(e["src"],
                                                                                                     e["dst"])


def _same(a, b):
    for f in ("count", "count_maxt", "order", "pairs"):
        assert (getattr(a, f) == getattr(b, f)).all(), f
    for f in ("R_good", "R_poor", "Z", "D", "P", "P_maxT", "Q"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f


def test_diffcoex_test_equals_the_oracle_on_ex_in_any_chunking_and_run():
    from g2vec_b200 import _capi
    x, lab, pairs = _ex()
    B = 200
    want = diffcoex_oracle.diffcoex_test(x, lab, pairs, B, seed=3, chunk=77)
    G, E = x.shape[1], pairs.shape[0]
    row = 160 + 16 * G + 8 * E
    for max_bytes, chunks in ((row * 70, 3), (None, 1), (None, 1)):
        before = _capi.launch_count()
        got = diffcoex.diffcoex_test(x, lab, pairs, B, seed=3, max_chunk_bytes=max_bytes)
        assert _capi.launch_count() - before == 3 + 5 * chunks
        _same(got, want)
    assert E == 140902 and (got.P_maxT >= got.P).all()


def test_diffcoex_test_equals_the_oracle_with_one_row_per_chunk_and_left_out_samples():
    x, lab = cohort(45, 30, 11, 20)
    x[:, 0] = 1.0
    x[:, 7] = x[:, 8]
    lab[:3] = 5                                         # left out
    x[0, 3] = np.nan                                    # in a left-out sample: ignored
    pairs = diffcoex.pairs_from_edges(*np.triu_indices(30, 1))
    _same(diffcoex.diffcoex_test(x, lab, pairs, 50, seed=-7, max_chunk_bytes=1),
          diffcoex_oracle.diffcoex_test(x, lab, pairs, 50, seed=-7))


def test_permutation_rows_are_the_permutation_tests():
    """The rows diffcoex_test draws are perm_test's for the same seed: the sums over the observed group's genes
    that both tests see (A through g2v_perm_sums) come from the same g2v_perm_labels rows."""
    x, lab = cohort(60, 10, 12, 25)
    prep_p, prep_d = perm.prepare(x, lab), diffcoex.prepare(x, lab, [[0, 1]])
    assert (prep_p["obs"] == prep_d["obs"]).all() and prep_p["k"] == prep_d["k"]
    # the oracle's rows are the device's (tests/test_gpu_perm.py), and the device test equals the oracle built on them
    _same(diffcoex.diffcoex_test(x, lab, diffcoex.pairs_from_edges(*np.triu_indices(10, 1)), 30, seed=9),
          diffcoex_oracle.diffcoex_test(x, lab, diffcoex.pairs_from_edges(*np.triu_indices(10, 1)), 30, seed=9))


def test_planted_pair_gets_the_smallest_p_value():
    x, lab = cohort(135, 200, 14, 77)
    rs = np.random.RandomState(0)
    x[lab == 1, 17] = x[lab == 1, 90] + 0.3 * rs.standard_normal(58)          # correlated in the poor group only
    pairs = diffcoex.pairs_from_edges(rs.randint(0, 200, 3000), rs.randint(0, 200, 3000))
    pairs = np.unique(np.vstack([pairs, [[17, 90]]]), axis=0).astype(np.int32)
    B = 2000
    r = diffcoex.diffcoex_test(x, lab, pairs, B, seed=1)
    e = int(np.nonzero((pairs[:, 0] == 17) & (pairs[:, 1] == 90))[0][0])
    assert r.P[e] == r.P_maxT[e] == 1.0 / (B + 1) and r.order[0] == e and r.Z[e] > 5


def test_null_p_values_are_roughly_uniform():
    from scipy import stats
    rs = np.random.RandomState(13)
    x = rs.standard_normal((80, 150))
    lab = np.array([0] * 37 + [1] * 43)
    pairs = diffcoex.pairs_from_edges(rs.randint(0, 150, 2000), rs.randint(0, 150, 2000))
    r = diffcoex.diffcoex_test(x, lab, pairs, 1000, seed=13)
    assert stats.kstest(r.P, "uniform").pvalue > 1e-3
    assert 0.02 < (r.P <= 0.05).mean() < 0.09 and (r.P_maxT > 0.05).all()


# ------------------------------------------------------------------------------------------------------- CLI
def test_command_line_writes_the_pairs_and_leaves_the_other_files_alone(tmp_path, capsys):
    from g2vec_b200 import cli, graph
    from tests import helpers
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    base = ["-r", "2", "-e", "5", "-n", "20", "--seed", "3", "--deterministic"]
    a, b = str(tmp_path / "plain"), str(tmp_path / "dcx")
    cli.main([ef, cf, nf, a] + base)
    log_a = capsys.readouterr().out
    cli.main([ef, cf, nf, b] + base + ["--diff-coexpression", "200"])
    log_b = capsys.readouterr().out
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt"):
        assert open(a + suffix).read() == open(b + suffix).read(), suffix
    assert not os.path.exists(a + "_diffcoex.txt")
    import re
    untimed = lambda log, prefix: [re.sub(r" \([0-9.]+ sec\)$", "", l).replace(prefix, "RES")
                                   for l in log.splitlines()]
    extra = [l for l in untimed(log_b, b) if l not in untimed(log_a, a)]
    assert len(extra) == 3 and extra[0].startswith("Namespace(") and "diff_coexpression=200" in extra[0]
    assert extra[1].startswith("    differential co-expression: 200 label permutations of 140902 gene pairs: ")
    assert extra[2] == "    RES_diffcoex.txt"
    data = cli.load_data(ef)
    data["label"] = cli.match_labels(cli.load_clinical(cf), data["sample"])
    data, net = cli.restrict(data, cli.load_network(nf))
    gi = {g: i for i, g in enumerate(data["gene"])}
    src = np.array([gi[e[0]] for e in net["edge"]]); dst = np.array([gi[e[1]] for e in net["edge"]])
    pairs = diffcoex.pairs_from_edges(src, dst)
    r = diffcoex.diffcoex_test(data["expr"], data["label"], pairs, 200, seed=3)
    flags = []
    for grp in (0, 1):
        rp, col, _ = graph.group_csr_gpu(data["expr"], data["label"], grp, src, dst)
        rp, col = rp.cpu().numpy(), col.cpu().numpy()
        on = set()
        for u in range(len(rp) - 1):
            for v in col[rp[u]:rp[u + 1]]:
                on.add((min(u, int(v)), max(u, int(v))))
        flags.append(np.array([(int(i), int(j)) in on for i, j in pairs], np.int64))
    assert flags[0].sum() > 0 and flags[1].sum() > 0
    bm = set(open(b + "_biomarkers.txt").read().split()[1:])
    rows = open(b + "_diffcoex.txt").read().splitlines()
    assert rows[0] == "Gene1\tGene2\tR_good\tR_poor\tZ\tP\tP_maxT\tQ\tInGood\tInPoor\tBiomarkers"
    assert len(rows) == 140903
    g = data["gene"]
    nbm = np.array([(g[i] in bm) + (g[j] in bm) for i, j in pairs])
    for e in range(0, 140902, 97):
        i, j = pairs[e]
        assert rows[1 + e] == "%s\t%s\t%.6f\t%.6f\t%.6f\t%.6g\t%.6g\t%.6g\t%d\t%d\t%d" % (
            g[i], g[j], r.R_good[e], r.R_poor[e], r.Z[e], r.P[e], r.P_maxT[e], r.Q[e], flags[0][e], flags[1][e],
            nbm[e])
    got_flags = np.array([[int(c) for c in l.split("\t")[8:11]] for l in rows[1:]])
    assert (got_flags[:, 0] == flags[0]).all() and (got_flags[:, 1] == flags[1]).all() and (got_flags[:, 2] == nbm).all()
    assert extra[1] == "    " + diffcoex.summary(r, flags[0], flags[1], nbm)
