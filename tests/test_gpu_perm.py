"""The label-permutation test on the H100 (csrc/g2v_perm.cu, g2vec_b200/perm.py; DESIGN.md §4.24) against the NumPy
restatement of tests/perm_oracle.py.  Every comparison is exact unless it says otherwise: the counts are integers."""
import os

import numpy as np
import pytest

from g2vec_b200 import perm
from tests import perm_oracle
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


# The device copies are held in locals until the result is back: a temporary freed before the kernel runs could
# hand its block to the next upload.
def gpu_labels(obs, S_pad, seed, b_begin, n_b):
    import torch
    capi, lib = _lib()
    M = torch.full((n_b, S_pad), 7, dtype=torch.uint8, device="cuda")       # padding must be written as 0
    od = _dev(obs)
    capi.check(lib.g2v_perm_labels(od.data_ptr(), len(obs), S_pad, seed, b_begin, n_b, M.data_ptr(), _st()),
               "g2v_perm_labels")
    return M.cpu().numpy()


def gpu_sums(M, pl):
    import torch
    capi, lib = _lib()
    n_b, S_pad = M.shape
    G = pl.shape[1]
    A = torch.empty((n_b, G), dtype=torch.int64, device="cuda")
    Md, pd = _dev(M), _dev(pl)
    capi.check(lib.g2v_perm_sums(Md.data_ptr(), pd.data_ptr(), n_b, S_pad, G, A.data_ptr(), _st()), "g2v_perm_sums")
    return A.cpu().numpy()


def gpu_tally(A, n, k, Q, W, absN, rho):
    import torch
    capi, lib = _lib()
    n_b, G = A.shape
    c = torch.zeros(G, dtype=torch.int64, device="cuda")
    cm = torch.zeros(G, dtype=torch.int64, device="cuda")
    d = [_dev(a) for a in (A, Q, W, absN, rho)]
    capi.check(lib.g2v_perm_tally(d[0].data_ptr(), n_b, G, n, k, d[1].data_ptr(), d[2].data_ptr(), d[3].data_ptr(),
                                  d[4].data_ptr(), c.data_ptr(), cm.data_ptr(), _st()), "g2v_perm_tally")
    return c.cpu().numpy(), cm.cpu().numpy()


# ---------------------------------------------------------------------------------------------------- labels
@pytest.mark.parametrize("n", [3, 31, 32, 33, 135, 1000, 4097, 32768])
def test_labels_equal_the_oracle(n):
    S_pad = -(-n // 32) * 32
    n_b = 5 if n > 5000 else 40                         # rows 3 and 4 are compared with a chunk below
    for k in sorted({1, n // 2, n - 1}):
        obs = np.zeros(n, np.uint8); obs[np.random.RandomState(n + k).choice(n, k, replace=False)] = 1
        got = gpu_labels(obs, S_pad, 987654321, 10, n_b)
        assert (got == perm_oracle.labels(obs, S_pad, 987654321, 10, n_b)).all(), (n, k)
        assert (got.sum(axis=1) == k).all() and (got[:, n:] == 0).all()
        part = gpu_labels(obs, S_pad, 987654321, 13, 2)                              # chunk offsets
        assert (part == got[3:5]).all(), (n, k, np.nonzero((part != got[3:5]).any(axis=1))[0],
                                          int((part != got[3:5]).sum()), part.sum(axis=1))


def test_labels_are_uniform_over_the_subsets():
    """n = 4, k = 2: the 6 subsets from 60 000 permutations, chi-square not rejected at 1e-3 (seeded, so the
    outcome is fixed)."""
    from scipy import stats
    M = gpu_labels(np.array([1, 1, 0, 0], np.uint8), 32, 2024, 0, 60000)[:, :4]
    code = M @ np.array([8, 4, 2, 1])
    counts = np.array([(code == c).sum() for c in (3, 5, 6, 9, 10, 12)])
    assert counts.sum() == 60000
    assert stats.chisquare(counts).pvalue > 1e-3


def test_entry_points_refuse_bad_sizes_and_launch_nothing():
    capi, lib = _lib()
    import torch
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p, st = buf.data_ptr(), _st()
    before = capi.launch_count()
    bad = [lib.g2v_perm_labels(p, 2, 32, 0, 0, 1, p, st), lib.g2v_perm_labels(p, 33, 32, 0, 0, 1, p, st),
           lib.g2v_perm_labels(p, 40, 48, 0, 0, 1, p, st), lib.g2v_perm_labels(p, 32769, 32800, 0, 0, 1, p, st),
           lib.g2v_perm_labels(p, 40, 64, 0, 0, 0, p, st), lib.g2v_perm_labels(p, 40, 64, 0, (1 << 24) - 1, 2, p, st),
           lib.g2v_perm_sums(p, p, 0, 32, 1, p, st), lib.g2v_perm_sums(p, p, 1, 16, 1, p, st),
           lib.g2v_perm_sums(p, p, 1, 32, 0, p, st), lib.g2v_perm_sums(p, p, 1, 32, 65535 * 64 + 1, p, st),
           lib.g2v_perm_tally(p, 1, 1, 2, 1, p, p, p, p, p, p, st), lib.g2v_perm_tally(p, 1, 1, 10, 10, p, p, p, p, p, p, st),
           lib.g2v_perm_tally(p, 1, 1, 10, 0, p, p, p, p, p, p, st), lib.g2v_perm_tally(p, 0, 1, 10, 3, p, p, p, p, p, p, st),
           lib.g2v_perm_tally(p, 1, 0, 10, 3, p, p, p, p, p, p, st)]
    assert all(rc != 0 for rc in bad)
    assert capi.launch_count() == before and len(lib.g2v_last_error()) > 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------ sums
def _random_planes(rs, n, G, S_pad, lo=-(1 << 22), hi=(1 << 22)):
    q = rs.randint(lo, hi + 1, size=(n, G)).astype(np.int64)
    return q, perm.planes(q, np.arange(G))


SUM_SHAPES = [(nb, G, S) for S in (32, 64, 160) for nb in (1, 15, 16, 17, 129, 257) for G in (1, 15, 16, 17, 129, 257)]
SUM_SHAPES += [(1, 1, 32768), (15, 17, 32768), (17, 16, 32768), (129, 15, 32768), (16, 129, 32768)]


def test_sums_equal_the_int64_matmul_at_every_tile_edge():
    rs = np.random.RandomState(0)
    for nb, G, S_pad in SUM_SHAPES:
        n = S_pad - rs.randint(0, 32) if S_pad > 32 else S_pad - rs.randint(0, 29)
        q, pl = _random_planes(rs, n, G, S_pad)
        M = np.zeros((nb, S_pad), np.uint8); M[:, :n] = rs.randint(0, 2, size=(nb, n))
        assert (gpu_sums(M, pl) == perm_oracle.sums(M, q)).all(), (nb, G, S_pad)


def test_sums_do_not_overflow_at_the_extremes():
    S_pad, G, nb = 32768, 20, 70
    for v in (1 << 22, -(1 << 22)):
        q = np.full((S_pad, G), v, np.int64)
        q[:, 3] = (1 << 22) - 1                         # every byte plane at 255 / 127 in one gene
        q[:, 4] = -(1 << 22) + 1
        M = np.ones((nb, S_pad), np.uint8)
        got = gpu_sums(M, perm.planes(q, np.arange(G)))
        assert (got == q.sum(axis=0)[None, :]).all()
        assert got[0, 0] == S_pad * v


# ----------------------------------------------------------------------------------------------------- tally
def _tally_case(rs, n, G, nb):
    x, lab = cohort(n, G, int(rs.randint(1 << 30)), n // 3)
    x[:, 1] = 2.0                                       # constant gene: W = 0, rho = 0
    x[:, 2] = (lab == 1) * 3.0                          # perfect separation: rho_obs = 1
    if G > 9:
        x[:, 5] = x[:, 9]                               # equal rho_obs
    prep = perm.prepare(x, lab)
    o = prep["order"]
    M = perm_oracle.labels(prep["obs"], -(-n // 32) * 32, 5, 0, nb)
    A = perm_oracle.sums(M, prep["q"][:, o])
    absN = np.abs(prep["N_obs"][o])
    N1 = n * A[nb // 2] - prep["k"] * prep["Q"][o]      # ties |N| = |N_obs| on every gene of one row
    absN[::2] = np.abs(N1[::2])
    rho = prep["rho_obs"][o].copy()
    rho[1::3] = perm.rho_of(N1, prep["W"][o])[1::3]     # and u = rho_obs ties
    return A, n, prep["k"], prep["Q"][o], prep["W"][o], absN, rho


@pytest.mark.parametrize("n,G,nb", [(12, 7, 1), (40, 127, 9), (135, 128, 64), (135, 129, 300), (60, 1000, 1000),
                                    (33, 3000, 2500)])
def test_tally_equals_the_oracle(n, G, nb):
    args = _tally_case(np.random.RandomState(G + nb), n, G, nb)
    got = gpu_tally(*args)
    want = perm_oracle.tally(*args)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
    assert want[0].max() > 0 and want[1].max() > 0


# ------------------------------------------------------------------------------------------------- perm_test
def _ex():
    from tests.helpers import GOLDEN
    e = np.load(os.path.join(GOLDEN, "ex_expr.npz"))
    return e["expr"], np.load(os.path.join(GOLDEN, "ex_graph.npz"))["label"]


def _same(a, b):
    for f in ("count", "count_maxt", "order"):
        assert (getattr(a, f) == getattr(b, f)).all(), f
    for f in ("T", "P", "P_maxT", "Q"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f


def test_perm_test_equals_the_oracle_on_ex_and_in_any_chunking():
    from g2vec_b200 import _capi
    x, lab = _ex()
    B = 200
    want = perm_oracle.perm_test(x, lab, B, seed=3, chunk=77)
    n, G = 135, x.shape[1]
    row = 160 + 8 * G
    for max_bytes, chunks in ((row, B), (row * 70, 3), (None, 1)):
        before = _capi.launch_count()
        got = perm.perm_test(x, lab, B, seed=3, max_chunk_bytes=max_bytes)
        assert _capi.launch_count() - before == 3 * chunks
        _same(got, want)
    assert (got.P_maxT >= got.P).all() and (np.diff(got.P_maxT[got.order]) >= 0).all()
    assert n == int(((lab == 0) | (lab == 1)).sum())


def test_perm_test_equals_the_oracle_on_a_synthetic_cohort():
    x, lab = cohort(301, 700, 11, 120)
    x[:, 0] = 1.0
    lab[:4] = 5                                         # left out
    x[0, 3] = np.nan                                    # in a left-out sample: ignored
    _same(perm.perm_test(x, lab, 999, seed=-7, max_chunk_bytes=300 * (320 + 8 * 700)),
          perm_oracle.perm_test(x, lab, 999, seed=-7))


def test_planted_gene_gets_the_smallest_p_values():
    x, lab = cohort(200, 500, 12, 100)
    x[:, 42] = np.random.RandomState(0).standard_normal(200) + 4.0 * lab
    B = 5000
    r = perm.perm_test(x, lab, B, seed=1)
    assert r.P[42] == r.P_maxT[42] == 1.0 / (B + 1) and r.order[0] == 42
    assert (r.P_maxT >= r.P).all()


def test_null_p_values_agree_with_the_t_distribution():
    """Gaussian null data, B = 20 000: each permutation P lies within 5 binomial sigma + 1/B of ttest_ind's p."""
    from scipy import stats
    rs = np.random.RandomState(13)
    n, G, B = 60, 200, 20000
    x = rs.standard_normal((n, G))
    lab = np.array([0] * 27 + [1] * 33)
    r = perm.perm_test(x, lab, B, seed=13)
    p = stats.ttest_ind(x[lab == 0], x[lab == 1]).pvalue
    assert (np.abs(r.P - p) <= 5 * np.sqrt(p * (1 - p) / B) + 1.0 / B).all()
    assert np.allclose(r.T, np.abs(stats.ttest_ind(x[lab == 0], x[lab == 1]).statistic), rtol=1e-5, atol=1e-4)


# ------------------------------------------------------------------------------------------------------- CLI
def test_command_line_writes_the_pvalues_and_leaves_the_other_files_alone(tmp_path, capsys):
    from g2vec_b200 import cli
    from tests import helpers
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    base = ["-r", "2", "-e", "5", "-n", "20", "--seed", "3", "--deterministic"]
    a, b = str(tmp_path / "plain"), str(tmp_path / "perm")
    cli.main([ef, cf, nf, a] + base)
    log_a = capsys.readouterr().out
    cli.main([ef, cf, nf, b] + base + ["--permutations", "200"])
    log_b = capsys.readouterr().out
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt"):
        assert open(a + suffix).read() == open(b + suffix).read(), suffix
    assert not os.path.exists(a + "_pvalues.txt")
    import re
    untimed = lambda log, prefix: [re.sub(r" \([0-9.]+ sec\)$", "", l).replace(prefix, "RES")
                                   for l in log.splitlines()]
    extra = [l for l in untimed(log_b, b) if l not in untimed(log_a, a)]
    assert len(extra) == 3 and extra[0].startswith("Namespace(") and "permutations=200" in extra[0]
    assert extra[1].startswith("    permutation test: 200 label permutations: ") and extra[2] == "    RES_pvalues.txt"
    data = cli.load_data(ef)
    data["label"] = cli.match_labels(cli.load_clinical(cf), data["sample"])
    data, _ = cli.restrict(data, cli.load_network(nf))
    r = perm.perm_test(data["expr"], data["label"], 200, seed=3)
    bm = set(open(b + "_biomarkers.txt").read().split()[1:])
    lg = [l.split("\t") for l in open(b + "_lgroups.txt").read().splitlines()[1:]]
    rows = open(b + "_pvalues.txt").read().splitlines()
    assert rows[0] == "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tT\tP\tP_maxT\tQ\tBiomarker" and len(rows) == 7524
    for i, line in enumerate(rows[1:]):
        assert line == "%s\t%s\t%.6f\t%.6g\t%.6g\t%.6g\t%d" % (lg[i][0], lg[i][1], r.T[i], r.P[i], r.P_maxT[i], r.Q[i],
                                                            lg[i][0] in bm)
    n_sig = int((r.P_maxT <= 0.05).sum())
    assert extra[1].endswith("%d genes with P_maxT <= 0.05 (%d of the biomarkers)"
                             % (n_sig, len(set(data["gene"][r.P_maxT <= 0.05]) & bm)))
