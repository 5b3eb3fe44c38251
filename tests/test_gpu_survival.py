"""The permutation Cox score test on the H100 (csrc/g2v_surv.cu, g2vec_b200/survival.py; DESIGN.md §4.31) against the
NumPy restatement of tests/survival_oracle.py.  Every comparison is bit for bit."""
import os

import numpy as np
import pytest

from g2vec_b200 import survival
from tests import survival_oracle

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


# The device copies are held in locals until the result is back.
def gpu_rows(slot, seed, b_begin, n_b):
    import torch
    capi, lib = _lib()
    n = len(slot)
    idx = torch.zeros((n_b, n), dtype=torch.uint16, device="cuda")
    s = _dev(np.asarray(slot, np.int32))
    capi.check(lib.g2v_surv_rows(s.data_ptr(), n, seed & 0xFFFFFFFFFFFFFFFF, b_begin, n_b, idx.data_ptr(), _st()),
               "g2v_surv_rows")
    return idx.cpu().numpy()


def gpu_scores(q, idx, flags, a, c):
    import torch
    capi, lib = _lib()
    n_b, n = idx.shape
    G = q.shape[1]
    T = torch.full((n_b, G), np.nan, dtype=torch.float64, device="cuda")
    UV = torch.full((2, n_b, G), np.nan, dtype=torch.float64, device="cuda")
    d = [_dev(x) for x in (np.asarray(q, np.int32), np.asarray(idx, np.uint16), flags, a, c)]
    capi.check(lib.g2v_surv_scores(d[0].data_ptr(), n, G, d[1].data_ptr(), n_b, d[2].data_ptr(), d[3].data_ptr(),
                                   d[4].data_ptr(), T.data_ptr(), UV.data_ptr(), _st()), "g2v_surv_scores")
    UV = UV.cpu().numpy()
    return T.cpu().numpy(), UV[0], UV[1]


def _records(rs, n, kind="random"):
    t = np.round(rs.exponential(10.0, n), 1)
    e = (rs.rand(n) < 0.6).astype(np.int64)
    if kind == "tied":                                  # every time equal
        t[:] = 5.0
    elif kind == "one_event":                           # every sample censored but one
        e[:] = 0; e[rs.randint(n)] = 1
    elif kind == "earliest":                            # events only at the earliest times
        e = (t <= np.quantile(t, 0.2)).astype(np.int64)
    elif kind == "latest":                              # events only at the latest times
        e = (t >= np.quantile(t, 0.8)).astype(np.int64)
    if kind in ("random", "tied"):
        e[np.argmin(t)] = 1                             # at least one event
    return t, e


# ------------------------------------------------------------------------------------------------------ rows
@pytest.mark.parametrize("n,b0,nb", [(3, 0, 1), (31, 5, 33), (32, 0, 7), (33, 100, 40), (1000, 0, 65),
                                     (32768, 1000, 3)])
def test_rows_equal_the_oracle_and_carry_the_permutation_labels(n, b0, nb):
    import torch
    capi, lib = _lib()
    rs = np.random.RandomState(n)
    t, e = _records(rs, n)
    order, slot, _, _, _ = survival.time_groups(t, e)
    seed = 12345678901
    got = gpu_rows(slot, seed, b0, nb)
    assert (got == survival_oracle.rows(slot, seed, b0, nb)).all()
    pi = order[np.argsort(got.astype(np.int64), axis=1)]   # pi_b(s) = order[the position holding s]
    obs = (rs.rand(n) < 0.5).astype(np.uint8)
    S_pad = -(-n // 32) * 32
    M = torch.empty((nb, S_pad), dtype=torch.uint8, device="cuda")
    o = _dev(obs)
    capi.check(lib.g2v_perm_labels(o.data_ptr(), n, S_pad, seed, b0, nb, M.data_ptr(), _st()), "g2v_perm_labels")
    assert (obs[pi] == M.cpu().numpy()[:, :n]).all()


# ------------------------------------------------------------------------------------------------------ scores
# genes around the 32-gene warp tile, rows around the 8-permutation CTA, samples around the 32-position and 8-step
# batches of the scan
SCORE_SHAPES = [(n, G, nb) for n in (3, 7, 8, 9, 31, 32, 33, 135) for G in (1, 31, 32, 33, 100) for nb in (1, 7, 8, 9)]
SCORE_SHAPES += [(1000, 65, 17), (32768, 40, 2)]


def _score_case(rs, n, G, nb, kind="random"):
    t, e = _records(rs, n, kind)
    order, slot, flags, a, c = survival.time_groups(t, e)
    q = rs.randint(-(1 << 16), (1 << 16) + 1, size=(n, G)).astype(np.int64)
    idx = np.vstack([order[None, :].astype(np.uint16), survival_oracle.rows(slot, 3, 0, nb - 1)]) if nb > 1 else \
        order[None, :].astype(np.uint16)
    return q, idx, flags, a, c


def _check(q, idx, flags, a, c):
    got, want = gpu_scores(q, idx, flags, a, c), survival_oracle.scan(q, idx, flags, a, c)
    for g_, w_ in zip(got, want):
        assert np.array_equal(g_, w_)
    return want


def test_scores_equal_the_oracle_at_every_tile_edge():
    rs = np.random.RandomState(0)
    for n, G, nb in SCORE_SHAPES:
        _check(*_score_case(rs, n, G, nb))


@pytest.mark.parametrize("kind", ["tied", "one_event", "earliest", "latest"])
@pytest.mark.parametrize("n", [3, 33, 135, 32768])
def test_scores_equal_the_oracle_on_special_records(kind, n):
    rs = np.random.RandomState(n + len(kind))
    T, U, V = _check(*_score_case(rs, n, 37, 3, kind))
    assert (V >= 0).all() and np.isfinite(T).all()


def test_scores_are_exact_at_the_magnitude_bound():
    """q = +-2^16 on 32768 samples: S0 S2 = 2^62 and |S1| = 2^31 at the last position."""
    n, v = 32768, 1 << 16
    rs = np.random.RandomState(1)
    t = rs.permutation(n).astype(np.float64)
    e = np.ones(n, np.int64)
    order, slot, flags, a, c = survival.time_groups(t, e)
    q = np.empty((n, 4), np.int64)
    q[:, 0] = v; q[:, 1] = -v
    q[:, 2] = np.where(t < n // 2, v, -v)              # the earliest half at +2^16: num_u at its extreme
    q[:, 3] = np.where(rs.rand(n) < 0.5, v, -v)
    idx = np.vstack([order, survival_oracle.rows(slot, 9, 0, 2)]).astype(np.uint16)
    T, U, V = _check(q, idx, flags, a, c)
    assert (V[:, :2] == 0).all() and (V[:, 2:] > 0).all() and T[0, 2] > 100


def test_counts_equal_the_oracle_in_any_chunking_and_run():
    from g2vec_b200 import _capi
    rs = np.random.RandomState(2)
    n, G = 70, 90
    x = rs.standard_normal((n, G))
    t, e = _records(rs, n)
    B = 150
    want = survival_oracle.survival_test(x, t, e, B, seed=-4, chunk=40)
    for max_bytes, chunks in ((1, B), ((2 * n + 8 * G) * 64, 3), (None, 1), (None, 1)):
        before = _capi.launch_count()
        got = survival.survival_test(x, t, e, B, seed=-4, max_chunk_bytes=max_bytes)
        assert _capi.launch_count() - before == 1 + 3 * chunks
        _same(got, want)


def _same(a, b):
    for f in ("count", "count_maxt", "order"):
        assert (getattr(a, f) == getattr(b, f)).all(), f
    for f in ("Z", "T", "P_score", "P", "P_maxT", "Q"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    assert (a.n_perm, a.n, a.n_events) == (b.n_perm, b.n, b.n_events)


def _ex_records(n, seed=20):
    rs = np.random.RandomState(seed)
    t = np.round(rs.exponential(36.0, n), 1)            # months, with ties
    e = (rs.rand(n) < 0.45).astype(np.int64)
    return t, e


def test_survival_test_equals_the_oracle_on_the_example_cohort():
    from tests.helpers import GOLDEN
    x = np.load(os.path.join(GOLDEN, "ex_expr.npz"))["expr"]
    t, e = _ex_records(x.shape[0])
    B = 100
    _same(survival.survival_test(x, t, e, B, seed=3), survival_oracle.survival_test(x, t, e, B, seed=3))


def test_planted_prognostic_gene_gets_the_smallest_p_value():
    rs = np.random.RandomState(3)
    n, G = 135, 300
    x = rs.standard_normal((n, G))
    hazard = np.exp(1.5 * x[:, 42])
    t = rs.exponential(1.0 / hazard)
    cens = rs.exponential(2.0, n)
    e = (t <= cens).astype(np.int64); t = np.minimum(t, cens)
    B = 2000
    r = survival.survival_test(x, t, e, B, seed=1)
    assert r.order[0] == 42 and r.P[42] == r.P_maxT[42] == 1.0 / (B + 1) and r.Z[42] > 5
    assert r.P_score[42] < 1e-6


def test_null_p_values_are_roughly_uniform():
    from scipy import stats
    rs = np.random.RandomState(13)
    n, G = 80, 400
    x = rs.standard_normal((n, G))
    t, e = _ex_records(n, 13)
    r = survival.survival_test(x, t, e, 1000, seed=13)
    assert stats.kstest(r.P, "uniform").pvalue > 1e-3
    assert 0.02 < (r.P <= 0.05).mean() < 0.09 and (r.P_maxT > 0.05).all()
    assert np.abs(r.P - r.P_score).max() < 0.1         # the permutation and the asymptotic p-values agree


def test_entry_points_refuse_bad_sizes_and_launch_nothing():
    capi, lib = _lib()
    import torch
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p, st = buf.data_ptr(), _st()
    N = None
    before = capi.launch_count()
    bad = [lib.g2v_surv_rows(N, 10, 0, 0, 1, p, st), lib.g2v_surv_rows(p, 10, 0, 0, 1, N, st),
           lib.g2v_surv_rows(p, 2, 0, 0, 1, p, st), lib.g2v_surv_rows(p, 32769, 0, 0, 1, p, st),
           lib.g2v_surv_rows(p, 10, 0, 0, 0, p, st), lib.g2v_surv_rows(p, 10, 0, -1, 1, p, st),
           lib.g2v_surv_rows(p, 10, 0, 1 << 20, 1, p, st),
           lib.g2v_surv_scores(N, 10, 1, p, 1, p, p, p, p, N, st), lib.g2v_surv_scores(p, 10, 1, N, 1, p, p, p, p, N, st),
           lib.g2v_surv_scores(p, 10, 1, p, 1, N, p, p, p, N, st), lib.g2v_surv_scores(p, 10, 1, p, 1, p, N, p, p, N, st),
           lib.g2v_surv_scores(p, 10, 1, p, 1, p, p, N, p, N, st), lib.g2v_surv_scores(p, 10, 1, p, 1, p, p, p, N, N, st),
           lib.g2v_surv_scores(p, 2, 1, p, 1, p, p, p, p, N, st), lib.g2v_surv_scores(p, 32769, 1, p, 1, p, p, p, p, N, st),
           lib.g2v_surv_scores(p, 10, 0, p, 1, p, p, p, p, N, st),
           lib.g2v_surv_scores(p, 10, (1 << 20) + 1, p, 1, p, p, p, p, N, st),
           lib.g2v_surv_scores(p, 10, 1, p, 0, p, p, p, p, N, st),
           lib.g2v_surv_scores(p, 10, 1, p, (1 << 20) + 1, p, p, p, p, N, st)]
    assert all(rc != 0 for rc in bad)
    assert capi.launch_count() == before and len(lib.g2v_last_error()) > 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------- CLI
def test_command_line_writes_the_genes_and_leaves_the_other_files_alone(tmp_path, capsys):
    import re
    from g2vec_b200 import cli
    from tests import helpers
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    samples = ["TCGA-%04d" % i for i in range(135)]
    t, e = _ex_records(135, 7)
    sf = str(tmp_path / "S.txt")
    with open(sf, "w") as f:
        f.write("PATIENT\tOS_MONTHS\tOS_EVENT\tSTAGE\n")
        for i, s in enumerate(samples):
            tt = "NA" if i % 17 == 3 else repr(float(t[i]))
            ee = "" if i % 23 == 5 else str(int(e[i]))
            f.write("%s\t%s\t%s\tII\n" % (s, tt, ee))
        f.write("NOT_IN_EXPRESSION\t3.0\t1\tIV\n")
    base = ["-r", "2", "-e", "5", "-n", "20", "--seed", "3", "--deterministic"]
    a, b = str(tmp_path / "plain"), str(tmp_path / "surv")
    cli.main([ef, cf, nf, a] + base)
    log_a = capsys.readouterr().out
    cli.main([ef, cf, nf, b] + base + ["--survival", sf, "--survival-permutations", "200"])
    log_b = capsys.readouterr().out
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt"):
        assert open(a + suffix).read() == open(b + suffix).read(), suffix
    assert not os.path.exists(a + "_survival.txt")
    untimed = lambda log, prefix: [re.sub(r" \([0-9.]+ sec\)$", "", l).replace(prefix, "RES")
                                   for l in log.splitlines()]
    extra = [l for l in untimed(log_b, b) if l not in untimed(log_a, a)]
    used = np.array([not (i % 17 == 3 or i % 23 == 5) for i in range(135)])
    assert len(extra) == 4 and extra[0].startswith("Namespace(") and "survival_permutations=200" in extra[0]
    assert extra[1] == "    survival: %d of 135 samples with a record, %d events, in %s" % (used.sum(), e[used].sum(), sf)
    assert extra[2].startswith("    survival: 200 permutations of %d samples (%d events): " % (used.sum(), e[used].sum()))
    assert extra[3] == "    RES_survival.txt"
    data = cli.load_data(ef)
    data["label"] = cli.match_labels(cli.load_clinical(cf), data["sample"])
    data, _ = cli.restrict(data, cli.load_network(nf))
    r = survival.survival_test(data["expr"][used], t[used], e[used], 200, seed=3)
    bm = set(open(b + "_biomarkers.txt").read().split()[1:])
    lg = [int(l.split("\t")[1]) for l in open(b + "_lgroups.txt").read().splitlines()[1:]]
    rows = open(b + "_survival.txt").read().splitlines()
    assert rows[0] == "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tZ\tP_score\tP\tP_maxT\tQ\tBiomarker"
    g = data["gene"]
    assert len(rows) == len(g) + 1
    for i in range(len(g)):
        assert rows[1 + i] == "%s\t%d\t%.6f\t%.6g\t%.6g\t%.6g\t%.6g\t%d" % (
            g[i], lg[i], r.Z[i], r.P_score[i], r.P[i], r.P_maxT[i], r.Q[i], g[i] in bm)
    lz, lp = survival.label_score(data["label"][used], t[used], e[used])
    assert extra[2] == "    " + survival.summary(r, np.array([x in bm for x in g]), lz, lp)


def test_command_line_refuses_a_bad_survival_file_before_the_walks(tmp_path, capsys):
    from g2vec_b200 import cli
    from tests import helpers
    ef, cf, nf, _ = helpers.write_ex_tsv(tmp_path)
    sf = str(tmp_path / "S.txt")
    with open(sf, "w") as f:
        f.write("SAMPLE\tTIME\tEVENT\n" + "".join("TCGA-%04d\t%d\t0\n" % (i, i) for i in range(135)))
    with pytest.raises(SystemExit) as ex:
        cli.main([ef, cf, nf, str(tmp_path / "R"), "--survival", sf])
    out = capsys.readouterr().out
    assert ex.value.code == 1 and "ERROR: --survival: no events" in out and ">>> 3." not in out
