"""The k-means restarts on the H100 (csrc/g2v_km.cu, g2vec_b200/kmeans.py; DESIGN.md §4.26) against the NumPy
restatement of tests/kmeans_oracle.py.  Every comparison is bitwise: the seeds, labels, n_iter, r*, the L-groups and the
restarts that reach r*'s partition as integers, the centres, inertia and agreement as float64 bit patterns.

Tile edges of g2v_km_assign: 64 rows per CTA with 16 or more restarts, 256 rows with fewer; g2v_km_blocks sums in blocks
of 256 rows (kmeans.BLOCK)."""
import os

import numpy as np
import pytest

from g2vec_b200 import kmeans
from tests import kmeans_oracle

pytestmark = pytest.mark.gpu

B = kmeans.BLOCK


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _same(got, want, what=""):
    assert (got.seeds == want.seeds).all(), (what, "seeds", got.seeds, want.seeds)
    assert got.labels.dtype == np.int8 and (got.labels == want.labels).all(), (what, "labels")
    assert (got.n_iter == want.n_iter).all(), (what, "n_iter", got.n_iter, want.n_iter)
    assert (_bits(got.centres) == _bits(want.centres)).all(), (what, "centres")
    assert (_bits(got.inertia) == _bits(want.inertia)).all(), (what, "inertia", got.inertia, want.inertia)
    assert got.best == want.best and got.reach == want.reach, (what, got.best, want.best, got.reach, want.reach)
    assert (_bits(got.agreement) == _bits(want.agreement)).all(), (what, "agreement")
    assert got.lgroups.dtype == np.int32 and (got.lgroups == want.lgroups).all(), (what, "lgroups")


def _random(n, D, seed):
    rs = np.random.RandomState(seed)
    return (rs.standard_normal((n, D)) * np.exp2(rs.randint(-4, 4, size=(n, 1)))).astype(np.float32)


def _check(W, R, seed=0, **kw):
    want = kmeans_oracle.kmeans_lgroups(W, R, seed=seed, max_iter=kw.get("max_iter", kmeans.MAX_ITER))
    got = kmeans.kmeans_lgroups(W, R, seed=seed, **kw)
    _same(got, want, (W.shape, R, seed, kw))
    return got


@pytest.mark.parametrize("D", (1, 2, 31, 32, 33, 128, 257, 512))
def test_bitwise_equal_to_the_oracle_over_dimensions(D):
    for n, R in ((3, 2), (4, 7), (B + 1, 2), (1000, 2)):
        _check(_random(n, D, n * 1000 + D), R, seed=D)


@pytest.mark.parametrize("n", (3, 4, B - 1, B, B + 1, 63, 64, 65, 255, 257, 1000, 4097))
def test_bitwise_equal_to_the_oracle_over_rows(n):
    _check(_random(n, 33, n), 7, seed=n)
    _check(_random(n, 33, n + 1), 17, seed=n + 1)       # the 64-row tiles of 16 restarts per CTA


@pytest.mark.parametrize("R", (1, 2, 7, 64))
def test_bitwise_equal_to_the_oracle_over_restarts(R):
    _check(_random(1000, 32, R), R, seed=11)


def test_large_rows_and_dimensions():
    _check(_random(4097, 128, 5), 2, seed=5)


def _special(case):
    rs = np.random.RandomState(3)
    if case == "duplicates":                            # two distinct rows: a cluster is always empty, relocated every
        W = np.repeat(rs.standard_normal((2, 9)).astype(np.float32), [300, 3], axis=0)
    elif case == "all_equal":                           # never converges: stops at max_iter
        W = np.tile(rs.standard_normal((1, 40)).astype(np.float32), (50, 1))
    elif case == "integer_ties":                        # exact distance ties between centres
        W = rs.randint(-2, 3, size=(600, 5)).astype(np.float32)
    elif case == "power_of_two_scaling":
        base = rs.standard_normal((200, 17)).astype(np.float32)
        W = np.concatenate([np.ldexp(base, e).astype(np.float32) for e in (-30, 0, 30)])
    elif case == "zero_rows":
        W = rs.standard_normal((300, 31)).astype(np.float32)
        W[::5] = 0.0
        W[7] = -0.0
    elif case == "all_zero":
        W = np.zeros((20, 3), np.float32)
    else:
        raise KeyError(case)
    return np.ascontiguousarray(W, dtype=np.float32)


@pytest.mark.parametrize("case", ["duplicates", "all_equal", "integer_ties", "power_of_two_scaling", "zero_rows",
                                  "all_zero"])
def test_special_data_bitwise(case):
    W = _special(case)
    never = case in ("duplicates", "all_equal", "all_zero")                # iteration, so they never converge
    max_iter = 20 if never else kmeans.MAX_ITER
    got = _check(W, 7, seed=2, max_iter=max_iter)
    assert (got.n_iter == max_iter).all() == never


def test_all_equal_rows_run_to_the_default_max_iter():
    got = _check(_special("all_equal"), 2, seed=4)
    assert (got.n_iter == kmeans.MAX_ITER).all()


def test_chunked_restarts_give_the_same_bits_and_two_calls_agree():
    W = _random(3000, 40, 8)
    whole = kmeans.kmeans_lgroups(W, 23, seed=9)
    per = 9 * 3000 + 24 * 40 + 12 * (24 * 40 + 20) + 64          # one restart's bytes: 12 blocks of 256 rows
    for k in (1, 5, 16):
        part = kmeans.kmeans_lgroups(W, 23, seed=9, max_chunk_bytes=k * per)
        assert kmeans.chunk_restarts(3000, 40, 23, k * per) == k
        _same(part, whole, k)
    _same(kmeans.kmeans_lgroups(W, 23, seed=9), whole, "again")
    _same(whole, kmeans_oracle.kmeans_lgroups(W, 23, seed=9), "oracle")


def test_planted_clusters_every_restart_reaches_the_partition():
    from sklearn.cluster import KMeans
    rs = np.random.RandomState(1)
    centres = np.array([[10, 0, 0, 0], [0, 10, 0, 0], [0, 0, 10, 0]], np.float64)
    truth = np.repeat([0, 1, 2], [500, 300, 200])
    W = (centres[truth] + 0.5 * rs.standard_normal((1000, 4))).astype(np.float32)
    got = _check(W, 10, seed=6)
    assert got.reach == 10 and (got.agreement == 1.0).all()
    best = got.labels[got.best]
    assert (kmeans_oracle.contingency(best, truth) > 0).sum() == 3            # the planted partition
    sk = KMeans(n_clusters=3, random_state=0, n_init=1).fit(W).labels_
    _, hits = kmeans.match(kmeans_oracle.contingency(sk, best))
    assert hits == 1000


def test_entry_points_refuse_bad_sizes_and_launch_nothing():
    from g2vec_b200 import _capi
    lib = _capi.load()
    import torch
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p, st = buf.data_ptr(), torch.cuda.current_stream().cuda_stream
    before = _capi.launch_count()
    bad = [lib.g2v_km_assign(p, 2, 4, p, 3, p, 1, p, p, p, st), lib.g2v_km_assign(p, 10, 0, p, 3, p, 1, p, p, p, st),
           lib.g2v_km_assign(p, 10, 4, p, 0, p, 1, p, p, p, st), lib.g2v_km_assign(p, 10, 4, p, 4, p, 1, p, p, p, st),
           lib.g2v_km_assign(p, 10, 4, p, 3, p, 0, p, p, p, st), lib.g2v_km_assign(p, 10, 4, p, 3, p, 1025, p, p, p, st),
           lib.g2v_km_assign(p, 10, 4, p, 3, p, 1, None, p, None, st), lib.g2v_km_assign(None, 10, 4, p, 1, p, 1, p, p, p, st),
           lib.g2v_km_seed(p, 10, 4, p, 0, 0, 3, 1, p, p, st), lib.g2v_km_seed(p, 10, 4, None, 0, 0, 1, 1, p, p, st),
           lib.g2v_km_seed(p, 10, 4, p, 0, 1020, 0, 5, p, p, st), lib.g2v_km_seed(p, 1 + (1 << 30), 4, p, 0, 0, 0, 1, p, p, st),
           lib.g2v_km_blocks(p, p, p, 10, 4, p, 0, p, p, p, st), lib.g2v_km_blocks(p, p, p, 2, 4, p, 1, p, p, p, st),
           lib.g2v_km_update(p, p, p, p, p, 10, 4, p, 1, 0, 300, p, p, p, p, p, st),
           lib.g2v_km_update(p, p, p, p, p, 10, 4, p, 1, 301, 300, p, p, p, p, p, st),
           lib.g2v_km_contingency(p, p, 10, 0, p, st), lib.g2v_km_contingency(p, p, 2, 1, p, st),
           lib.g2v_km_agree(p, p, p, 10, 1025, p, st), lib.g2v_km_agree(p, p, None, 10, 1, p, st)]
    assert all(rc != 0 for rc in bad)
    assert _capi.launch_count() == before and len(lib.g2v_last_error()) > 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------- CLI
def test_command_line_writes_the_kmeans_file_and_leaves_the_vectors_alone(tmp_path, capsys, monkeypatch):
    from g2vec_b200 import cbow, cli
    from tests import helpers
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    base = ["-r", "2", "-e", "5", "-n", "20", "--seed", "3", "--deterministic"]
    a, b = str(tmp_path / "plain"), str(tmp_path / "km")
    cli.main([ef, cf, nf, a] + base)
    log_a = capsys.readouterr().out
    captured = []
    train = cbow.train_cbow

    def wrapped(*args, **kw):
        out = train(*args, **kw)
        captured.append(np.array(out, copy=True))
        return out
    monkeypatch.setattr(cbow, "train_cbow", wrapped)
    cli.main([ef, cf, nf, b] + base + ["--kmeans-restarts", "8"])
    log_b = capsys.readouterr().out
    assert open(a + "_vectors.txt").read() == open(b + "_vectors.txt").read()
    assert not os.path.exists(a + "_kmeans.txt") and "k-means:" not in log_a
    import re
    untimed = lambda log, prefix: [re.sub(r" \([0-9.]+ sec\)$", "", l).replace(prefix, "RES")
                                   for l in log.splitlines()]
    la, lb = untimed(log_a, a), untimed(log_b, b)
    assert "kmeans_restarts=0" in la[1] and "kmeans_restarts=8" in lb[1]
    mat = captured[0]
    want = kmeans_oracle.kmeans_lgroups(mat, 8, seed=3)
    names = np.array([l.split("\t")[0] for l in open(b + "_lgroups.txt").read().splitlines()[1:]])
    lg = np.array([int(l.split("\t")[1]) for l in open(b + "_lgroups.txt").read().splitlines()[1:]])
    assert (lg == want.lgroups).all()
    line = kmeans.summary(want)
    extra = [l for l in lb if l not in la]
    assert len(lb) == len(la) + 2 and len(extra) == 3 and extra[0].startswith("Namespace(")
    assert extra[1] == "    " + line and extra[2] == "    RES_kmeans.txt"
    body = open(b + "_kmeans.txt").read()
    assert body == ("GeneSymbol\tLgroup(0:good,1:poor,2:other)\tAgreement\n"
                    + "".join("%s\t%d\t%.6f\n" % (g, k, x) for g, k, x in zip(names, want.lgroups, want.agreement))
                    + line + "\n")
