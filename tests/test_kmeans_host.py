"""CPU checks of the k-means restarts (DESIGN.md §4.26): the oracle of tests/kmeans_oracle.py against plain Python
float arithmetic, big-integer seeding, a Python loop over the blocked sums and brute-force matching; the naming helper
against the old find_lgroups; every refusal of kmeans_lgroups (raised before the library is loaded), the
--kmeans-restarts option and the _kmeans.txt writer."""
import itertools

import numpy as np
import pytest

from g2vec_b200 import cli, kmeans
from tests import kmeans_oracle


def _python_dist(x, c):
    acc = 0.0
    for a, b in zip(x, c):
        t = float(a) - float(b)
        acc = acc + t * t
    return acc


@pytest.mark.parametrize("n,D,seed", [(3, 1, 0), (5, 7, 1), (9, 40, 2)])
def test_distance_chain_equals_python_floats(n, D, seed):
    rs = np.random.RandomState(seed)
    X = (rs.standard_normal((n, D)) * np.exp2(rs.randint(-20, 20, size=(n, 1)))).astype(np.float32).astype(np.float64)
    C = rs.standard_normal((3, D)) * 3.0
    got = kmeans_oracle.dist(X, C)
    for i in range(n):
        for c in range(3):
            assert got[i, c] == _python_dist(X[i], C[c])


def test_chain_starts_from_plus_zero_and_runs_in_order():
    assert not np.signbit(kmeans_oracle.chain(np.array([-0.0, -0.0])))
    a = np.array([1e16, 1.0, -1e16, 1.0])
    assert kmeans_oracle.chain(a) == ((((0.0 + 1e16) + 1.0) + -1e16) + 1.0)


def test_blocked_sums_equal_a_python_loop_in_the_contract_order():
    rs = np.random.RandomState(3)
    n = 2 * kmeans.BLOCK + 17
    v = rs.standard_normal(n) * np.exp2(rs.randint(-30, 30, size=n))
    total = 0.0
    for b0 in range(0, n, kmeans.BLOCK):
        part = 0.0
        for i in range(b0, min(n, b0 + kmeans.BLOCK)):
            part = part + float(v[i])
        total = total + part
    assert kmeans_oracle.blocked(v) == total
    M = rs.standard_normal((n, 3))
    got = kmeans_oracle.blocked(M)
    for d in range(3):
        assert got[d] == kmeans_oracle.blocked(M[:, d])


def _bigint_seed_rows(X, seed, r):
    n = X.shape[0]
    u = kmeans_oracle.draws(seed, r)
    rows = [u[0] * n // 2 ** 64]
    for t in (1, 2):
        Dm = [min(_python_dist(X[i], X[j]) for j in rows) for i in range(n)]
        mx = max(Dm)
        if mx == 0.0:
            rows.append(u[t] * n // 2 ** 64)
            continue
        q = [int((d / mx) * 2.0 ** 32) for d in Dm]
        target = u[t] * sum(q) // 2 ** 64
        acc = 0
        for i, qi in enumerate(q):
            acc += qi
            if acc > target:
                rows.append(i)
                break
    return rows


@pytest.mark.parametrize("case", ["gauss", "ints", "dup", "zeros"])
def test_seeding_equals_the_big_integer_form(case):
    rs = np.random.RandomState(4)
    X = {"gauss": rs.standard_normal((60, 5)), "ints": rs.randint(-1, 2, size=(40, 3)).astype(float),
         "dup": np.repeat(rs.standard_normal((2, 4)), [20, 1], axis=0), "zeros": np.zeros((7, 2))}[case]
    X = X.astype(np.float32).astype(np.float64)
    for seed in (0, 5, (1 << 64) - 1):
        for r in (0, 1, 1023):
            assert kmeans_oracle.seed_rows(X, seed, r) == _bigint_seed_rows(X, seed, r)


def test_matching_equals_brute_force():
    rs = np.random.RandomState(5)
    for _ in range(200):
        n = int(rs.randint(3, 12))
        a, b = rs.randint(0, 3, n), rs.randint(0, 3, n)
        p, hits = kmeans.match(kmeans_oracle.contingency(a, b))
        scores = [int((np.array(q)[a] == b).sum()) for q in itertools.permutations((0, 1, 2))]
        assert hits == max(scores) and p == list(itertools.permutations((0, 1, 2)))[scores.index(max(scores))]


def test_oracle_lloyd_relocates_and_stops():
    X = np.repeat(np.array([[0.0, 0.0], [1.0, 0.0]]), [5, 1], axis=0)     # two distinct rows: a cluster stays empty
    a, C, it, inertia = kmeans_oracle.lloyd(X, X[[0, 0, 0]], max_iter=9)
    assert it == 9 and list(np.bincount(a, minlength=3)) == [5, 1, 0] and (C[1] == [1.0, 0.0]).all()
    X = np.array([[0.0], [0.0], [1.0], [5.0], [6.0]])
    a, C, it, inertia = kmeans_oracle.lloyd(X, X[[0, 1, 2]])                # centres 0 and 1 coincide: relocation
    assert it == 4 and list(a) == [0, 0, 2, 1, 1] and list(C[:, 0]) == [0.0, 5.5, 1.0] and inertia == 0.5
    a, C, it, inertia = kmeans_oracle.lloyd(np.zeros((4, 2)), np.zeros((3, 2)), max_iter=7)
    assert it == 7 and inertia == 0.0 and (a == 0).all()


# ------------------------------------------------------------------------------------------------- naming
def _old_find_lgroups(km):
    sizes = [int(np.count_nonzero(km == k)) for k in range(3)]
    largest = 0
    for k in (1, 2):
        if sizes[k] > sizes[largest]:
            largest = k
    rest = [k for k in (0, 1, 2) if k != largest]
    out = np.zeros(km.shape[0], dtype=np.int32)
    out[km == rest[1]] = 0
    out[km == rest[0]] = 1
    out[km == largest] = 2
    return out


def test_naming_helper_gives_the_old_find_lgroups_output():
    from sklearn.cluster import KMeans
    rs = np.random.RandomState(6)
    for n in (10, 57, 300):
        mat = rs.standard_normal((n, 8)).astype(np.float32)
        km = KMeans(n_clusters=3, random_state=0).fit(mat).labels_
        assert (kmeans.name_lgroups(km) == _old_find_lgroups(km)).all()
        assert (cli.find_lgroups(mat, None, None) == _old_find_lgroups(km)).all()
    for lab in ([0, 1, 2], [2, 2, 1, 1, 0], [1, 1, 0, 0, 2, 2], [0, 0, 0, 1]):
        lab = np.array(lab)
        assert (kmeans.name_lgroups(lab) == _old_find_lgroups(lab)).all()


# ---------------------------------------------------------------------------------------------- refusals
def _no_library(monkeypatch):
    from g2vec_b200 import _capi

    def boom():
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(_capi, "load", boom)


@pytest.mark.parametrize("case", ["1d", "3d", "n0", "n2", "D0", "nan", "inf", "f32_overflow", "r0", "r_neg", "r_1025",
                                  "r_float", "r_str", "max_iter0"])
def test_refusals_raise_before_the_library_is_loaded(case, monkeypatch):
    _no_library(monkeypatch)
    W = np.random.RandomState(0).standard_normal((100, 8)).astype(np.float32)
    R, kw = 5, {}
    if case == "1d":
        W = W[0]
    elif case == "3d":
        W = W.reshape(10, 10, 8)
    elif case == "n0":
        W = W[:0]
    elif case == "n2":
        W = W[:2]
    elif case == "D0":
        W = W[:, :0]
    elif case == "nan":
        W[3, 2] = np.nan
    elif case == "inf":
        W[3, 2] = -np.inf
    elif case == "f32_overflow":
        W = W.astype(np.float64); W[0, 0] = 1e300
    elif case == "r0":
        R = 0
    elif case == "r_neg":
        R = -1
    elif case == "r_1025":
        R = 1025
    elif case == "r_float":
        R = 2.0
    elif case == "r_str":
        R = "3"
    else:
        kw = {"max_iter": 0}
    with pytest.raises(ValueError):
        kmeans.kmeans_lgroups(W, R, **kw)


def test_admitted_inputs():
    W = kmeans.check_inputs(np.ones((3, 1)), 1)
    assert W.dtype == np.float32 and W.shape == (3, 1)
    kmeans.check_inputs(np.zeros((3, 2), np.float32), 1024)
    kmeans.check_inputs(np.zeros((3, 2), np.float32), np.int64(7))


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        kmeans.kmeans_lgroups(np.ones((4, 2), np.float32), 2)


def test_chunk_restarts():
    per = 9 * 1000 + 24 * 8 + 4 * (24 * 8 + 20) + 64
    assert kmeans.chunk_restarts(1000, 8, 10, 3 * per) == 3
    assert kmeans.chunk_restarts(1000, 8, 10, 1) == 1
    assert kmeans.chunk_restarts(1000, 8, 10, 1 << 40) == 10


# ----------------------------------------------------------------------------------------- command line
def test_kmeans_restarts_option():
    a = cli.parse_arguments(["E", "C", "N", "R"])
    assert a.kmeans_restarts == 0 and "kmeans_restarts=0" in repr(a)
    assert cli.parse_arguments(["E", "C", "N", "R", "--kmeans-restarts", "10"]).kmeans_restarts == 10
    assert cli.parse_arguments(["E", "C", "N", "R", "--kmeans-restarts", "1024"]).kmeans_restarts == 1024
    for bad in ("-1", "1025", "1.5", "x"):
        with pytest.raises(SystemExit):
            cli.parse_arguments(["E", "C", "N", "R", "--kmeans-restarts", bad])


def test_command_line_refuses_fewer_than_three_genes(tmp_path, capsys):
    ef, cf, nf = (str(tmp_path / f) for f in ("E.txt", "C.txt", "N.txt"))
    with open(ef, "w") as f:
        f.write("G\tS0\tS1\tS2\nA\t1\t2\t3\nB\t2\t1\t0\nC\t0\t0\t1\n")
    with open(cf, "w") as f:
        f.write("P\tLABEL\nS0\t0\nS1\t1\nS2\t0\n")
    with open(nf, "w") as f:
        f.write("src\tdest\nA\tB\n")
    with pytest.raises(SystemExit):
        cli.main([ef, cf, nf, str(tmp_path / "res"), "--kmeans-restarts", "3"])
    out = capsys.readouterr().out
    assert "ERROR: --kmeans-restarts needs at least 3 common genes, found 2" in out and ">>> 3." not in out


def test_kmeans_writer_format(tmp_path):
    p = str(tmp_path / "res")
    genes = np.array(["A1CF", "AAK1", "ABL1", "ACTB"])
    res = kmeans.KMeansResult(labels=np.array([[0, 1, 1, 2], [1, 0, 0, 2]], np.int8), centres=np.zeros((2, 3, 1)),
                              inertia=np.array([2.5, 2.5]), n_iter=np.array([4, 3], np.int32),
                              seeds=np.zeros((2, 3), np.int32), best=0, agreement=np.array([1.0, 1.0, 0.5, 1 / 3.0]),
                              lgroups=np.array([1, 2, 2, 0], np.int32), reach=1)
    cli.write_kmeans(p, genes, res)
    assert open(p + "_kmeans.txt").read() == (
        "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tAgreement\n"
        "A1CF\t1\t1.000000\n"
        "AAK1\t2\t1.000000\n"
        "ABL1\t2\t0.500000\n"
        "ACTB\t0\t0.333333\n"
        "k-means: best of 2 restarts on the GPU: inertia 2.5 (restart 0, 4 iterations); 1 of 2 restarts reach its "
        "partition; 50.0 % of the genes agree in every restart\n")
