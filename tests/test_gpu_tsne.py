"""The exact t-SNE map on the H100 (csrc/g2v_tsne.cu, g2vec_b200/tsne.py; DESIGN.md §4.27) against the NumPy
restatement of tests/tsne_oracle.py.  d and the iterates Y are compared bit for bit; beta and the step counts through the
tolerance recomputed on the host; P against the oracle run from the GPU's betas; the KL divergence at a tolerance.

Edges: g2v_tsne_dist tiles 64 x 64; g2v_tsne_symmetrize 32 x 32; the gradient chains run in blocks of 256 columns and Z
in blocks of 256 rows (tsne.BLOCK); the stage switch is at iteration 250."""
import os
import re

import numpy as np
import pytest

from g2vec_b200 import tsne
from tests import tsne_oracle

pytestmark = pytest.mark.gpu

B = tsne.BLOCK


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _random(m, D, seed):
    rs = np.random.RandomState(seed)
    return (rs.standard_normal((m, D)) * np.exp2(rs.randint(-3, 3, size=(m, 1)))).astype(np.float32)


def _gpu_dist(W):
    import torch
    from g2vec_b200 import _capi
    lib = _capi.load()
    m, D = W.shape
    P = torch.empty((m, m), dtype=torch.float64, device="cuda")
    Wd = torch.from_numpy(np.ascontiguousarray(W, np.float32)).cuda()
    _capi.check(lib.g2v_tsne_dist(Wd.data_ptr(), m, D, P.data_ptr(), torch.cuda.current_stream().cuda_stream),
                "g2v_tsne_dist")
    return P.cpu().numpy()


def _check_dist(m, D):
    W = _random(m, D, m * 1000 + D)
    got = _gpu_dist(W)
    want = tsne_oracle.dist(W.astype(np.float64))
    assert (_bits(got) == _bits(want)).all(), (m, D)
    assert (_bits(got) == _bits(got.T)).all() and (np.diag(got) == 0).all()


@pytest.mark.parametrize("D", (1, 2, 31, 32, 33, 128, 257, 512))
def test_distances_bitwise_over_dimensions(D):
    for m in (65, 257):
        _check_dist(m, D)


@pytest.mark.parametrize("m", (2, 3, 63, 64, 65, 255, 256, 257, 1000, 4097))
def test_distances_bitwise_over_rows(m):
    _check_dist(m, 33)


def test_distances_bitwise_large():
    _check_dist(1000, 512)


def _check_affinities(W, perplexity):
    """beta meets the tolerance on the host wherever steps < 100; P equals the oracle's from the GPU's beta (rtol 1e-12;
    atol only for values in the subnormal range, where one unit of exp's last place is a large relative error).  A row
    whose sum S is itself subnormal (every e_ij below 2^-1022: only at extreme magnitudes, where the bisection does not
    converge) has c set by the last bits of exp, which are CUDA's, so P is compared outside those rows and columns."""
    P, beta, steps = tsne.affinities(W, perplexity)
    d = tsne_oracle.dist(W.astype(np.float64))
    ok = steps < tsne.MAX_STEPS
    H = tsne_oracle.entropy(d, beta)
    assert (np.abs(H[ok] - np.log(perplexity)) <= tsne.TOLERANCE + 1e-12).all()
    want = tsne_oracle.joint(tsne_oracle.conditional_from_beta(d, beta))
    S = tsne_oracle.row_sums(d, beta)
    normal = ~((S > 0) & (S < np.finfo(np.float64).tiny))
    np.testing.assert_allclose(P[np.ix_(normal, normal)], want[np.ix_(normal, normal)], rtol=1e-12, atol=1e-300)
    assert np.isfinite(P).all() and (P >= 0).all()
    assert (_bits(P) == _bits(P.T)).all() and (np.diag(P) == 0).all()
    return P, beta, steps


@pytest.mark.parametrize("m,D,perplexity", [(2, 3, 1.0), (3, 5, 2.0), (63, 8, 5.0), (257, 33, 30.0),
                                            (1000, 128, 30.0), (4097, 16, 50.0)])
def test_affinities_meet_the_tolerance_and_equal_the_oracle(m, D, perplexity):
    P, beta, steps = _check_affinities(_random(m, D, m + D), perplexity)
    assert (steps < tsne.MAX_STEPS).all() and abs(P.sum() - 1.0) < 1e-9
    # the bisection of the oracle from the same d reaches the same betas (no row sits within rounding of the tolerance)
    _, b2, s2 = tsne_oracle.conditional(tsne_oracle.dist(_random(m, D, m + D).astype(np.float64)), perplexity)
    assert (beta == b2).all() and (steps == s2).all()


SNAPSHOTS = (1, 2, 249, 250, 251, 300)


@pytest.mark.parametrize("m", (2, 3, 255, 256, 257, 513))
def test_iterations_bitwise_equal_to_the_oracle(m):
    W = _random(m, 12, m)
    P, _, _ = tsne.affinities(W, min(30.0, m - 0.5))
    Y0 = tsne.pca_init(W, seed=m)
    _, snap = tsne_oracle.optimize(P, Y0, max(SNAPSHOTS), snapshots=SNAPSHOTS)
    for n in SNAPSHOTS:
        Y, kl = tsne.optimize(P, Y0, n)
        assert Y.dtype == np.float64 and (_bits(Y) == _bits(snap[n])).all(), (m, n)
    assert abs(kl - tsne_oracle.kl(P, Y)) <= 1e-10 * max(abs(kl), 1e-300)


def test_two_maps_give_the_same_bits():
    W = _random(700, 32, 1)
    a = tsne.tsne_map(W, 20.0, n_iter=400, seed=2)
    b = tsne.tsne_map(W, 20.0, n_iter=400, seed=2)
    assert (_bits(a.Y) == _bits(b.Y)).all() and (_bits(a.beta) == _bits(b.beta)).all()
    assert (a.steps == b.steps).all() and _bits(a.kl) == _bits(b.kl)
    assert a.learning_rate == 50.0 and np.isfinite(a.Y).all()


def _special(case):
    rs = np.random.RandomState(3)
    if case == "duplicates":
        return np.repeat(rs.standard_normal((30, 9)).astype(np.float32), 10, axis=0)
    if case == "all_equal":
        return np.tile(rs.standard_normal((1, 40)).astype(np.float32), (300, 1))
    if case == "magnitudes":
        W = rs.standard_normal((300, 17))
        return (W * 10.0 ** rs.randint(-30, 31, size=(300, 1))).astype(np.float32)
    raise KeyError(case)


@pytest.mark.parametrize("case", ["duplicates", "all_equal", "magnitudes"])
def test_special_data(case):
    W = _special(case)
    P, beta, steps = _check_affinities(W, 10.0)
    if case == "all_equal":                            # d = 0 everywhere: H = log(m - 1) at every beta
        assert (steps == tsne.MAX_STEPS).all() and (P[~np.eye(300, dtype=bool)] == P[0, 1]).all()
    res = tsne.tsne_map(W, 10.0, n_iter=300, seed=4)
    assert (_bits(res.beta) == _bits(beta)).all() and (res.steps == steps).all()
    Y0 = tsne.pca_init(W, seed=4)
    if case == "all_equal":
        assert (Y0 == np.random.default_rng(4).standard_normal((300, 2)) * 1e-4).all()
    want, _ = tsne_oracle.optimize(P, Y0, 300)
    assert np.isfinite(res.Y).all() and (_bits(res.Y) == _bits(want)).all()
    assert np.isfinite(res.kl)


def _knn_agreement(Y, labels, k=10):
    d = ((Y[:, None, :] - Y[None, :, :]) ** 2).sum(-1)
    np.fill_diagonal(d, np.inf)
    nn = np.argsort(d, axis=1, kind="stable")[:, :k]
    return float((labels[nn] == labels[:, None]).mean())


def test_planted_clusters_stay_apart_in_the_map(capsys):
    rs = np.random.RandomState(9)
    centres = rs.standard_normal((3, 32)) * 10.0
    labels = np.repeat([0, 1, 2], 200)
    W = (centres[labels] + rs.standard_normal((600, 32))).astype(np.float32)
    res = tsne.tsne_map(W, 30.0)
    share = _knn_agreement(res.Y, labels)
    with capsys.disabled():
        print("\nplanted clusters 3 x 200, D = 32: 10-NN label agreement in the map %.4f, KL %.4f" % (share, res.kl))
    assert share >= 0.95


def test_close_to_scikit_learn_exact_on_the_same_distances(capsys):
    """A sanity check, not a contract: scikit-learn's exact TSNE from the same d and Y0 (its P is normalised by the sum
    and clamped at eps, and it multiplies P by 12 in place; the trajectories part in the last bits and then diverge)."""
    from sklearn.manifold import TSNE, trustworthiness
    rs = np.random.RandomState(10)
    centres = rs.standard_normal((5, 16)) * 4.0
    labels = rs.randint(0, 5, size=500)
    W = (centres[labels] + rs.standard_normal((500, 16))).astype(np.float32)
    res = tsne.tsne_map(W, 30.0)
    Y0 = tsne.pca_init(W)
    d = tsne_oracle.dist(W.astype(np.float64))
    sk = TSNE(n_components=2, perplexity=30.0, method="exact", metric="precomputed", init=Y0.copy(),
              learning_rate="auto", n_iter_without_progress=1000, min_grad_norm=0, max_iter=1000,
              random_state=0).fit(d)
    t_ours = trustworthiness(W, res.Y, n_neighbors=10)
    t_sk = trustworthiness(W, sk.embedding_, n_neighbors=10)
    with capsys.disabled():
        print("\nscikit-learn exact, m = 500: KL ours %.5f, scikit-learn %.5f; trustworthiness ours %.5f, "
              "scikit-learn %.5f" % (res.kl, sk.kl_divergence_, t_ours, t_sk))
    assert abs(res.kl - sk.kl_divergence_) <= 0.1 * sk.kl_divergence_
    assert abs(t_ours - t_sk) <= 0.02 and t_ours >= 0.9


def test_entry_points_refuse_bad_sizes_and_launch_nothing():
    from g2vec_b200 import _capi
    lib = _capi.load()
    import torch
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p, st = buf.data_ptr(), torch.cuda.current_stream().cuda_stream
    before = _capi.launch_count()
    big = tsne.MAX_GENES + 1
    bad = [lib.g2v_tsne_dist(p, 1, 4, p, st), lib.g2v_tsne_dist(p, big, 4, p, st), lib.g2v_tsne_dist(p, 10, 0, p, st),
           lib.g2v_tsne_dist(None, 10, 4, p, st), lib.g2v_tsne_dist(p, 10, 4, None, st),
           lib.g2v_tsne_affinity(p, 10, 0.999, p, p, st), lib.g2v_tsne_affinity(p, 10, 10.0, p, p, st),
           lib.g2v_tsne_affinity(p, 10, float("nan"), p, p, st), lib.g2v_tsne_affinity(p, 1, 1.0, p, p, st),
           lib.g2v_tsne_affinity(p, 10, 3.0, None, p, st),
           lib.g2v_tsne_symmetrize(p, big, st), lib.g2v_tsne_symmetrize(None, 10, st),
           lib.g2v_tsne_grad(p, p, 1, p, st), lib.g2v_tsne_grad(p, None, 10, p, st),
           lib.g2v_tsne_update(p, 10, -1, 50.0, p, p, p, st), lib.g2v_tsne_update(p, 10, 0, 0.0, p, p, p, st),
           lib.g2v_tsne_update(p, 10, 0, float("inf"), p, p, p, st),
           lib.g2v_tsne_update(p, 10, 0, float("nan"), p, p, p, st), lib.g2v_tsne_update(p, 10, 0, 50.0, p, None, p, st),
           lib.g2v_tsne_update(p, big, 0, 50.0, p, p, p, st),
           lib.g2v_tsne_kl(p, p, big, p, p, st), lib.g2v_tsne_kl(p, p, 10, p, None, st)]
    assert all(rc != 0 for rc in bad)
    assert _capi.launch_count() == before and len(lib.g2v_last_error()) > 0
    assert lib.g2v_tsne_workspace_bytes(1) == 0 and lib.g2v_tsne_workspace_bytes(big) == 0
    assert lib.g2v_tsne_workspace_bytes(257) == 8 * (5 * 257 * 2 + 5 * 257 + 2)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------- CLI
def test_command_line_writes_the_map_twice_the_same(tmp_path, capsys, monkeypatch):
    from g2vec_b200 import cbow, cli
    from tests import helpers
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    base = ["-r", "2", "-e", "5", "-n", "20", "--seed", "3", "--deterministic"]
    a, b, c = str(tmp_path / "plain"), str(tmp_path / "map1"), str(tmp_path / "map2")
    cli.main([ef, cf, nf, a] + base)
    log_a = capsys.readouterr().out
    captured = []
    train = cbow.train_cbow

    def wrapped(*args, **kw):
        out = train(*args, **kw)
        captured.append(np.array(out, copy=True))
        return out
    monkeypatch.setattr(cbow, "train_cbow", wrapped)
    cli.main([ef, cf, nf, b] + base + ["--tsne", "30"])
    log_b = capsys.readouterr().out
    cli.main([ef, cf, nf, c] + base + ["--tsne", "30"])
    capsys.readouterr()
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt"):
        assert open(a + suffix).read() == open(b + suffix).read(), suffix
    assert not os.path.exists(a + "_tsne.txt") and "t-SNE:" not in log_a
    assert open(b + "_tsne.txt", "rb").read() == open(c + "_tsne.txt", "rb").read()
    untimed = lambda log, prefix: [re.sub(r" \([0-9.]+ sec\)$", "", l).replace(prefix, "RES")
                                   for l in log.splitlines()]
    la, lb = untimed(log_a, a), untimed(log_b, b)
    assert "tsne=0.0" in la[1] and "tsne=30.0" in lb[1]
    n_paths = int(re.search(r"n_genes : (\d+)\t\(genes in good or poor random paths\)", log_b).group(1))
    rows = open(b + "_tsne.txt").read().splitlines()
    assert rows[0] == "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tX\tY" and len(rows) == 1 + n_paths

    lg = [l.split("\t") for l in open(b + "_lgroups.txt").read().splitlines()[1:]]
    names = np.array([g for g, _ in lg])
    lgroup = np.array([int(k) for _, k in lg])
    body = [r.split("\t") for r in rows[1:]]
    sub = np.array([int(np.nonzero(names == r[0])[0][0]) for r in body])
    assert (np.diff(sub) > 0).all()                     # in the order of _lgroups.txt
    mat = captured[0]
    want = tsne.tsne_map(mat[sub], 30.0, seed=3)
    assert rows[1:] == ["%s\t%d\t%.6f\t%.6f" % (names[g], lgroup[g], x, y) for g, (x, y) in zip(sub, want.Y)]
    line = "    " + tsne.summary(n_paths, 30.0, 1000, want.kl)
    extra = [l for l in lb if l not in la]
    assert len(lb) == len(la) + 2 and len(extra) == 3 and extra[0].startswith("Namespace(")
    assert extra[1] == line and extra[2] == "    RES_tsne.txt"


def test_command_line_refuses_a_perplexity_not_below_the_genes_in_paths(tmp_path, capsys):
    from g2vec_b200 import cli
    rs = np.random.RandomState(5)
    G, S = 30, 40
    x = rs.standard_normal((G, S))
    ef, cf, nf = (str(tmp_path / f) for f in ("E.txt", "C.txt", "N.txt"))
    with open(ef, "w") as f:
        f.write("G\t" + "\t".join("S%d" % s for s in range(S)) + "\n")
        f.writelines("G%02d\t%s\n" % (g, "\t".join("%.4f" % v for v in x[g])) for g in range(G))
    with open(cf, "w") as f:
        f.write("P\tLABEL\n")
        f.writelines("S%d\t%d\n" % (s, s % 2) for s in range(S))
    with open(nf, "w") as f:
        f.write("src\tdest\n")
        f.writelines("G%02d\tG%02d\n" % (g, h) for g in range(G) for h in (g + 1, g + 2) if h < G)
    with pytest.raises(SystemExit):
        cli.main([ef, cf, nf, str(tmp_path / "res"), "-r", "2", "--min-corr", "0", "--tsne", "30"])
    out = capsys.readouterr().out
    assert ">>> 3." in out and "ERROR: --tsne 30 needs more than 30 and at most 32768 genes in the random paths" in out
    assert ">>> 4." not in out and not os.path.exists(str(tmp_path / "res_vectors.txt"))
