"""The nearest-genes search on the H100 (csrc/g2v_nbr.cu, g2vec_b200/neighbors.py; DESIGN.md §4.25) against the NumPy
restatement of tests/nbr_oracle.py.  Every comparison is bitwise: idx as integers, sim as the float64 bit patterns.

Column splits on an H100 SXM (132 SMs): m <= 64 (one column tile) runs with one split, so g2v_nbr_partial writes the
result itself; m = 65, 1000 and 4097 run with 2, 16 and 4 splits and go through g2v_nbr_merge."""
import os

import numpy as np
import pytest

from g2vec_b200 import neighbors
from tests import nbr_oracle

pytestmark = pytest.mark.gpu

DS = (1, 2, 31, 32, 33, 128, 257, 512)
MS = (2, 3, 63, 64, 65, 1000, 4097)
KS = (1, 7, 64)


def _lib():
    from g2vec_b200 import _capi
    return _capi, _capi.load()


def _same(got, want, what=""):
    gi, gs = got
    wi, ws = want
    assert gi.dtype == np.int32 and gs.dtype == np.float64 and gi.shape == wi.shape, what
    bad = np.nonzero((gi != wi).any(axis=1) | (gs.view(np.int64) != ws.view(np.int64)).any(axis=1))[0]
    assert bad.size == 0, (what, bad[:5], gi[bad[:1]], wi[bad[:1]], gs[bad[:1]], ws[bad[:1]])


def _ks(m):
    return sorted(k for k in set(KS) | {m - 1} if 1 <= k <= min(64, m - 1))


def _random(m, D, seed):
    rs = np.random.RandomState(seed)
    return (rs.standard_normal((m, D)) * np.exp2(rs.randint(-8, 8, size=(m, 1)))).astype(np.float32)


def test_split_counts_of_the_named_cases():
    capi, lib = _lib()
    for m in (2, 3, 63, 64):
        assert lib.g2v_nbr_splits(m) == 1
    for m in (65, 1000, 4097):
        assert lib.g2v_nbr_splits(m) > 1
    assert lib.g2v_nbr_splits(1) == 0 and len(lib.g2v_last_error()) > 0


@pytest.mark.parametrize("D", DS)
def test_bitwise_equal_to_the_oracle(D):
    from g2vec_b200 import _capi
    for m in MS:
        W = _random(m, D, m * 1000 + D)
        ks = _ks(m)
        wi, ws = nbr_oracle.nearest(W, ks[-1])
        splits = _capi.load().g2v_nbr_splits(m)
        for k in ks:
            before = _capi.launch_count()
            got = neighbors.nearest_genes(W, k)
            assert _capi.launch_count() - before == (2 if splits == 1 else 3)
            _same(got, (wi[:, :k], ws[:, :k]), (m, D, k))


def _special(case):
    rs = np.random.RandomState(7)
    if case == "duplicates":                            # every row three times: equal cosines, ordered by j
        W = np.repeat(rs.standard_normal((40, 33)).astype(np.float32), 3, axis=0)
    elif case == "power_of_two_scaling":                # bit-identical cosines across scaled copies
        base = rs.standard_normal((30, 65)).astype(np.float32)
        W = np.concatenate([np.ldexp(base, e).astype(np.float32) for e in (-40, -3, 0, 5, 60)])
    elif case == "all_equal":
        W = np.tile(rs.standard_normal((1, 128)).astype(np.float32), (300, 1))
    elif case == "zero_rows":
        W = rs.standard_normal((200, 31)).astype(np.float32)
        W[::7] = 0.0
        W[5] = -0.0
    elif case == "antipodal_clusters":                  # 40 genes near c, 20 near -c: K = m - 1 = 59 runs into
        c = rs.standard_normal(64).astype(np.float32)   # negative similarities for the first cluster
        a = c + 0.01 * rs.standard_normal((40, 64)).astype(np.float32)
        W = np.concatenate([a, -c - 0.01 * rs.standard_normal((20, 64)).astype(np.float32)])
    elif case == "magnitudes":                          # |w| from 1e-30 to 1e30
        W = (rs.standard_normal((500, 48)) * 10.0 ** rs.uniform(-30, 30, size=(500, 48))).astype(np.float32)
        W[:50] *= np.float32(1e-10)
        W[50:100] = (np.sign(W[50:100]) * 10.0 ** rs.uniform(-30, -25, size=(50, 48))).astype(np.float32)
        W[100:150] = (np.sign(W[100:150]) * 10.0 ** rs.uniform(25, 30, size=(50, 48))).astype(np.float32)
    else:
        raise KeyError(case)
    return np.ascontiguousarray(W, dtype=np.float32)


@pytest.mark.parametrize("case", ["duplicates", "power_of_two_scaling", "all_equal", "zero_rows", "antipodal_clusters",
                                  "magnitudes"])
def test_ties_and_special_rows_bitwise(case):
    W = _special(case)
    assert np.isfinite(W).all()
    m = W.shape[0]
    ks = _ks(m)
    want = nbr_oracle.nearest(W, ks[-1])
    for k in ks:
        _same(neighbors.nearest_genes(W, k), (want[0][:, :k], want[1][:, :k]), (case, k))
    if case == "power_of_two_scaling":                  # scaled copies of one row have the same cosines to every gene
        full = nbr_oracle.similarities(W, [0, 30, 60, 90, 120])
        assert (full[0] == full[1]).all() and (full[0] == full[4]).all()
    if case == "antipodal_clusters":
        assert (want[1][:40, 38] > 0.9).all() and (want[1][:40, 39:] < -0.9).all()
    if case == "all_equal":
        assert (want[0][0] == np.arange(1, 65)).all()


def test_two_calls_give_the_same_bits():
    W = _random(4097, 128, 99)
    a = neighbors.nearest_genes(W, 64)
    b = neighbors.nearest_genes(W, 64)
    assert (a[0] == b[0]).all() and (a[1].view(np.int64) == b[1].view(np.int64)).all()


def test_entry_points_refuse_bad_sizes_and_launch_nothing():
    capi, lib = _lib()
    import torch
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p, st = buf.data_ptr(), torch.cuda.current_stream().cuda_stream
    before = capi.launch_count()
    bad = [lib.g2v_nbr_norms(p, 1, 4, p, st), lib.g2v_nbr_norms(p, 10, 0, p, st), lib.g2v_nbr_norms(None, 10, 4, p, st),
           lib.g2v_nbr_partial(p, p, 10, 4, 0, p, p, st), lib.g2v_nbr_partial(p, p, 10, 4, 10, p, p, st),
           lib.g2v_nbr_partial(p, p, 100, 4, 65, p, p, st), lib.g2v_nbr_partial(p, p, 1, 4, 1, p, p, st),
           lib.g2v_nbr_merge(p, p, 1, 64, 4, p, p, st), lib.g2v_nbr_merge(p, p, 3, 1000, 4, p, p, st),
           lib.g2v_nbr_merge(p, p, 16, 1000, 0, p, p, st)]
    assert all(rc != 0 for rc in bad)
    assert capi.launch_count() == before and len(lib.g2v_last_error()) > 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------- CLI
def test_command_line_writes_the_neighbors_and_leaves_the_other_files_alone(tmp_path, capsys, monkeypatch):
    from g2vec_b200 import cbow, cli
    from tests import helpers
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    base = ["-r", "2", "-e", "5", "-n", "20", "--seed", "3", "--deterministic"]
    a, b = str(tmp_path / "plain"), str(tmp_path / "nbr")
    cli.main([ef, cf, nf, a] + base)
    log_a = capsys.readouterr().out
    captured = []
    train = cbow.train_cbow

    def wrapped(*args, **kw):
        out = train(*args, **kw)
        captured.append(np.array(out, copy=True))
        return out
    monkeypatch.setattr(cbow, "train_cbow", wrapped)
    cli.main([ef, cf, nf, b] + base + ["--neighbors", "10"])
    log_b = capsys.readouterr().out
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt"):
        assert open(a + suffix).read() == open(b + suffix).read(), suffix
    assert not os.path.exists(a + "_neighbors.txt") and "neighbors:" not in log_a
    import re
    untimed = lambda log, prefix: [re.sub(r" \([0-9.]+ sec\)$", "", l).replace(prefix, "RES")
                                   for l in log.splitlines()]
    extra = [l for l in untimed(log_b, b) if l not in untimed(log_a, a)]
    assert len(extra) == 3 and extra[0].startswith("Namespace(") and "neighbors=10" in extra[0]
    assert extra[1].startswith("    neighbors: 10 nearest genes by cosine for each of ") and extra[2] == "    RES_neighbors.txt"
    assert "neighbors=0" in untimed(log_a, a)[1]
    n_paths = int(re.search(r"n_genes : (\d+)\t\(genes in good or poor random paths\)", log_b).group(1))

    mat = captured[0]
    lg = [l.split("\t") for l in open(b + "_lgroups.txt").read().splitlines()[1:]]
    names = np.array([g for g, _ in lg])
    lgroup = np.array([int(k) for _, k in lg])
    rows = open(b + "_neighbors.txt").read().splitlines()
    assert rows[0] == "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tRank\tNeighbor\tNeighborLgroup\tCosine"
    assert len(rows) == 1 + 10 * n_paths
    body = [r.split("\t") for r in rows[1:]]
    sub = np.array([int(np.nonzero(names == body[10 * t][0])[0][0]) for t in range(n_paths)])
    assert (np.diff(sub) > 0).all()                     # in the order of _lgroups.txt
    wi, ws = nbr_oracle.nearest(mat[sub], 10)
    pos = {g: i for i, g in enumerate(names)}
    for t in range(n_paths):
        for r in range(10):
            g, glg, rank, nb, nlg, cos = body[10 * t + r]
            assert g == names[sub[t]] and int(glg) == lgroup[sub[t]] and int(rank) == r + 1
            assert nb == names[sub[wi[t, r]]] and int(nlg) == lgroup[pos[nb]] and cos == "%.6f" % ws[t, r]
    share = float((lgroup[sub][wi] == lgroup[sub][:, None]).mean())
    assert extra[1] == ("    neighbors: 10 nearest genes by cosine for each of %d genes in paths; %.1f %% of the pairs "
                        "share the gene's L-group" % (n_paths, 100.0 * share))


def test_command_line_refuses_k_not_below_the_genes_in_paths(tmp_path, capsys):
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
        cli.main([ef, cf, nf, str(tmp_path / "res"), "-r", "2", "--min-corr", "0", "--neighbors", "30"])
    out = capsys.readouterr().out
    assert ">>> 3." in out and "ERROR: --neighbors 30 needs more than 30 genes in the random paths" in out
    assert ">>> 4." not in out and not os.path.exists(str(tmp_path / "res_vectors.txt"))
