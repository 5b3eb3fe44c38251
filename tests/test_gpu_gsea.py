"""The gene-set enrichment test on the H100 (csrc/g2v_gsea.cu, g2vec_b200/gsea.py; DESIGN.md §4.28) against the NumPy
restatement of tests/gsea_oracle.py.  Every comparison is exact unless it says otherwise."""
import os

import numpy as np
import pytest

from g2vec_b200 import perm
from g2vec_b200.gsea import gsea
from tests import gsea_oracle as go
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


def gpu_keys(A, n, k, s, Q, W):
    import torch
    capi, lib = _lib()
    n_b, G = A.shape
    key = torch.empty((n_b, G), dtype=torch.int64, device="cuda")
    u = torch.empty((n_b, G), dtype=torch.int64, device="cuda")
    d = [_dev(a) for a in (A, Q, W)]
    capi.check(lib.g2v_gsea_keys(d[0].data_ptr(), n_b, G, n, k, s, d[1].data_ptr(), d[2].data_ptr(), key.data_ptr(),
                                 u.data_ptr(), _st()), "g2v_gsea_keys")
    return key.cpu().numpy(), u.cpu().numpy()


def gpu_rank(key):
    import torch
    capi, lib = _lib()
    n_b, G = key.shape
    pos = torch.empty((n_b, G), dtype=torch.int32, device="cuda")
    nbytes = int(lib.g2v_gsea_rank_workspace_bytes(n_b, G))
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    kd = _dev(key)
    capi.check(lib.g2v_gsea_rank(kd.data_ptr(), n_b, G, pos.data_ptr(), ws.data_ptr(), nbytes, _st()), "g2v_gsea_rank")
    return pos.cpu().numpy()


def gpu_es(pos, u, set_ptr, set_gene):
    import torch
    capi, lib = _lib()
    n_b, G = pos.shape
    S = len(set_ptr) - 1
    es = torch.full((n_b, S), 7.0, dtype=torch.float64, device="cuda")
    d = [_dev(a) for a in (pos, u, set_ptr, set_gene)]
    capi.check(lib.g2v_gsea_es(d[0].data_ptr(), d[1].data_ptr(), n_b, G, d[2].data_ptr(), d[3].data_ptr(), S,
                               int(np.diff(set_ptr).max()), es.data_ptr(), _st()), "g2v_gsea_es")
    return es.cpu().numpy()


def gpu_norm(es_null, es_obs):
    import torch
    capi, lib = _lib()
    B, S = es_null.shape
    nes = torch.empty((B, S), dtype=torch.float64, device="cuda")
    mp, mn, no = (torch.empty(S, dtype=torch.float64, device="cuda") for _ in range(3))
    counts = torch.empty((3, S), dtype=torch.int64, device="cuda")
    ed, od = _dev(es_null), _dev(es_obs)
    capi.check(lib.g2v_gsea_norm(ed.data_ptr(), B, S, od.data_ptr(), nes.data_ptr(), mp.data_ptr(), mn.data_ptr(),
                                 no.data_ptr(), counts.data_ptr(), _st()), "g2v_gsea_norm")
    return nes.cpu().numpy(), mp.cpu().numpy(), mn.cpu().numpy(), no.cpu().numpy(), counts.cpu().numpy()


def _eq(a, b):
    """Bit-identical float64 arrays, any NaN equal to any NaN (the payload is the platform's)."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and (na == nb).all() and (a[~na].view(np.int64) == b[~nb].view(np.int64)).all()


def _case(n, G, n_b, seed, dup=True):
    """A cohort's sums over the observed and n_b permuted labellings, with a constant gene (W = 0) and, when dup, two
    duplicated gene columns (tied r)."""
    x, lab = cohort(n, G, seed, n // 3)
    x[:, 1] = 4.0
    if dup and G > 8:
        x[:, 5] = x[:, 3]
        x[:, G - 1] = x[:, 3]
    prep = perm.prepare(x, lab)
    S_pad = -(-n // 32) * 32
    M = perm_oracle.labels(prep["obs"], S_pad, seed, 0, n_b)
    M[0, :n] = prep["obs"]
    A = perm_oracle.sums(M, prep["q"])
    from g2vec_b200.gsea import sign_of
    return A, prep["n"], prep["k"], sign_of(prep), prep["Q"], prep["W"]


# ------------------------------------------------------------------------------------------------ keys and rank
@pytest.mark.parametrize("n,G,n_b", [(12, 2, 1), (40, 255, 3), (135, 256, 7), (135, 257, 64), (60, 7523, 5),
                                     (33, 20000, 2)])
def test_keys_and_ranks_equal_the_oracle(n, G, n_b):
    A, n, k, s, Q, W = _case(n, G, n_b, G + n_b)
    key, u = gpu_keys(A, n, k, s, Q, W)
    _, wu, wkey = go.keys(A, n, k, s, Q, W)
    assert (key == wkey).all() and (u == wu).all()
    assert (gpu_rank(key) == go.rank(wkey)).all()


# -------------------------------------------------------------------------------------------------------- ES
SIZES = [1, 2, 31, 32, 33, 63, 64, 65, 511, 512, 513, 4096]


@pytest.mark.parametrize("G", [4097, 4353, 9001])
def test_es_equals_the_oracle_at_every_set_size(G):
    A, n, k, s, Q, W = _case(70, G, 4, G)
    _, u, key = go.keys(A, n, k, s, Q, W)
    pos = go.rank(key)
    rs = np.random.RandomState(G)
    members = [rs.choice(G, m, replace=False) for m in SIZES]
    top, bottom = int(np.argmin(pos[0])), int(np.argmax(pos[0]))
    members += [np.array([top]), np.array([bottom]), np.array([top, bottom]), np.array([1]),   # ranks 0, G-1; W = 0
                np.array([1, 3, 5, G - 1]), np.array([3, 5, G - 1])]                          # tied r
    set_ptr = np.concatenate([[0], np.cumsum([len(m) for m in members])]).astype(np.int32)
    set_gene = np.concatenate(members).astype(np.int32)
    got = gpu_es(pos, u, set_ptr, set_gene)
    want = go.es(pos, u, set_ptr, set_gene)
    assert _eq(got, want)
    assert (got[:, len(SIZES) + 3] == 0.0).all()        # the weightless set


def test_es_with_one_set_per_row_and_many_rows():
    A, n, k, s, Q, W = _case(50, 300, 300, 2)
    _, u, key = go.keys(A, n, k, s, Q, W)
    pos = go.rank(key)
    set_ptr, set_gene = np.array([0, 15], np.int32), np.arange(100, 115, dtype=np.int32)
    assert _eq(gpu_es(pos, u, set_ptr, set_gene), go.es(pos, u, set_ptr, set_gene))


def test_norm_equals_the_oracle():
    rs = np.random.RandomState(0)
    B, S = 1000, 333
    es_null = rs.uniform(-1, 1, (B, S))
    es_null[:, 5] = np.abs(es_null[:, 5])               # NaN NES for a negative ES
    es_null[:, 6] = 0.0
    es_null[::3, 7] = np.round(es_null[::3, 7], 1)
    es_obs = rs.uniform(-1, 1, S)
    es_obs[5], es_obs[6], es_obs[7] = -0.5, 0.0, es_null[3, 7]
    got, want = gpu_norm(es_null, es_obs), go.norm(es_null, es_obs)
    for g, w in zip(got, want):
        assert _eq(g, w) if g.dtype == np.float64 else (g == w).all()


# -------------------------------------------------------------------------------------------------------- gsea
def _ex():
    from tests.helpers import GOLDEN
    e = np.load(os.path.join(GOLDEN, "ex_expr.npz"))
    return e["expr"], np.load(os.path.join(GOLDEN, "ex_graph.npz"))["label"]


def _same(a, b):
    assert a.name == b.name
    for f in ("size", "count_pos", "count_neg", "count_extreme", "count_null", "count_null_side", "count_obs",
              "count_obs_side", "count_fwer"):
        assert (getattr(a, f) == getattr(b, f)).all(), f
    for f in ("ES", "NES", "P", "FDR", "FWER", "mean_pos", "mean_neg"):
        assert _eq(getattr(a, f), getattr(b, f)), f
    assert all((x == y).all() for x, y in zip(a.leading_edge, b.leading_edge))


def test_gsea_equals_the_oracle_on_ex_in_any_chunking():
    from g2vec_b200 import _capi
    x, lab = _ex()
    G = x.shape[1]
    rs = np.random.RandomState(1)
    sets = [("set%d" % i, rs.choice(G, int(rs.randint(15, 120)), replace=False)) for i in range(25)]
    sets.append(("tiny", [0, 1]))                       # dropped by the size filter
    B = 60
    want = go.gsea(x, lab, sets, B, seed=3, chunk=17)
    assert len(want.name) == 25
    row = 160 + 44 * G
    for max_bytes in (row, row * 25, None):
        before = _capi.launch_count()
        got = gsea(x, lab, sets, B, seed=3, max_chunk_bytes=max_bytes)
        assert _capi.launch_count() > before
        _same(got, want)


def test_gsea_label_rows_are_perm_tests():
    """The label rows are perm_test's for the same seed (g2v_perm_labels from b_begin = 0, as perm_oracle.labels), and
    gsea through them equals the oracle built on those rows."""
    import torch
    x, lab = cohort(45, 40, 9, 20)
    prep = perm.prepare(x, lab)
    capi, lib = _lib()
    S_pad, B = 64, 30
    M = torch.zeros((B, S_pad), dtype=torch.uint8, device="cuda")
    od = _dev(prep["obs"])
    capi.check(lib.g2v_perm_labels(od.data_ptr(), 45, S_pad, 11, 0, B, M.data_ptr(), _st()), "labels")
    assert (M.cpu().numpy() == perm_oracle.labels(prep["obs"], S_pad, 11, 0, B)).all()
    sets = [("g%d" % g, [g, (g + 1) % 40, (g + 2) % 40]) for g in range(40)]
    a = gsea(x, lab, sets, B, seed=11, min_size=3, max_size=3)
    _same(a, go.gsea(x, lab, sets, B, seed=11, min_size=3, max_size=3))


def test_planted_set_is_enriched_on_the_side_it_was_shifted():
    rs = np.random.RandomState(5)
    n, G = 120, 2000
    x = rs.standard_normal((n, G))
    lab = np.array([0] * 60 + [1] * 60)
    rs.shuffle(lab)
    sets = [("random%d" % i, rs.choice(np.arange(100, G), 30, replace=False)) for i in range(40)]
    for shift_label, sign in ((1, 1), (0, -1)):
        xx = x.copy()
        xx[:, :30] += 0.8 * (lab == shift_label)[:, None]
        r = gsea(xx, lab, [("planted", np.arange(30))] + sets, 1000, seed=2)
        assert np.sign(r.ES[0]) == sign and r.FDR[0] <= 0.05 and r.P[0] <= 0.01
        assert len(r.leading_edge[0]) >= 10


def test_null_p_values_are_close_to_uniform():
    from scipy import stats
    rs = np.random.RandomState(8)
    n, G = 80, 1500
    x = rs.standard_normal((n, G))
    lab = rs.randint(0, 2, n)
    sets = [("s%d" % i, rs.choice(G, int(rs.randint(15, 60)), replace=False)) for i in range(200)]
    r = gsea(x, lab, sets, 400, seed=4)
    assert stats.kstest(r.P, "uniform").pvalue > 1e-4


def test_entry_points_refuse_bad_sizes_and_launch_nothing():
    capi, lib = _lib()
    import torch
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p, st = buf.data_ptr(), _st()
    before = capi.launch_count()
    bad = [lib.g2v_gsea_keys(p, 1, 1, 10, 3, 1, p, p, p, p, st), lib.g2v_gsea_keys(p, 0, 10, 10, 3, 1, p, p, p, p, st),
           lib.g2v_gsea_keys(p, 1, 10, 10, 3, 0, p, p, p, p, st), lib.g2v_gsea_keys(p, 1, 10, 10, 10, 1, p, p, p, p, st),
           lib.g2v_gsea_keys(p, 1, (1 << 20) + 1, 10, 3, 1, p, p, p, p, st),
           lib.g2v_gsea_keys(p, 65536, 10, 10, 3, 1, p, p, p, p, st),
           lib.g2v_gsea_rank(p, 1, 10, p, p, 0, st), lib.g2v_gsea_rank(p, 3000, 1 << 20, p, p, 1 << 20, st),
           lib.g2v_gsea_es(p, p, 1, 10, p, p, 0, 3, p, st), lib.g2v_gsea_es(p, p, 1, 10, p, p, 1, 10, p, st),
           lib.g2v_gsea_es(p, p, 1, 5000, p, p, 1, 4097, p, st), lib.g2v_gsea_es(p, p, 1, 10, p, p, 1, 0, p, st),
           lib.g2v_gsea_norm(p, 0, 1, p, p, p, p, p, p, st), lib.g2v_gsea_norm(p, 1, 0, p, p, p, p, p, p, st),
           lib.g2v_gsea_norm(p, 1 << 20, 257, p, p, p, p, p, p, st)]
    assert all(rc != 0 for rc in bad)
    assert int(lib.g2v_gsea_rank_workspace_bytes(0, 10)) == 0
    assert capi.launch_count() == before and len(lib.g2v_last_error()) > 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------- CLI
def test_command_line_writes_the_gsea_file_and_leaves_the_other_files_alone(tmp_path, capsys):
    from g2vec_b200 import cli
    from tests import helpers
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    rs = np.random.RandomState(0)
    gmt = tmp_path / "sets.gmt"
    with open(gmt, "w") as f:
        for i in range(12):
            f.write("SET_%d\tdesc\t%s\tNOT_A_GENE\n" % (i, "\t".join(genes[rs.choice(len(genes), 20 + 10 * i, replace=False)])))
        f.write("SMALL\tdesc\t%s\n" % "\t".join(genes[:5]))
    base = ["-r", "2", "-e", "5", "-n", "20", "--seed", "3", "--deterministic"]
    a, b = str(tmp_path / "plain"), str(tmp_path / "gs")
    cli.main([ef, cf, nf, a] + base)
    log_a = capsys.readouterr().out
    cli.main([ef, cf, nf, b] + base + ["--gene-sets", str(gmt), "--gene-set-permutations", "100"])
    log_b = capsys.readouterr().out
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt"):
        assert open(a + suffix).read() == open(b + suffix).read(), suffix
    assert not os.path.exists(a + "_gsea.txt")
    import re
    untimed = lambda log, prefix: [re.sub(r" \([0-9.]+ sec\)$", "", l).replace(prefix, "RES")
                                   for l in log.splitlines()]
    extra = [l for l in untimed(log_b, b) if l not in untimed(log_a, a)]
    assert len(extra) == 4 and extra[0].startswith("Namespace(") and "gene_set_permutations=100" in extra[0]
    assert extra[1] == "    gene sets: 12 of 13 in %s with 15..500 genes in the analysis" % gmt
    assert extra[2].startswith("    gene-set test: 100 label permutations: ") and extra[3] == "    RES_gsea.txt"
    data = cli.load_data(ef)
    data["label"] = cli.match_labels(cli.load_clinical(cf), data["sample"])
    data, _ = cli.restrict(data, cli.load_network(nf))
    from g2vec_b200.gsea import read_gmt
    r = gsea(data["expr"], data["label"], read_gmt(str(gmt)), 100, seed=3, genes=data["gene"])
    bm = set(open(b + "_biomarkers.txt").read().split()[1:])
    rows = open(b + "_gsea.txt").read().splitlines()
    assert rows[0] == "GeneSet\tSize\tES\tNES\tP\tFDR_Q\tFWER_P\tBiomarkers\tLeadingEdge" and len(rows) == 13
    g = data["gene"]
    for i, line in enumerate(rows[1:]):
        assert line == "SET_%d\t%d\t%.6f\t%.6f\t%.6g\t%.6g\t%.6g\t%d\t%s" % (
            i, 20 + 10 * i, r.ES[i], r.NES[i], r.P[i], r.FDR[i], r.FWER[i], sum(g[j] in bm for j in r.members[i]),
            ",".join(g[j] for j in r.leading_edge[i]))
    assert extra[2].endswith("(%d up in poor, %d up in good)" % (int(((r.FDR <= 0.25) & (r.NES > 0)).sum()),
                                                                  int(((r.FDR <= 0.25) & (r.NES < 0)).sum())))
