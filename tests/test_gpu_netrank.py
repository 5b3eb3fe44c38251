"""The NetRank test on the H100 (csrc/g2v_nr.cu, g2vec_b200/netrank.py; DESIGN.md §4.35) against the NumPy restatement
of tests/netrank_oracle.py.  Every comparison of scores and counts is bit for bit."""
import os

import numpy as np
import pytest

from g2vec_b200 import diffcoex, netrank, perm
from tests import netrank_cohorts, netrank_oracle, perm_oracle
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


# The device copies are held in locals until the result is back.
def gpu_seed(A, n, k, Q, W, ld):
    import torch
    capi, lib = _lib()
    n_b, G = A.shape
    S = torch.full((G, ld), np.nan, dtype=torch.float64, device="cuda")
    d = [_dev(a) for a in (A, Q, W)]
    capi.check(lib.g2v_nr_seed(d[0].data_ptr(), n_b, G, n, k, d[1].data_ptr(), d[2].data_ptr(), S.data_ptr(), ld,
                               _st()), "g2v_nr_seed")
    return S.cpu().numpy()


def gpu_propagate(S, pairs, d, tile, n_cols=None):
    """netrank.propagate on the columns 0 .. n_cols - 1 of S [G][ld] with the given column tile."""
    import torch
    capi, lib = _lib()
    G, ld = S.shape
    rowptr, col, deg, w = netrank.csr(pairs, G)
    net = tuple(_dev(a) for a in (rowptr, col, w, netrank.row_order(deg)))
    S_d = _dev(S)
    xa, xb = (torch.full((G, ld), np.nan, dtype=torch.float64, device="cuda") for _ in range(2))
    out = netrank.propagate(lib, net, S_d, xa, xb, G, ld, n_cols or ld, netrank.n_iterations(d), d, tile, _st())
    return out.cpu().numpy()


def gpu_tally(x, n_b, score_obs):
    import torch
    capi, lib = _lib()
    G, ld = x.shape
    c = torch.full((G,), 5, dtype=torch.int64, device="cuda")
    d = [_dev(a) for a in (x, score_obs)]
    capi.check(lib.g2v_nr_tally(d[0].data_ptr(), G, n_b, ld, d[1].data_ptr(), c.data_ptr(), _st()), "g2v_nr_tally")
    return c.cpu().numpy() - 5


# ------------------------------------------------------------------------------------------------------ seed
@pytest.mark.parametrize("n_b,G,ld", [(1, 1, 1), (31, 33, 31), (33, 64, 64), (70, 257, 96), (1, 300, 1)])
def test_seed_equals_the_oracle(n_b, G, ld):
    rs = np.random.RandomState(n_b + G)
    n, k = 135, 58
    A = rs.randint(-(1 << 37), 1 << 37, size=(n_b, G)).astype(np.int64)
    Q = rs.randint(-(1 << 37), 1 << 37, size=G).astype(np.int64)
    N = n * A - k * Q[None, :]
    W = (N.astype(np.float64) ** 2).max(axis=0) * rs.uniform(1.0, 3.0, G)
    W[::7] = 0.0                                        # constant genes: S = 0
    got = gpu_seed(A, n, k, Q, W, ld)
    want = netrank_oracle.seeds(A, n, k, Q, W)
    assert np.array_equal(got[:, :n_b], want) and np.isnan(got[:, n_b:]).all()
    assert (want[::7] == 0.0).all()


# ------------------------------------------------------------------------------------------------------ step
def hub_network():
    """Degrees 5000, 1024, 33, 32, 31, 1 and 0 with a random background: G = 5200."""
    G = 5200
    rs = np.random.RandomState(7)
    src = [np.zeros(5000, int), np.full(1024, 5001), np.full(33, 5002), np.full(32, 5003), np.full(31, 5004),
           [5005], rs.randint(5006, 5150, 300)]
    dst = [np.arange(1, 5001), np.arange(2, 1026), np.arange(5100, 5133), np.arange(5100, 5132),
           np.arange(5100, 5131), [5199 - 60], rs.randint(5006, 5150, 300)]
    pairs = diffcoex.pairs_from_edges(np.concatenate(src), np.concatenate(dst))
    deg = netrank.csr(pairs, G)[2]
    assert deg[0] == 5000 and deg[5001] == 1024 and (deg == 0).sum() > 20
    assert {1, 31, 32, 33} <= set(deg[5002:5006].tolist())
    return pairs, G


@pytest.mark.parametrize("cols", [1, 37, 96])
def test_step_is_bit_exact_at_every_degree_and_column_tile(cols):
    pairs, G = hub_network()
    rs = np.random.RandomState(cols)
    ld = -(-cols // 32) * 32
    S = rs.uniform(size=(G, ld))
    S[::9] = 0.0
    want = netrank_oracle.propagate(S[:, :cols], pairs, 0.5)
    for tile in (32, 64, 1 << 20):
        got = gpu_propagate(S, pairs, 0.5, tile, n_cols=cols)
        assert np.array_equal(got[:, :cols], want), tile


def test_step_is_bit_exact_at_the_largest_damping():
    rs = np.random.RandomState(3)
    G = 300
    pairs = diffcoex.pairs_from_edges(rs.randint(0, 280, 2500), rs.randint(0, 280, 2500))
    S = rs.uniform(size=(G, 40))
    assert np.array_equal(gpu_propagate(S, pairs, 0.95, 32, n_cols=33)[:, :33],
                          netrank_oracle.propagate(S[:, :33], pairs, 0.95))


# ----------------------------------------------------------------------------------------------------- tally
@pytest.mark.parametrize("G,n_b,ld", [(1, 1, 1), (7, 31, 32), (9, 33, 64), (300, 1000, 1024)])
def test_tally_equals_the_oracle(G, n_b, ld):
    rs = np.random.RandomState(G + n_b)
    x = rs.uniform(size=(G, ld))
    obs = rs.uniform(size=G)
    x[:, 0] = obs                                       # ties count
    x[:, n_b:] = 2.0                                    # past n_b: never read
    got = gpu_tally(x, n_b, obs)
    assert (got == (x[:, :n_b] >= obs[:, None]).sum(axis=1)).all() and (got >= 1).all()


# ------------------------------------------------------------------------------------------------ netrank_test
def _same(a, b):
    for f in ("degree", "count", "order"):
        assert (getattr(a, f) == getattr(b, f)).all(), f
    for f in ("S", "score", "P", "Q"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    assert a.n_iter == b.n_iter and a.n_perm == b.n_perm


def _case(name):
    if name == "hubs":
        pairs, G = hub_network()
        x, lab = cohort(40, G, 1, 17)
        x[:, 0] = 2.0                                   # the largest hub is constant
        x[:, 5150:5160] = -1.0                          # isolated and constant
        return x, lab, pairs
    rs = np.random.RandomState(len(name))
    G = {"small": 300, "G2": 2, "G33": 33, "G257": 257}[name]
    x, lab = cohort(45, G, len(name), 20)
    x[:, 1] = 0.5
    pairs = diffcoex.pairs_from_edges(rs.randint(0, G, 3 * G), rs.randint(0, G, 3 * G))
    if not pairs.size:
        pairs = np.array([[0, 1]], np.int32)
    return x, lab, pairs


@pytest.mark.parametrize("name,d,B", [("hubs", 0.5, 70), ("small", 0.95, 37), ("small", 0.0, 33), ("G2", 0.5, 1),
                                      ("G33", 0.3, 31), ("G257", 0.5, 65)])
def test_netrank_test_equals_the_oracle(name, d, B):
    x, lab, pairs = _case(name)
    want = netrank_oracle.netrank_test(x, lab, pairs, B, damping=d, seed=11)
    _same(netrank.netrank_test(x, lab, pairs, B, damping=d, seed=11), want)


def _ex():
    from tests.helpers import GOLDEN
    e = np.load(os.path.join(GOLDEN, "ex_expr.npz"))
    return e["expr"], np.load(os.path.join(GOLDEN, "ex_graph.npz"))["label"], diffcoex.pairs_from_edges(e["src"],
                                                                                                     e["dst"])


def test_same_bits_in_any_chunking_and_run_on_the_example_cohort():
    from g2vec_b200 import _capi
    x, lab, pairs = _ex()
    B, G = 200, x.shape[1]
    want = netrank_oracle.netrank_test(x, lab, pairs, B, damping=0.5, seed=3, chunk=70)
    tile = int(_capi.load().g2v_nr_tile_cols(G))
    row = 160 + 32 * G
    for max_bytes, chunks in ((row * 70, [70, 70, 60]), (None, [200]), (None, [200])):
        before = _capi.launch_count()
        got = netrank.netrank_test(x, lab, pairs, B, damping=0.5, seed=3, max_chunk_bytes=max_bytes)
        steps = sum(-(-c // tile) for c in chunks) * 40
        assert _capi.launch_count() - before == 2 + 40 + 4 * len(chunks) + steps
        _same(got, want)
    assert pairs.shape[0] == 140902 and (got.degree == 0).sum() == 78 and got.degree.max() == 840


def test_zero_damping_counts_come_from_the_permutation_tests_rows():
    import torch
    capi, lib = _lib()
    x, lab = cohort(50, 40, 21, 22)
    pairs = diffcoex.pairs_from_edges(np.arange(39), np.arange(1, 40))
    B, seed = 300, 4
    r = netrank.netrank_test(x, lab, pairs, B, damping=0.0, seed=seed)
    prep = perm.prepare(x, lab)
    n, S_pad = prep["n"], 64
    M = torch.empty((B, S_pad), dtype=torch.uint8, device="cuda")
    obs = _dev(prep["obs"])
    capi.check(lib.g2v_perm_labels(obs.data_ptr(), n, S_pad, seed, 0, B, M.data_ptr(), _st()), "g2v_perm_labels")
    rho_b = perm.rho_of(n * perm_oracle.sums(M.cpu().numpy(), prep["q"]) - prep["k"] * prep["Q"][None, :],
                        prep["W"][None, :])
    assert (r.count == (rho_b >= prep["rho_obs"][None, :]).sum(axis=0)).all()
    assert (r.count == perm.perm_test(x, lab, B, seed=seed).count).all()
    assert np.array_equal(r.score, np.sqrt(prep["rho_obs"])) and r.n_iter == 0


def test_bridge_gene_is_found_by_propagation_only():
    B = 1000
    for seed in (0, 1, 2):
        x, lab, pairs = netrank_cohorts.bridge(seed)
        r = netrank.netrank_test(x, lab, pairs, B, damping=0.5, seed=seed)
        own = perm.perm_test(x, lab, B, seed=seed)
        b = netrank_cohorts.BRIDGE
        assert r.P[b] <= 0.01 and own.P[b] > 0.05, (seed, r.P[b], own.P[b])
        assert r.S[b] == 0.0 and r.degree[b] == 10


def test_null_cohort_share_of_small_p_values():
    for seed in (0, 1, 2):
        x, lab, pairs = netrank_cohorts.null(seed)
        r = netrank.netrank_test(x, lab, pairs, 200, damping=0.5, seed=seed)
        assert 0.005 <= (r.P <= 0.05).mean() <= 0.12, seed


# ----------------------------------------------------------------------------------------------------- C ABI
def test_entry_points_refuse_bad_sizes_and_launch_nothing():
    capi, lib = _lib()
    import torch
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p, st, N = buf.data_ptr(), _st(), None
    q = p + 4096                                        # a second buffer for x_out
    before = capi.launch_count()
    bad = [lib.g2v_nr_seed(N, 1, 1, 10, 3, p, p, p, 1, st), lib.g2v_nr_seed(p, 1, 1, 10, 3, p, p, N, 1, st),
           lib.g2v_nr_seed(p, 0, 1, 10, 3, p, p, p, 1, st), lib.g2v_nr_seed(p, 2, 1, 10, 3, p, p, p, 1, st),
           lib.g2v_nr_seed(p, 1, 0, 10, 3, p, p, p, 1, st), lib.g2v_nr_seed(p, 1, (1 << 24) + 1, 10, 3, p, p, p, 1, st),
           lib.g2v_nr_seed(p, 1, 1, 2, 1, p, p, p, 1, st), lib.g2v_nr_seed(p, 1, 1, 32769, 3, p, p, p, 1, st),
           lib.g2v_nr_seed(p, 1, 1, 10, 0, p, p, p, 1, st), lib.g2v_nr_seed(p, 1, 1, 10, 10, p, p, p, 1, st),
           lib.g2v_nr_seed(p, 1, 1, 10, 3, p, p, p, (1 << 20) + 1, st),
           lib.g2v_nr_step(N, p, p, p, p, p, q, 1, 1, 0, 1, 0.5, st),
           lib.g2v_nr_step(p, p, p, p, p, p, N, 1, 1, 0, 1, 0.5, st),
           lib.g2v_nr_step(p, p, p, p, p, q, q, 1, 1, 0, 1, 0.5, st),         # x_out = x_in
           lib.g2v_nr_step(p, p, p, p, q, p, q, 1, 1, 0, 1, 0.5, st),         # x_out = S
           lib.g2v_nr_step(p, p, p, p, p, p, q, 0, 1, 0, 1, 0.5, st),
           lib.g2v_nr_step(p, p, p, p, p, p, q, 1, 0, 0, 1, 0.5, st),
           lib.g2v_nr_step(p, p, p, p, p, p, q, 1, 4, 3, 2, 0.5, st),         # past ld
           lib.g2v_nr_step(p, p, p, p, p, p, q, 1, 4, -1, 2, 0.5, st),
           lib.g2v_nr_step(p, p, p, p, p, p, q, 1, 4, 0, 0, 0.5, st),
           lib.g2v_nr_step(p, p, p, p, p, p, q, 1, 1, 0, 1, 0.96, st),
           lib.g2v_nr_step(p, p, p, p, p, p, q, 1, 1, 0, 1, -0.1, st),
           lib.g2v_nr_step(p, p, p, p, p, p, q, 1, 1, 0, 1, float("nan"), st),
           lib.g2v_nr_tally(N, 1, 1, 1, p, p, st), lib.g2v_nr_tally(p, 1, 1, 1, p, N, st),
           lib.g2v_nr_tally(p, 0, 1, 1, p, p, st), lib.g2v_nr_tally(p, 1, 0, 1, p, p, st),
           lib.g2v_nr_tally(p, 1, 2, 1, p, p, st)]
    assert all(rc != 0 for rc in bad)
    assert capi.launch_count() == before and len(lib.g2v_last_error()) > 0
    assert lib.g2v_nr_tile_cols(0) == 0 and lib.g2v_nr_tile_cols(1 << 25) == 0
    t = lib.g2v_nr_tile_cols(7523)
    assert t >= 32 and t % 32 == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------- CLI
def test_command_line_writes_the_scores_and_leaves_the_other_files_alone(tmp_path, capsys):
    from g2vec_b200 import cli, signature
    from tests import helpers
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    base = ["-r", "2", "-e", "5", "-n", "20", "--seed", "3", "--deterministic", "--signature-cv", "20"]
    a, b, c = str(tmp_path / "plain"), str(tmp_path / "nr"), str(tmp_path / "again")
    cli.main([ef, cf, nf, a] + base)
    log_a = capsys.readouterr().out
    cli.main([ef, cf, nf, b] + base + ["--netrank", "200"])
    log_b = capsys.readouterr().out
    cli.main([ef, cf, nf, c] + base + ["--netrank", "200"])
    capsys.readouterr()
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt", "_signature.txt"):
        assert open(a + suffix).read() == open(b + suffix).read(), suffix
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt", "_signature.txt", "_netrank.txt"):
        assert open(b + suffix).read() == open(c + suffix).read(), suffix
    assert not os.path.exists(a + "_netrank.txt")
    import re
    untimed = lambda log, prefix: [re.sub(r" \([0-9.]+ sec\)$", "", l).replace(prefix, "RES")
                                   for l in log.splitlines()]
    extra = [l for l in untimed(log_b, b) if l not in untimed(log_a, a)]
    assert len(extra) == 3 and extra[0].startswith("Namespace(") and "netrank=200, netrank_damping=0.5" in extra[0]
    assert extra[1].startswith("    netrank: 200 label permutations, d = 0.5 (40 iterations), 7523 genes, 140902 pairs: ")
    assert extra[2] == "    RES_netrank.txt"
    data = cli.load_data(ef)
    data["label"] = cli.match_labels(cli.load_clinical(cf), data["sample"])
    data, net = cli.restrict(data, cli.load_network(nf))
    gi = {g: i for i, g in enumerate(data["gene"])}
    pairs = diffcoex.pairs_from_edges([gi[e[0]] for e in net["edge"]], [gi[e[1]] for e in net["edge"]])
    r = netrank.netrank_test(data["expr"], data["label"], pairs, 200, damping=0.5, seed=3)
    g = data["gene"]
    bm = open(b + "_biomarkers.txt").read().split()[1:]
    is_bm = np.array([s in set(bm) for s in g])
    lgroup = [int(l.split("\t")[1]) for l in open(b + "_lgroups.txt").read().splitlines()[1:]]
    # the AUC of top_netrank is its row of a cv_fits call whose head also holds the biomarkers and top_t
    x, lab = perm.check_inputs(data["expr"], data["label"], 1)
    p = len(bm)
    head = np.stack([np.sort([gi[s] for s in bm]).astype(np.int32), signature.top_t(data["expr"], data["label"], p),
                     netrank.top_netrank(r, p)])
    auc = signature.cv_fits(x, lab, head, 0, 10, 5, 3)[2]
    sig_auc = float([l for l in open(b + "_signature.txt").read().splitlines() if l.startswith("biomarkers\t")][0]
                    .split("\t")[2])
    line = netrank.summary(r, 0.5, 140902, is_bm, (float(auc[2].reshape(-1).mean()), float(auc[0].reshape(-1).mean())))
    assert abs(float(auc[0].reshape(-1).mean()) - sig_auc) < 1e-6
    assert extra[1] == "    " + line
    rows = open(b + "_netrank.txt").read().splitlines()
    assert rows[0] == "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tDegree\tS\tScore\tRank\tP\tQ\tBiomarker"
    assert len(rows) == 7523 + 2 and rows[-1] == line
    rank = np.empty(7523, np.int64)
    rank[r.order] = np.arange(1, 7524)
    for j in range(0, 7523, 37):
        assert rows[1 + j] == "%s\t%d\t%d\t%.6f\t%.6f\t%d\t%.6g\t%.6g\t%d" % (
            g[j], lgroup[j], r.degree[j], r.S[j], r.score[j], rank[j], r.P[j], r.Q[j], is_bm[j])
