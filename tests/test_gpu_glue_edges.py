"""Exact checks of the glue kernels at the sizes where their extra branches start: the set pipeline over more than 1024
scan tiles (the multi-chunk carry of the scan), canonicalisation of rows longer than 1024 genes (opt-in shared
memory), and the edge weights against float64 numpy on tiny, constant, offset and perfectly correlated data."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
PAD = 2 ** 31 - 1


@pytest.fixture(scope="module")
def lib():
    import torch
    assert torch.cuda.is_available()
    from g2vec_b200 import _capi
    return _capi.load()


def stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def canonicalise(lib, nodes):
    import torch
    from g2vec_b200 import _capi
    d = torch.from_numpy(np.ascontiguousarray(nodes, np.int32)).cuda()
    n, L = d.shape
    rows = torch.empty_like(d)
    key = torch.empty(n, dtype=torch.int64, device="cuda")
    _capi.check(lib.g2v_paths_canonicalise(d.data_ptr(), n, L, rows.data_ptr(), key.data_ptr(), stream()),
                "g2v_paths_canonicalise")
    return rows.cpu().numpy(), key.cpu().numpy()


@pytest.mark.parametrize("n", [512 * 1024 - 1, 512 * 1024, 512 * 1024 + 1, 600_000])
def test_set_pipeline_over_more_than_1024_scan_tiles(lib, n):
    import torch
    from g2vec_b200 import paths
    rs = np.random.RandomState(n % 1000)
    V, L = 3000, 6
    lens = rs.randint(1, L + 1, n).astype(np.int32)
    nodes = np.full((n, L), -1, np.int32)
    step = rs.randint(1, V // L, n)                                   # distinct genes per row, in visit order
    walk = (rs.randint(0, V, n)[:, None] + step[:, None] * np.arange(L)[None, :]) % V
    for l in range(1, L + 1):
        idx = np.nonzero(lens == l)[0]
        nodes[idx, :l] = walk[idx, :l]
    group = (np.arange(n) >= n // 2).astype(np.uint8)
    # duplicates inside a group (some permuted: the same path in another visit order), paths common to both groups,
    # spread over the whole list so that kept rows sit in every scan chunk
    src = rs.randint(0, n, 40_000); dst = rs.randint(0, n, 40_000)
    for a, b in zip(src, dst):
        nodes[b] = -1
        nodes[b, :lens[a]] = rs.permutation(nodes[a, :lens[a]])
        lens[b] = lens[a]
    rows, key = canonicalise(lib, nodes)
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).astype(dt)).cuda()
    rowptr, gene, label, code = paths.build_windows(dev(rows, np.int32), dev(lens, np.int32), dev(key, np.int64),
                                                    dev(group, np.uint8), V)
    # Python sets: first occurrence per group, minus the paths of both groups, in input order
    tup = [tuple(r[:l]) for r, l in zip(rows.tolist(), lens.tolist())]
    seen = [set(), set()]
    first = []
    for i, t in enumerate(tup):
        g = int(group[i])
        if t not in seen[g]:
            seen[g].add(t)
            first.append(i)
    common = seen[0] & seen[1]
    kept = [i for i in first if tup[i] not in common]
    assert len(common) > 100 and len(kept) < len(first)
    want_lens = np.array([len(tup[i]) for i in kept], np.int64)
    want_rowptr = np.concatenate([[0], np.cumsum(want_lens)])
    assert (rowptr.cpu().numpy() == want_rowptr).all()
    assert (gene.cpu().numpy() == np.concatenate([tup[i] for i in kept])).all()
    assert (label.cpu().numpy() == group[kept]).all()
    fg = np.zeros(V, np.int64); fp = np.zeros(V, np.int64)
    for i in kept:
        (fp if group[i] else fg)[list(tup[i])] += 1
    want_code = np.where(fg + fp == 0, -1, np.where(fg > fp, 0, np.where(fg < fp, 1, 2)))
    assert (code.cpu().numpy() == want_code).all()


@pytest.mark.parametrize("L", [1024, 1025, 2048, 4096])
def test_canonicalise_long_rows_equals_numpy_sort(lib, L):
    rs = np.random.RandomState(L)
    n = 300
    nodes = np.full((n, L), -1, np.int32)
    lens = rs.randint(0, L + 1, n)
    lens[:3] = [L, L - 1, 1]
    for i, l in enumerate(lens):
        nodes[i, :l] = rs.choice(2 * L, l, replace=False)
    nodes[7] = np.where(nodes[7] < 0, PAD, nodes[7])                  # INT32_MAX padding is accepted too
    perm_of = {10: 0, 11: 1, 12: 5}                                   # rows that are permutations of other rows
    for b, a in perm_of.items():
        nodes[b] = -1
        nodes[b, :lens[a]] = rs.permutation(nodes[a, :lens[a]])
    rows, key = canonicalise(lib, nodes)
    want = np.where(nodes < 0, PAD, nodes)
    want = np.sort(want.astype(np.int64), axis=1).astype(np.int32)
    assert (rows == want).all()
    assert (key >= 0).all()
    for b, a in perm_of.items():
        assert key[b] == key[a]
    assert len(set(key.tolist())) == len({tuple(r) for r in want.tolist()})


def path_graph(V=3000):
    """0 -> 1 -> ... -> V-1: walker v visits v, v+1, ... up to the end or L nodes."""
    rp = np.minimum(np.arange(V + 1), V - 1).astype(np.int32)
    return rp, np.arange(1, V, dtype=np.int32), np.full(V - 1, 50000, np.uint32)


@pytest.mark.parametrize("L,vis", [(4096, "bitmap"), (1365, "hash")])
def test_fused_canonical_walks_longer_than_300_nodes(lib, monkeypatch, L, vis):
    """The sampler's fused tuple(sorted(path)) epilogue on walks of up to 3000 nodes: the bitmap visited set at
    L = 4096, and the hash set at L = 1365, the largest L the header promises for any V (the bitonic sort over a
    2048-slot path buffer).  Rows equal the oracle's walks sorted, keys equal g2v_paths_canonicalise's."""
    import torch
    import oracle
    import g2vec_b200 as g2v
    from g2vec_b200 import paths
    monkeypatch.setenv("G2V_WALK_VISITED", vis)
    rp, col, q = path_graph()
    V = len(rp) - 1
    want, wl = oracle.walks(rp, col, q, L, 3, 1, 0, V)
    assert wl.max() == min(L, V) and (wl == np.minimum(V - np.arange(V), L)).all()
    g = g2v.WalkGraph(rp, col, qw=q)
    rows, lens, key = g2v.generate_paths(g, L, 1, seed=3, group=1, canonical=True)
    torch.cuda.synchronize()
    assert (lens.cpu().numpy() == wl).all()
    want_rows = np.where(want < 0, PAD, want)
    want_rows = np.sort(want_rows.astype(np.int64), axis=1).astype(np.int32)
    assert (rows.cpu().numpy() == want_rows).all()
    _, want_key = canonicalise(lib, want)
    assert (key.cpu().numpy() == want_key).all()


def test_hash_visited_set_at_4096_nodes_is_refused(lib, monkeypatch):
    """A hash visited set at L = 4096 (3L slots + a 4096-slot path buffer per warp) does not fit shared memory: the call
    is refused with the lenPath message, leaves no CUDA error behind, and the bitmap form of the same call then runs."""
    import torch
    import g2vec_b200 as g2v
    rp, col, q = path_graph()
    g = g2v.WalkGraph(rp, col, qw=q)
    monkeypatch.setenv("G2V_WALK_VISITED", "hash")
    for canonical in (True, False):
        with pytest.raises(RuntimeError, match="lenPath"):
            g2v.generate_paths(g, 4096, 1, seed=3, group=1, canonical=canonical, walker_end=4)
    torch.cuda.synchronize()
    monkeypatch.setenv("G2V_WALK_VISITED", "bitmap")
    nodes, lens = g2v.generate_paths(g, 4096, 1, seed=3, group=1, walker_end=4)
    torch.cuda.synchronize()
    assert lens.cpu().tolist() == [3000, 2999, 2998, 2997]


def pcc64(expr, src, dst):
    x = expr.astype(np.float64)
    mu = x.mean(0)
    sd = np.where(np.ptp(x, 0) > 0, np.sqrt(((x - mu) ** 2).mean(0)), 0.0)   # a constant gene has no spread at all
    z = np.where(sd > 0, (x - mu) / np.where(sd > 0, sd, 1), 0.0)
    return np.abs((z[:, src] * z[:, dst]).mean(0)), z


def pcc_gpu(lib, expr, src, dst):
    import torch
    from g2vec_b200 import _capi
    S, V = expr.shape
    x = torch.from_numpy(np.ascontiguousarray(expr, np.float32)).cuda()
    z = torch.empty(V * S, dtype=torch.float32, device="cuda")
    _capi.check(lib.g2v_pcc_zscore(x.data_ptr(), S, V, z.data_ptr(), stream()), "g2v_pcc_zscore")
    s = torch.from_numpy(src.astype(np.int32)).cuda(); d = torch.from_numpy(dst.astype(np.int32)).cuda()
    w = torch.empty(len(src), dtype=torch.float32, device="cuda")
    _capi.check(lib.g2v_pcc_edge_weights(z.data_ptr(), S, V, s.data_ptr(), d.data_ptr(), len(src), w.data_ptr(),
                                         stream()), "g2v_pcc_edge_weights")
    return w.cpu().numpy(), z.cpu().numpy().reshape(V, S)


@pytest.mark.parametrize("S", [1, 2, 7, 8, 9, 1000])
@pytest.mark.parametrize("V", [1, 31, 33])
@pytest.mark.parametrize("kind", ["normal", "offset"])
def test_edge_weights_against_float64(lib, S, V, kind):
    rs = np.random.RandomState(S * 100 + V)
    if kind == "normal":
        expr = rs.randn(S, V).astype(np.float32)
    else:                                                             # 1e4 offset, 1e-2 spread: cancellation
        expr = (1e4 + 1e-2 * rs.randn(S, V)).astype(np.float32)
    const = [g for g in range(V) if g % 5 == 2]
    for k, g in enumerate(const):                                     # constant genes, zero and non-zero values
        expr[:, g] = [0.0, 0.1, 3.7, -1e4, 1e4 + 0.01][k % 5]
    if V >= 4:
        expr[:, 1] = np.float32(2) * expr[:, 0]                       # perfectly correlated ...
        expr[:, 3] = -expr[:, 0]                                      # ... and anti-correlated (exact in float32)
    src, dst = np.meshgrid(np.arange(V), np.arange(V))
    src, dst = src.ravel(), dst.ravel()
    w64, z64 = pcc64(expr, src, dst)
    w, z = pcc_gpu(lib, expr, src, dst)
    u = 2.0 ** -24
    zerr = 2 * u * np.abs(z64) + 1e-300
    assert (np.abs(z - z64.T) <= zerr.T).all()
    mag = (np.abs(z64[:, src]) * np.abs(z64[:, dst])).mean(0)
    assert (np.abs(w - w64) <= 4 * u * mag + u * w64).all()
    for g in const:
        assert (z[g] == 0).all() and (w[(src == g) | (dst == g)] == 0).all()
    if V >= 4 and S >= 2 and np.ptp(expr[:, 0]) > 0:
        from g2vec_b200 import graph
        pair = ((src == 0) & (dst == 1)) | ((src == 0) & (dst == 3)) | ((src == 1) & (dst == 3))
        assert (graph.quantise_weights(w[pair]) == 65536).all()
