"""Graph side of the walk path: edge weighting, CSR construction, weight quantisation and the
synthetic networks of the benchmark configs (SURVEY.md 8d).

Reference: construct_adjMat / compute_PCC, /root/reference/G2Vec.py:354-391 -- a dense
[V, V] float32 matrix with adjMat[src][dest] = |PCC| when |PCC| > 0.5.  Here the same graph
is CSR (rows = out-edges, neighbours ascending by dest = dense row order, which the sampler's
inverse-CDF parity needs) and is never materialised densely.
"""
import numpy as np

Q_ONE = 65536  # weights are quantised to q = rint(w * 2^16); |PCC| in (0.5, 1] -> [32769, 65536]
Q_MAX = 1 << 24


def quantise_weights(w):
    """float weights -> uint32 integer weights for the bit-exact integer sampler."""
    w = np.asarray(w, dtype=np.float32)
    if w.size and (not np.isfinite(w).all() or (w < 0).any()):
        raise ValueError("edge weights must be finite and non-negative")
    q = np.rint(w.astype(np.float64) * Q_ONE)
    q[(w > 0) & (q < 1)] = 1
    if q.size and q.max() > Q_MAX:
        raise ValueError("edge weight too large to quantise (max %g)" % float(w.max()))
    return q.astype(np.uint32)


def csr_from_edges(src, dst, w, V):
    """Directed edges -> CSR sorted by (src, dst).  A duplicated (src, dst) keeps the LAST
    weight, as repeated assignment to adjMat[src][dest] does (G2Vec.py:390)."""
    src = np.asarray(src, dtype=np.int64); dst = np.asarray(dst, dtype=np.int64)
    w = np.asarray(w, dtype=np.float32)
    if src.size:
        if src.min() < 0 or dst.min() < 0 or src.max() >= V or dst.max() >= V:
            raise ValueError("edge endpoint out of range")
    key = src * V + dst
    order = np.argsort(key, kind="stable")
    key = key[order]
    last = np.ones(key.shape[0], dtype=bool)
    last[:-1] = key[1:] != key[:-1]
    order = order[last]
    s, d = src[order], dst[order]
    rowptr = np.zeros(V + 1, dtype=np.int64)
    np.add.at(rowptr, s + 1, 1)
    rowptr = np.cumsum(rowptr)
    if rowptr[-1] >= 2**31:
        raise ValueError("too many edges for int32 CSR")
    return rowptr.astype(np.int32), d.astype(np.int32), w[order]


def csr_from_dense(adjMat):
    """The reference's dense adjacency (generate_pathSet's first argument) -> CSR."""
    A = np.asarray(adjMat)
    if A.ndim != 2 or A.shape[0] != A.shape[1]:
        raise ValueError("adjMat must be square")
    r, c = np.nonzero(A)
    rowptr = np.zeros(A.shape[0] + 1, dtype=np.int64)
    np.add.at(rowptr, r + 1, 1)
    return np.cumsum(rowptr).astype(np.int32), c.astype(np.int32), A[r, c].astype(np.float32)


def edge_abs_pcc(expr_group, src, dst):
    """|PCC| per edge over one group's samples (G2Vec.py:354-368, 378-385): population std,
    weight 0 when either gene has zero variance.  Vectorised over edges in float32; agrees with
    the reference's per-edge loop to ~1e-6 (summation order), see tests."""
    X = np.asarray(expr_group, dtype=np.float32)
    mu = X.mean(axis=0, dtype=np.float32)
    sd = X.std(axis=0, dtype=np.float32)
    ok = sd > 0
    Z = np.zeros_like(X)
    Z[:, ok] = (X[:, ok] - mu[ok]) / sd[ok]
    src = np.asarray(src); dst = np.asarray(dst)
    out = np.empty(src.shape[0], dtype=np.float32)
    step = 1 << 16
    for a in range(0, src.shape[0], step):
        s, d = src[a:a + step], dst[a:a + step]
        out[a:a + step] = np.abs((Z[:, s] * Z[:, d]).mean(axis=0, dtype=np.float32))
    return out


CORR_METHODS = {"pearson": 0, "spearman": 1, "bicor": 2}    # codes of g2v_corr_transform (pearson: g2v_pcc_zscore)
CORR_MAX_SAMPLES = 32768                                    # G2V_CORR_MAX_SAMPLES: samples per group, spearman / bicor


def check_corr(method, threshold):
    """ValueError unless `method` is one of CORR_METHODS and the cutoff is finite with 0 <= threshold < 1."""
    if method not in CORR_METHODS:
        raise ValueError("correlation method must be one of %s, got %r" % (", ".join(CORR_METHODS), method))
    t = float(threshold)
    if not (np.isfinite(t) and 0.0 <= t < 1.0):
        raise ValueError("correlation cutoff must be a finite number with 0 <= T < 1, got %r" % threshold)


def _check_expr(x, method):
    """The rank and biweight transforms need finite values (bicor would make NaN of inf * 0)."""
    if method != "pearson" and x.size and not np.isfinite(x).all():
        raise ValueError("correlation method %r needs finite expression values" % method)


def corr_transform(expr_group, method):
    """Host restatement of g2v_corr_transform: the per-gene transform z [S, V] (float32, sample-major as the
    group's expression) with mean_s z[s, a] * z[s, b] = the coefficient of genes a and b (DESIGN.md §4.22).
    spearman: Pearson z-score of the average ranks, population std, 0 for a constant gene -- the same bits as the
    kernel (every sum is exact).  bicor: Tukey's biweight, t * sqrt(S) / ||t||, and the Pearson z-score (float64)
    for a gene with MAD = 0; agrees with the kernel to float32 rounding."""
    if method not in ("spearman", "bicor"):
        raise ValueError("corr_transform: method must be 'spearman' or 'bicor', got %r" % (method,))
    X = np.asarray(expr_group, dtype=np.float32)
    _check_expr(X, method)
    S, V = X.shape
    if S == 0:
        return np.zeros((S, V), dtype=np.float32)
    if method == "spearman":
        Xc = X + np.float32(0.0)                            # -0.0 ties with +0.0
        srt = np.sort(Xc, axis=0)
        d = np.empty((S, V), dtype=np.int64)                # 2r - (S+1), r = average rank
        for v in range(V):
            d[:, v] = (np.searchsorted(srt[:, v], Xc[:, v], "left") + np.searchsorted(srt[:, v], Xc[:, v], "right")
                       - S)
        ss = (d * d).sum(axis=0)
        sd = np.sqrt(ss.astype(np.float64) * 0.25 / S)
        with np.errstate(divide="ignore", invalid="ignore"):
            z = np.where(sd > 0, d * 0.5 / sd, 0.0)
        return z.astype(np.float32)
    Xd = X.astype(np.float64)
    z = np.zeros((S, V), dtype=np.float64)
    med = np.median(Xd, axis=0)
    dev = Xd - med
    mad = np.median(np.abs(dev), axis=0)
    ok = mad > 0
    u = dev[:, ok] / (9.0 * mad[ok])
    t = np.where(np.abs(u) < 1.0, dev[:, ok] * (1.0 - u * u) ** 2, 0.0)
    z[:, ok] = t * (np.sqrt(S) / np.sqrt((t * t).sum(axis=0)))
    xf = Xd[:, ~ok]                                         # MAD = 0: WGCNA's individual Pearson fallback
    mu = xf.mean(axis=0)
    sd = np.sqrt(((xf - mu) ** 2).sum(axis=0) / S)
    with np.errstate(divide="ignore", invalid="ignore"):
        z[:, ~ok] = np.where(sd > 0, (xf - mu) / sd, 0.0)
    return z.astype(np.float32)


def edge_abs_corr(expr_group, src, dst, method="pearson"):
    """|coefficient| per edge over one group's samples: edge_abs_pcc for 'pearson', else the mean product of the
    two genes' corr_transform columns (summed in float64)."""
    if method == "pearson":
        return edge_abs_pcc(expr_group, src, dst)
    Z = corr_transform(expr_group, method)
    S = Z.shape[0]
    src = np.asarray(src); dst = np.asarray(dst)
    out = np.empty(src.shape[0], dtype=np.float32)
    step = 1 << 16
    for a in range(0, src.shape[0], step):
        s, d = src[a:a + step], dst[a:a + step]
        acc = (Z[:, s].astype(np.float64) * Z[:, d].astype(np.float64)).sum(axis=0)
        out[a:a + step] = np.abs(acc / S) if S else 0.0
    return out


def group_csr(expr, label, group, src, dst, threshold=0.5, method="pearson"):
    """construct_adjMat (G2Vec.py:370-391) as CSR for one patient group; an edge is kept iff its |coefficient| of
    `method` (CORR_METHODS) is > threshold."""
    check_corr(method, threshold)
    V = expr.shape[1]
    w = edge_abs_corr(expr[np.asarray(label) == group], src, dst, method)
    # last assignment wins BEFORE thresholding only matters for duplicated edges with equal weight
    keep = w > threshold
    return csr_from_edges(np.asarray(src)[keep], np.asarray(dst)[keep], w[keep], V)


def group_csr_gpu(expr, label, group, src, dst, threshold=0.5, device=None, method="pearson"):
    """construct_adjMat (G2Vec.py:370-391) for one group on the GPU: z-scores (csrc/g2v_pcc.cu, or the Spearman /
    bicor transform of csrc/g2v_corr.cu) and per-edge |coefficient| by csrc/g2v_pcc.cu, threshold + (src, dest)
    sort + last-duplicate-wins on the device with torch as plumbing.  Returns device tensors (rowptr int32 [V+1],
    col int32 [nnz], w float32 [nnz])."""
    check_corr(method, threshold)
    x = np.ascontiguousarray(np.asarray(expr, dtype=np.float32)[np.asarray(label) == group])
    S, V = x.shape
    _check_expr(x, method)
    if method != "pearson" and S > CORR_MAX_SAMPLES:
        raise ValueError("correlation method %r takes at most %d samples per group, got %d"
                         % (method, CORR_MAX_SAMPLES, S))
    import torch
    from . import _capi
    lib = _capi.load()
    if not torch.cuda.is_available():
        raise RuntimeError("g2vec_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    xd = torch.from_numpy(x).to(dev)
    sd = torch.from_numpy(np.ascontiguousarray(src, dtype=np.int32)).to(dev)
    dd = torch.from_numpy(np.ascontiguousarray(dst, dtype=np.int32)).to(dev)
    E = int(sd.shape[0])
    z = torch.empty((V, S), dtype=torch.float32, device=dev)
    w = torch.empty((E,), dtype=torch.float32, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    if method == "pearson":
        _capi.check(lib.g2v_pcc_zscore(xd.data_ptr(), S, V, z.data_ptr(), st), "g2v_pcc_zscore")
    else:
        _capi.check(lib.g2v_corr_transform(xd.data_ptr(), S, V, CORR_METHODS[method], z.data_ptr(), st),
                    "g2v_corr_transform")
    _capi.check(lib.g2v_pcc_edge_weights(z.data_ptr(), S, V, sd.data_ptr(), dd.data_ptr(), E, w.data_ptr(), st),
                "g2v_pcc_edge_weights")
    keep = w > threshold
    key = sd[keep].to(torch.int64) * V + dd[keep].to(torch.int64)
    wk = w[keep]
    key, order = torch.sort(key, stable=True)
    wk = wk[order]
    last = torch.ones_like(key, dtype=torch.bool)
    last[:-1] = key[1:] != key[:-1]                    # adjMat[src][dest] = w: the last duplicate wins
    key, wk = key[last], wk[last]
    rowptr = torch.zeros(V + 1, dtype=torch.int64, device=dev)
    rowptr[1:] = torch.cumsum(torch.bincount(key // V, minlength=V), dim=0)
    return rowptr.to(torch.int32), (key % V).to(torch.int32), wk


def synthetic_graph(V, E, group, seed=1000):
    """SURVEY.md 8d generator: E distinct ordered pairs (src != dest) uniform over V^2 from
    numpy Generator(PCG64(seed + group)), weights U(0.5, 1.0) float32, sorted by (src, dest)."""
    rng = np.random.Generator(np.random.PCG64(seed + group))
    need = E
    keys = np.empty(0, dtype=np.int64)
    while True:
        cand = rng.integers(0, V * V, size=int(need * 1.1) + 16, dtype=np.int64)
        cand = cand[(cand // V) != (cand % V)]
        keys = np.unique(np.concatenate([keys, cand]))
        if keys.shape[0] >= E:
            break
        need = E - keys.shape[0]
    if keys.shape[0] > E:
        keys = np.sort(rng.choice(keys, size=E, replace=False))
    w = rng.uniform(0.5, 1.0, size=E).astype(np.float32)
    w = np.maximum(w, np.float32(0.5000001))
    src, dst = keys // V, keys % V
    rowptr = np.zeros(V + 1, dtype=np.int64)
    np.add.at(rowptr, src + 1, 1)
    return np.cumsum(rowptr).astype(np.int32), dst.astype(np.int32), w


BENCH_CONFIGS = {
    # name: (V, E per group, D, lenPath)  -- BASELINE.json configs[1..4]
    "syn10k": (10_000, 500_000, 128, 80),
    "syn20k": (20_000, 2_000_000, 256, 80),
    "syn50k": (50_000, 5_000_000, 128, 160),
    "stress200k": (200_000, 20_000_000, 512, 80),
}
