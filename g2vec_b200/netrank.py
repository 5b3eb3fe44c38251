"""Network-propagated gene scores with a label-permutation test, NetRank (DESIGN.md §4.35): each gene's association
with the good / poor label, smoothed over the interaction network by personalised PageRank (GeneRank, Morrison et
al. 2005; NetRank, Winter et al. 2012), with a raw permutation p-value and the Benjamini & Hochberg q-value per gene.

Per labelling the seed is s_j = sqrt(rho_j), rho_j = perm.rho_of(N_j, W_j) from perm.prepare's exact integer sums
(|point-biserial r|, 0 for a constant gene).  From x = s, T iterations of the column-normalised NetRank step
x_j <- (1 - d) s_j + d sum over the neighbours i of j of x_i / deg_i give the score x^(T); the operator is
column-substochastic, so |x^(T) - x*|_1 <= d^T |s - x*|_1, and T is the smallest with d^T <= 1e-12.

Host side (NumPy): the checks, perm.prepare, the CSR and the byte planes.  Device side (csrc/g2v_nr.cu,
csrc/g2v_perm.cu): the observed labelling as a one-row M through g2v_perm_sums, g2v_nr_seed and T g2v_nr_step; then
per chunk of permutations g2v_perm_labels (the rows of --permutations for the same seed), g2v_perm_sums, g2v_nr_seed,
T g2v_nr_step per column tile and g2v_nr_tally.  The counts compare float64 scores computed in a fixed order, so P and
Q depend only on the expression, the labels, the pairs, d, the seed and B.
"""
from collections import namedtuple

import numpy as np

from . import perm

MAX_PERMUTATIONS = 1 << 20   # G2V_NR_MAX_ROWS
MAX_PAIRS = 1 << 26
MAX_GENES = 1 << 24          # G2V_NR_MAX_GENES
MAX_DAMPING = 0.95           # G2V_NR_MAX_DAMPING
TOLERANCE = 1e-12            # d^T

NetRankResult = namedtuple("NetRankResult", "degree S score order P Q count n_iter n_perm")
NetRankResult.__doc__ = """netrank_test's result, every array over the genes in their input order except `order`:
degree  int64, the number of pairs that hold the gene;
S       the observed seed sqrt(rho), |point-biserial r| in [0, 1];
score   the observed propagated score x^(T);
order   the genes by score descending, ties by index (rank r -> gene order[r]);
P       (1 + count) / (B + 1);  Q: Benjamini-Hochberg q-values of P;
count   #{b : score_b >= score_obs}, compared in float64;
n_iter  T;  n_perm: B."""


def n_iterations(d):
    """T: 0 when d = 0, else the smallest T >= 1 with d^T <= 1e-12, d^T formed by T float64 products from 1.0."""
    d = float(d)
    if d == 0.0:
        return 0
    p, T = 1.0, 0
    while True:
        p *= d
        T += 1
        if p <= TOLERANCE:
            return T


def check_inputs(expr, label, pairs, n_perm, damping):
    """ValueError unless the test can run: perm.check_inputs' conditions (labels 0 and 1 both present, 3 <= n <= 32768
    samples with label 0 or 1, finite expression), 1 <= n_perm <= 2^20, a finite damping 0 <= d <= 0.95, and 1 to 2^26
    pairs (i, j) of gene indices with i < j, sorted and distinct (diffcoex.pairs_from_edges makes them).  Returns
    (x, lab, pairs): the used samples' expression as float64 [n, G], their labels and the pairs as int32 [E, 2].  Needs
    no GPU."""
    x = np.asarray(expr)
    lab = np.asarray(label).reshape(-1)
    if x.ndim != 2 or x.shape[0] != lab.shape[0]:
        raise ValueError("netrank: expression must be [samples, genes] with one label per sample, got %s and %d labels"
                         % (x.shape, lab.shape[0]))
    G = x.shape[1]
    if not 1 <= G <= MAX_GENES:
        raise ValueError("netrank: %d genes, must be in [1, %d]" % (G, MAX_GENES))
    try:
        B = int(n_perm)
    except (TypeError, ValueError):
        B = None
    if B is None or B != n_perm or not 1 <= B <= MAX_PERMUTATIONS:
        raise ValueError("netrank: the number of permutations must be an integer in [1, %d], got %r"
                         % (MAX_PERMUTATIONS, n_perm))
    try:
        d = float(damping)
    except (TypeError, ValueError):
        d = float("nan")
    if not (np.isfinite(d) and 0.0 <= d <= MAX_DAMPING):
        raise ValueError("netrank: the damping must be a finite number in [0, %g], got %r" % (MAX_DAMPING, damping))
    p = np.asarray(pairs)
    if p.ndim != 2 or p.shape[1] != 2 or not np.issubdtype(p.dtype, np.integer):
        raise ValueError("netrank: pairs must be an integer array [E, 2]")
    E = p.shape[0]
    if not 1 <= E <= MAX_PAIRS:
        raise ValueError("netrank: %d gene pairs, must be in [1, %d]" % (E, MAX_PAIRS))
    p = p.astype(np.int64)
    if (p[:, 0] < 0).any() or (p[:, 1] >= G).any() or (p[:, 0] >= p[:, 1]).any():
        raise ValueError("netrank: every pair must be (i, j) with 0 <= i < j < %d" % G)
    key = p[:, 0] * G + p[:, 1]
    if E > 1 and (np.diff(key) <= 0).any():
        raise ValueError("netrank: the pairs must be distinct and sorted by (i, j)")
    try:
        x, lab = perm.check_inputs(x, lab, 1)
    except ValueError as e:
        raise ValueError(str(e).replace("permutation test: ", "netrank: ")) from None
    return x, lab, p.astype(np.int32)


def csr(pairs, G):
    """The undirected network of the pairs as CSR: (rowptr int32 [G + 1], col int32 [2E], deg int64 [G], w float64
    [G]); each row's neighbours ascending, w = 1.0 / deg (0 for a gene without neighbours, never read)."""
    p = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    src = np.concatenate([p[:, 0], p[:, 1]])
    dst = np.concatenate([p[:, 1], p[:, 0]])
    o = np.lexsort((dst, src))
    deg = np.bincount(src, minlength=G).astype(np.int64)
    rowptr = np.zeros(G + 1, dtype=np.int64)
    np.cumsum(deg, out=rowptr[1:])
    w = np.zeros(G)
    np.divide(1.0, deg, out=w, where=deg > 0)
    return rowptr.astype(np.int32), dst[o].astype(np.int32), deg, w


def row_order(deg):
    """The order the step kernel's warps take the genes in: degree descending, ties by index."""
    return np.argsort(-np.asarray(deg), kind="stable").astype(np.int32)


def finish(S, score, deg, count, n_iter, n_perm):
    """Observed seed and score, degrees and counts -> NetRankResult."""
    B = int(n_perm)
    count = np.asarray(count, dtype=np.int64)
    P = (1.0 + count) / (B + 1.0)
    return NetRankResult(degree=deg, S=S, score=score, order=np.argsort(-score, kind="stable"), P=P, Q=perm.bh(P),
                         count=count, n_iter=int(n_iter), n_perm=B)


def top_netrank(res, p):
    """The p genes of highest score (ties by index), ascending."""
    return np.sort(res.order[:p]).astype(np.int32)


def jaccard(a, b):
    a, b = set(int(v) for v in a), set(int(v) for v in b)
    return len(a & b) / float(len(a | b)) if a | b else 0.0


def chunk_rows(S_pad, G, n_perm, max_chunk_bytes):
    """Permutations per chunk: M (S_pad bytes), A (8 G bytes), S and two x buffers (24 G bytes) of every row within
    max_chunk_bytes, at least 1 (the column buffers are then padded to a multiple of 32)."""
    return int(max(1, min(int(n_perm), int(max_chunk_bytes) // (S_pad + 32 * G))))


def propagate(lib, net, S, xa, xb, G, ld, n_cols, n_iter, damping, tile, stream):
    """T = n_iter steps of g2v_nr_step on columns 0 .. n_cols - 1 of S [G][ld], one column tile at a time (T steps on
    a tile before the next); net = (rowptr, col, w, rows) on the device.  Returns the buffer holding x^(T) (S itself
    when T = 0)."""
    from . import _capi
    rp, col, w, rows = net
    if n_iter == 0:
        return S
    for c0 in range(0, n_cols, tile):
        nc = min(tile, n_cols - c0)
        src, dst = S, xa
        for _ in range(n_iter):
            _capi.check(lib.g2v_nr_step(rp.data_ptr(), col.data_ptr(), w.data_ptr(), rows.data_ptr(), S.data_ptr(),
                                        src.data_ptr(), dst.data_ptr(), G, ld, c0, nc, float(damping), stream),
                        "g2v_nr_step")
            src, dst = dst, (xb if dst is xa else xa)
    return src


def netrank_test(expr, label, pairs, n_perm, damping=0.5, seed=0, max_chunk_bytes=None):
    """NetRank scores of every gene over the network of the pairs and their label-permutation test, on the GPU.

    expr: host float array [samples, genes]; label: one int per sample (0 good, 1 poor; other labels are left out);
    pairs: int [E, 2], (i, j) with i < j, sorted and distinct; n_perm: B, 1 <= B <= 2^20 permutations (the observed
    labelling is not among them), the rows perm.perm_test uses for the same seed; damping: d in [0, 0.95]; seed: the
    Philox key (--seed).  max_chunk_bytes: bound on the device memory of one chunk's rows, sums, seeds and scores
    (default: half the free device memory); the result does not depend on it.  Returns a NetRankResult; ValueError
    (before anything is uploaded) on inputs check_inputs refuses."""
    x, lab, pairs = check_inputs(expr, label, pairs, n_perm, damping)
    prep = perm.prepare(x, lab)
    import torch
    from . import _capi
    lib = _capi.load()
    if not torch.cuda.is_available():
        raise RuntimeError("g2vec_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    dev = torch.device("cuda", torch.cuda.current_device())
    n, k, B, G = prep["n"], prep["k"], int(n_perm), x.shape[1]
    d, T = float(damping), n_iterations(damping)
    rowptr, col, deg, w = csr(pairs, G)
    S_pad = -(-n // 32) * 32
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    pl_d, Q_d, W_d = up(perm.planes(prep["q"], np.arange(G))), up(prep["Q"]), up(prep["W"])
    net = (up(rowptr), up(col), up(w), up(row_order(deg)))
    st = torch.cuda.current_stream(dev).cuda_stream
    tile = int(lib.g2v_nr_tile_cols(G))
    if tile <= 0:
        _capi.check(1, "g2v_nr_tile_cols")

    def scores(M, nb, A, S, xa, xb, ld):
        _capi.check(lib.g2v_perm_sums(M.data_ptr(), pl_d.data_ptr(), nb, S_pad, G, A.data_ptr(), st), "g2v_perm_sums")
        _capi.check(lib.g2v_nr_seed(A.data_ptr(), nb, G, n, k, Q_d.data_ptr(), W_d.data_ptr(), S.data_ptr(), ld, st),
                    "g2v_nr_seed")
        return propagate(lib, net, S, xa, xb, G, ld, nb, T, d, tile, st)

    M1 = np.zeros((1, S_pad), dtype=np.uint8)
    M1[0, :n] = prep["obs"]
    obs = [torch.empty((1, G), dtype=torch.int64, device=dev)] + [torch.empty(G, dtype=torch.float64, device=dev)
                                                                  for _ in range(3)]
    S_obs = obs[1]
    score_obs = scores(up(M1), 1, *obs, 1)
    cnt = torch.zeros(G, dtype=torch.int64, device=dev)
    if max_chunk_bytes is None:
        max_chunk_bytes = torch.cuda.mem_get_info(dev)[0] // 2
    rows = chunk_rows(S_pad, G, B, max_chunk_bytes)
    ld = -(-rows // 32) * 32
    M = torch.empty((rows, S_pad), dtype=torch.uint8, device=dev)
    A = torch.empty((rows, G), dtype=torch.int64, device=dev)
    S, xa, xb = (torch.empty((G, ld), dtype=torch.float64, device=dev) for _ in range(3))
    obs_d = up(prep["obs"])
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    for b0 in range(0, B, rows):
        nb = min(rows, B - b0)
        _capi.check(lib.g2v_perm_labels(obs_d.data_ptr(), n, S_pad, seed, b0, nb, M.data_ptr(), st), "g2v_perm_labels")
        xT = scores(M, nb, A, S, xa, xb, ld)
        _capi.check(lib.g2v_nr_tally(xT.data_ptr(), G, nb, ld, score_obs.data_ptr(), cnt.data_ptr(), st),
                    "g2v_nr_tally")
    return finish(S_obs.cpu().numpy(), score_obs.cpu().numpy(), deg, cnt.cpu().numpy(), T, B)


def summary(res, damping, n_pairs, biomarker, auc=None):
    """The command line's line: the damping d, the pair count, biomarker bool [G]; top_netrank has as many genes as
    there are biomarkers; auc = the cross-validated AUC of (top_netrank, biomarkers) on --signature-cv's splits, or
    None."""
    bm = np.asarray(biomarker, dtype=bool)
    p = int(bm.sum())
    sq = res.Q <= 0.05
    line = ("netrank: %d label permutations, d = %g (%d iterations), %d genes, %d pairs: %d genes with Q <= 0.05 (%d "
            "of the biomarkers); top_netrank (%d genes) Jaccard %.3f with the biomarkers"
            % (res.n_perm, damping, res.n_iter, res.score.shape[0], n_pairs, int(sq.sum()),
               int((sq & bm).sum()), p, jaccard(top_netrank(res, p), np.nonzero(bm)[0])))
    if auc is not None:
        line += "; CV AUC %.3f (top_netrank), %.3f (biomarkers)" % auc
    return line
