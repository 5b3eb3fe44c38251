"""Label-permutation test of differential co-expression for every network pair (DESIGN.md §4.30): per gene pair the
Pearson correlations over the good and the poor samples, Fisher's z contrast, a raw permutation p-value, the
Westfall & Young step-down maxT adjusted p-value and the Benjamini & Hochberg q-value (DiffCoEx, DCGL and others).

The test is always Pearson's coefficient, whatever --correlation chose for the walks' graphs.

Host side (NumPy): the samples with label 0 or 1, each gene quantised to integers q with |q| <= 2^16
(perm.quantise(x, bits=16)), the pairs, and r and D of the observed labelling from the device's exact sums.
Device side (csrc/g2v_dcx.cu, csrc/g2v_perm.cu): one launch each of g2v_perm_sums and g2v_dcx_sums (twice) on the
all-ones and observed rows for the totals and the observed sums; then per chunk of permutations g2v_perm_labels (the
rows of --permutations for the same seed), g2v_perm_sums (A = sums of q), g2v_dcx_sums on the pairs (g, g) (B = sums
of q^2), g2v_dcx_sums with the fused D epilogue, and g2v_dcx_tally.

For a labelling whose group has m samples: C = m P - A_i A_j, V_g = m B_g - A_g^2 (exact int64),
r = C / sqrt(V_i V_j) (0 when V_i or V_j is 0, clamped to [-1, 1]) and D = |r1 - r0| / (1 - r0 r1), which orders the
pairs as |atanh r1 - atanh r0| does.  The counts are integers, so P, P_maxT and Q depend only on the expression, the
labels, the pairs, the seed and B.
"""
from collections import namedtuple

import numpy as np

from . import perm

MAX_SAMPLES = 32768          # G2V_DCX_MAX_SAMPLES
MAX_PAIRS = 1 << 26          # G2V_DCX_MAX_PAIRS
MAX_PERMUTATIONS = 1 << 20   # the option's bound (G2V_DCX_MAX_ROWS rows per launch)
Q_BITS = 16                  # |q| <= 2^16
MIN_GROUP = 4                # Fisher's n - 3 in both groups

DiffCoexResult = namedtuple("DiffCoexResult", "pairs R_good R_poor Z D P P_maxT Q count count_maxt order n_perm")
DiffCoexResult.__doc__ = """diffcoex_test's result, every array over the pairs in their input order except `order`:
pairs   int32 [E, 2], (i, j) with i < j;
R_good, R_poor  the observed Pearson r over the label-0 and the label-1 samples;
Z       (atanh R_poor - atanh R_good) / sqrt(1/(n0-3) + 1/(n1-3)), +-inf at |R| = 1, 0 when R_good = R_poor;
D       the observed statistic |R_poor - R_good| / (1 - R_good R_poor), 0 when they are equal;
P       (1 + count) / (B + 1);
P_maxT  step-down maxT adjusted p-values, (1 + count_maxt) / (B + 1) made non-decreasing along the ranks;
Q       Benjamini-Hochberg q-values of P;
count   #{b : D_b >= D_obs};  count_maxt: #{b : max of D_b over the ranks >= this one's >= D_obs} (before the
        running max);
order   the pairs by D descending, ties by pair index (rank j -> pair order[j]);
n_perm  B."""


def pairs_from_edges(src, dst):
    """Directed edges (gene indices) -> the distinct unordered pairs as int32 [E, 2], (i, j) with i < j, sorted by
    (i, j): self-loops dropped, reversed and repeated edges collapsed."""
    s = np.asarray(src, dtype=np.int64).reshape(-1)
    d = np.asarray(dst, dtype=np.int64).reshape(-1)
    if s.shape != d.shape:
        raise ValueError("differential co-expression: src and dst must have the same length")
    keep = s != d
    a, b = np.minimum(s, d)[keep], np.maximum(s, d)[keep]
    key = np.unique((a << 32) | b)
    return np.stack([key >> 32, key & 0xFFFFFFFF], axis=1).astype(np.int32).reshape(-1, 2)


def check_inputs(expr, label, pairs, n_perm):
    """ValueError unless the test can run: at least 4 samples of each label 0 and 1 and at most 32768 of the two
    together, every expression value of those samples finite, 1 <= n_perm <= 2^20, and 1 to 2^26 pairs (i, j) of
    gene indices with i < j, sorted and distinct.  Returns (x, lab, pairs): the used samples' expression as float64
    [n, G], their labels and the pairs as int32 [E, 2].  Needs no GPU."""
    x = np.asarray(expr)
    lab = np.asarray(label).reshape(-1)
    if x.ndim != 2 or x.shape[0] != lab.shape[0]:
        raise ValueError("differential co-expression: expression must be [samples, genes] with one label per sample, "
                         "got %s and %d labels" % (x.shape, lab.shape[0]))
    G = x.shape[1]
    B = int(n_perm)
    if B != n_perm or not 1 <= B <= MAX_PERMUTATIONS:
        raise ValueError("differential co-expression: the number of permutations must be an integer in [1, %d], got %r"
                         % (MAX_PERMUTATIONS, n_perm))
    n0, n1 = int((lab == 0).sum()), int((lab == 1).sum())
    if n0 < MIN_GROUP or n1 < MIN_GROUP:
        raise ValueError("differential co-expression: needs at least %d samples of each label 0 and 1, got %d and %d"
                         % (MIN_GROUP, n0, n1))
    if n0 + n1 > MAX_SAMPLES:
        raise ValueError("differential co-expression: n = %d samples with label 0 or 1, must be at most %d"
                         % (n0 + n1, MAX_SAMPLES))
    p = np.asarray(pairs)
    if p.ndim != 2 or p.shape[1] != 2 or not np.issubdtype(p.dtype, np.integer):
        raise ValueError("differential co-expression: pairs must be an integer array [E, 2]")
    E = p.shape[0]
    if not 1 <= E <= MAX_PAIRS:
        raise ValueError("differential co-expression: %d gene pairs, must be in [1, %d]" % (E, MAX_PAIRS))
    p = p.astype(np.int64)
    if (p[:, 0] < 0).any() or (p[:, 1] >= G).any() or (p[:, 0] >= p[:, 1]).any():
        raise ValueError("differential co-expression: every pair must be (i, j) with 0 <= i < j < %d" % G)
    key = p[:, 0] * G + p[:, 1]
    if E > 1 and (np.diff(key) <= 0).any():
        raise ValueError("differential co-expression: the pairs must be distinct and sorted by (i, j)")
    used = (lab == 0) | (lab == 1)
    x = x[used].astype(np.float64)
    if not np.isfinite(x).all():
        raise ValueError("differential co-expression: expression values must be finite")
    return x, lab[used], p.astype(np.int32)


def corr_of(m, P, Ai, Aj, Bi, Bj):
    """r of a group of m samples from its exact sums (int64 arrays): C = m P - Ai Aj, V = m B - A^2,
    r = double(C) / sqrt(double(Vi) * double(Vj)) clamped to [-1, 1], 0 where Vi or Vj is 0 -- the bits of
    g2v_dcx_sums."""
    m = np.int64(m)
    C = m * np.asarray(P, np.int64) - np.asarray(Ai, np.int64) * np.asarray(Aj, np.int64)
    Vi = m * np.asarray(Bi, np.int64) - np.asarray(Ai, np.int64) ** 2
    Vj = m * np.asarray(Bj, np.int64) - np.asarray(Aj, np.int64) ** 2
    den = np.sqrt(Vi.astype(np.float64) * Vj.astype(np.float64))
    ok = (Vi != 0) & (Vj != 0)
    r = np.zeros(np.broadcast(C, den).shape)
    np.divide(C.astype(np.float64), den, out=r, where=ok)
    return np.clip(r, -1.0, 1.0)


def stat_of(r0, r1):
    """D = |r1 - r0| / (1 - r0 r1), 0 where r0 = r1 -- the bits of g2v_dcx_sums."""
    r0 = np.asarray(r0, np.float64); r1 = np.asarray(r1, np.float64)
    out = np.zeros(np.broadcast(r0, r1).shape)
    np.divide(np.abs(r1 - r0), 1.0 - r0 * r1, out=out, where=r0 != r1)
    return out


def z_of(r_good, r_poor, n0, n1):
    """Fisher's z contrast (atanh r_poor - atanh r_good) / sqrt(1/(n0-3) + 1/(n1-3)); 0 where r_good = r_poor."""
    r_good = np.asarray(r_good, np.float64); r_poor = np.asarray(r_poor, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        z = (np.arctanh(r_poor) - np.arctanh(r_good)) / np.sqrt(1.0 / (n0 - 3) + 1.0 / (n1 - 3))
    return np.where(r_good == r_poor, 0.0, z)


def prepare(expr, label, pairs, n_perm=1):
    """Host side up to the upload: a dict with n, n0, n1, k, sel (the selected label: the smaller group, label 1 on a
    tie), obs (u8 indicator of the selected group), q (int64 [n, G], |q| <= 2^16) and pairs."""
    x, lab, pairs = check_inputs(expr, label, pairs, n_perm)
    n0, n1 = int((lab == 0).sum()), int((lab == 1).sum())
    sel = 1 if n1 <= n0 else 0
    obs = (lab == sel).astype(np.uint8)
    return {"n": n0 + n1, "n0": n0, "n1": n1, "k": int(obs.sum()), "sel": sel, "obs": obs,
            "q": perm.quantise(x, bits=Q_BITS), "pairs": pairs}


def observed(prep, A2, B2, P2):
    """The observed statistics from the sums of the all-ones (row 0) and observed (row 1) labellings: A2, B2 [2, G]
    and P2 [2, E] int64.  Returns (R_good, R_poor, D_obs)."""
    n, k, pi, pj = prep["n"], prep["k"], prep["pairs"][:, 0], prep["pairs"][:, 1]
    r_sel = corr_of(k, P2[1], A2[1][pi], A2[1][pj], B2[1][pi], B2[1][pj])
    A_c, B_c, P_c = A2[0] - A2[1], B2[0] - B2[1], P2[0] - P2[1]
    r_oth = corr_of(n - k, P_c, A_c[pi], A_c[pj], B_c[pi], B_c[pj])
    r_good, r_poor = (r_oth, r_sel) if prep["sel"] == 1 else (r_sel, r_oth)
    return r_good, r_poor, stat_of(r_sel, r_oth)


def finish(prep, R_good, R_poor, D_obs, order, count_rank, count_maxt_rank, n_perm):
    """Counts in rank order -> DiffCoexResult."""
    B, E = int(n_perm), order.shape[0]
    count = np.empty(E, dtype=np.int64); count[order] = count_rank
    count_maxt = np.empty(E, dtype=np.int64); count_maxt[order] = count_maxt_rank
    P = (1.0 + count) / (B + 1.0)
    pm = np.empty(E); pm[order] = np.maximum.accumulate((1.0 + np.asarray(count_maxt_rank)) / (B + 1.0))
    return DiffCoexResult(pairs=prep["pairs"], R_good=R_good, R_poor=R_poor,
                          Z=z_of(R_good, R_poor, prep["n0"], prep["n1"]), D=D_obs, P=P, P_maxT=pm, Q=perm.bh(P),
                          count=count, count_maxt=count_maxt, order=order, n_perm=B)


def chunk_rows(S_pad, G, E, n_perm, max_chunk_bytes):
    """Permutations per chunk: M (S_pad bytes), A and B (8 G bytes each) and D (8 E bytes) of every row within
    max_chunk_bytes, at least 1."""
    return int(max(1, min(int(n_perm), int(max_chunk_bytes) // (S_pad + 16 * G + 8 * E))))


def diffcoex_test(expr, label, pairs, n_perm, seed=0, max_chunk_bytes=None):
    """Label-permutation test of differential co-expression of every gene pair on the GPU (Pearson r).

    expr: host float array [samples, genes]; label: one int per sample (0 good, 1 poor; other labels are left out);
    pairs: int [E, 2], (i, j) with i < j, sorted and distinct (pairs_from_edges makes them from a network).
    n_perm: B, 1 <= B <= 2^20 permutations (the observed labelling is not among them), the rows perm.perm_test uses for
    the same seed; seed: the Philox key (--seed).  max_chunk_bytes: bound on the device memory of one chunk's rows,
    sums and D (default: half the free device memory).  Makes 3 launches, then 5 per chunk.  Returns a
    DiffCoexResult; ValueError (before anything is uploaded) on inputs check_inputs refuses."""
    prep = prepare(expr, label, pairs, n_perm)
    import torch
    from . import _capi
    lib = _capi.load()
    if not torch.cuda.is_available():
        raise RuntimeError("g2vec_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    dev = torch.device("cuda", torch.cuda.current_device())
    n, k, B, q = prep["n"], prep["k"], int(n_perm), prep["q"]
    G, E = q.shape[1], prep["pairs"].shape[0]
    S_pad = -(-n // 32) * 32
    qt = np.zeros((G, S_pad), dtype=np.int32)
    qt[:, :n] = q.T
    pl = perm.planes(q, np.arange(G))
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    q_d, pl_d = up(qt), up(pl)
    diag_d = up(np.arange(G, dtype=np.int32))
    pi_d, pj_d = up(prep["pairs"][:, 0]), up(prep["pairs"][:, 1])
    M2 = np.zeros((2, S_pad), dtype=np.uint8)
    M2[0, :n] = 1
    M2[1, :n] = prep["obs"]
    M2_d = up(M2)
    A2 = torch.empty((2, G), dtype=torch.int64, device=dev)
    B2 = torch.empty((2, G), dtype=torch.int64, device=dev)
    P2 = torch.empty((2, E), dtype=torch.int64, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    raw = lambda M, nb, gi, gj, ne, out, what: _capi.check(lib.g2v_dcx_sums(
        M, nb, S_pad, q_d.data_ptr(), G, gi, gj, ne, 0, 0, None, None, None, None, None, out, None, st), what)
    _capi.check(lib.g2v_perm_sums(M2_d.data_ptr(), pl_d.data_ptr(), 2, S_pad, G, A2.data_ptr(), st), "g2v_perm_sums")
    raw(M2_d.data_ptr(), 2, diag_d.data_ptr(), diag_d.data_ptr(), G, B2.data_ptr(), "g2v_dcx_sums")
    raw(M2_d.data_ptr(), 2, pi_d.data_ptr(), pj_d.data_ptr(), E, P2.data_ptr(), "g2v_dcx_sums")
    A2h, B2h, P2h = A2.cpu().numpy(), B2.cpu().numpy(), P2.cpu().numpy()
    R_good, R_poor, D_obs = observed(prep, A2h, B2h, P2h)
    order = np.argsort(-D_obs, kind="stable")
    # the permutations run over the pairs in rank order, so the tally reads every row of D front to back
    ri_d, rj_d = up(prep["pairs"][order, 0]), up(prep["pairs"][order, 1])
    Pt_d, Dobs_d = up(P2h[0][order]), up(D_obs[order])
    At_d, Bt_d = A2[0].contiguous(), B2[0].contiguous()
    obs_d = up(prep["obs"])
    cnt = torch.zeros(E, dtype=torch.int64, device=dev)
    cmax = torch.zeros(E, dtype=torch.int64, device=dev)
    if max_chunk_bytes is None:
        max_chunk_bytes = torch.cuda.mem_get_info(dev)[0] // 2
    rows = chunk_rows(S_pad, G, E, B, max_chunk_bytes)
    M = torch.empty((rows, S_pad), dtype=torch.uint8, device=dev)
    A = torch.empty((rows, G), dtype=torch.int64, device=dev)
    Bq = torch.empty((rows, G), dtype=torch.int64, device=dev)
    D = torch.empty((rows, E), dtype=torch.float64, device=dev)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    for b0 in range(0, B, rows):
        nb = min(rows, B - b0)
        _capi.check(lib.g2v_perm_labels(obs_d.data_ptr(), n, S_pad, seed, b0, nb, M.data_ptr(), st), "g2v_perm_labels")
        _capi.check(lib.g2v_perm_sums(M.data_ptr(), pl_d.data_ptr(), nb, S_pad, G, A.data_ptr(), st), "g2v_perm_sums")
        raw(M.data_ptr(), nb, diag_d.data_ptr(), diag_d.data_ptr(), G, Bq.data_ptr(), "g2v_dcx_sums")
        _capi.check(lib.g2v_dcx_sums(M.data_ptr(), nb, S_pad, q_d.data_ptr(), G, ri_d.data_ptr(), rj_d.data_ptr(), E, n,
                                     k, A.data_ptr(), Bq.data_ptr(), At_d.data_ptr(), Bt_d.data_ptr(), Pt_d.data_ptr(),
                                     None, D.data_ptr(), st), "g2v_dcx_sums")
        _capi.check(lib.g2v_dcx_tally(D.data_ptr(), nb, E, Dobs_d.data_ptr(), cnt.data_ptr(), cmax.data_ptr(), st),
                    "g2v_dcx_tally")
    return finish(prep, R_good, R_poor, D_obs, order, cnt.cpu().numpy(), cmax.cpu().numpy(), B)


def graph_pairs(pairs, G, rowptr, col):
    """uint8 [E]: 1 where the pair (i, j) is an edge of the CSR graph (rowptr [G+1], col) in either direction."""
    rp = np.asarray(rowptr, dtype=np.int64)
    c = np.asarray(col, dtype=np.int64)
    s = np.repeat(np.arange(G, dtype=np.int64), np.diff(rp))
    key = np.minimum(s, c) * G + np.maximum(s, c)
    pk = pairs[:, 0].astype(np.int64) * G + pairs[:, 1]
    pos = np.searchsorted(pk, key)
    hit = pos < pk.shape[0]
    hit[hit] = pk[pos[hit]] == key[hit]
    out = np.zeros(pk.shape[0], dtype=np.uint8)
    out[pos[hit]] = 1
    return out


def summary(res, in_good, in_poor, biomarkers):
    """The command line's line: in_good, in_poor (0/1) and biomarkers (0..2) per pair; the last two counts are over
    the pairs with Q <= 0.05."""
    sq = res.Q <= 0.05
    one = sq & (np.asarray(in_good) != np.asarray(in_poor))
    touch = sq & (np.asarray(biomarkers) > 0)
    return ("differential co-expression: %d label permutations of %d gene pairs: %d with Q <= 0.05, %d with "
            "P_maxT <= 0.05; %d of them in one group's graph only, %d touching a biomarker"
            % (res.n_perm, res.pairs.shape[0], int(sq.sum()), int((res.P_maxT <= 0.05).sum()), int(one.sum()),
               int(touch.sum())))
