"""Label-permutation p-values of the gene t statistics (DESIGN.md §4.24): per gene a raw permutation p-value, the
Westfall & Young step-down maxT adjusted p-value (Ge, Dudoit & Speed 2003, as multtest's mt.maxT) and Benjamini &
Hochberg q-values.

Host side (NumPy, float64): the samples with label 0 or 1 (n of them, n0 + n1), the selected group (the smaller one,
label 1 on a tie; k samples), each gene quantised to integers q with |q| <= 2^22, and the observed statistics.
Device side (csrc/g2v_perm.cu): per chunk of permutations one launch each of g2v_perm_labels (the permuted
indicators), g2v_perm_sums (A = M . q on the INT8 tensor cores) and g2v_perm_tally (the integer counts).

For a permutation and a gene, N = n A - k Q_g with A the sum of q over the selected samples and Q_g the sum over all,
W_g = n0 n1 (n sum q^2 - Q_g^2) and rho = N^2 / W_g, the squared point-biserial correlation; the pooled two-sample t of
cli.tscore satisfies t^2 = (n-2) rho / (1-rho).  The per-gene test compares |N| exactly, maxT compares rho across
genes.  The counts are integers, so P, P_maxT and Q depend only on the expression, the labels, the seed and B.
"""
from collections import namedtuple

import numpy as np

MAX_SAMPLES = 32768          # G2V_PERM_MAX_SAMPLES
MAX_PERMUTATIONS = 1 << 24   # G2V_PERM_MAX_PERMUTATIONS
Q_BITS = 22                  # |q| <= 2^22

PermResult = namedtuple("PermResult", "T P P_maxT Q count count_maxt order n_perm")
PermResult.__doc__ = """perm_test's result, every array over the genes in their input order except `order`:
T       the observed |t| = sqrt((n-2) rho / (1-rho)), inf at perfect separation (rho = 1);
P       (1 + count) / (B + 1);
P_maxT  step-down maxT adjusted p-values, (1 + count_maxt) / (B + 1) made non-decreasing along the ranks;
Q       Benjamini-Hochberg q-values of P;
count   #{b : |N_b| >= |N_obs|};  count_maxt: #{b : u_b >= rho_obs} at the gene's rank (before the running max);
order   the genes by observed rho descending, ties by index ascending (rank j -> gene order[j]);
n_perm  B."""


def check_inputs(expr, label, n_perm):
    """ValueError unless the permutation test can run: labels 0 and 1 both present, 3 <= n <= 32768 samples with
    label 0 or 1, 1 <= n_perm <= 2^24, and every expression value of those samples finite.  Returns (x, lab): the
    used samples' expression as float64 [n, G] and their labels.  Needs no GPU."""
    x = np.asarray(expr)
    lab = np.asarray(label).reshape(-1)
    if x.ndim != 2 or x.shape[0] != lab.shape[0]:
        raise ValueError("permutation test: expression must be [samples, genes] with one label per sample, got %s "
                         "and %d labels" % (x.shape, lab.shape[0]))
    if x.shape[1] < 1:
        raise ValueError("permutation test: no genes")
    B = int(n_perm)
    if B != n_perm or not 1 <= B <= MAX_PERMUTATIONS:
        raise ValueError("permutation test: the number of permutations must be an integer in [1, %d], got %r"
                         % (MAX_PERMUTATIONS, n_perm))
    used = (lab == 0) | (lab == 1)
    n0, n1 = int((lab == 0).sum()), int((lab == 1).sum())
    if n0 == 0 or n1 == 0:
        raise ValueError("permutation test: needs samples of both labels 0 and 1, got %d and %d" % (n0, n1))
    n = n0 + n1
    if not 3 <= n <= MAX_SAMPLES:
        raise ValueError("permutation test: n = %d samples with label 0 or 1, must be in [3, %d]" % (n, MAX_SAMPLES))
    x = x[used].astype(np.float64)
    if not np.isfinite(x).all():
        raise ValueError("permutation test: expression values must be finite")
    return x, lab[used]


def quantise(x, bits=Q_BITS):
    """float64 [n, G] -> int64 q [n, G]: per gene c = the mean, m = max |x - c|; q = 0 if m = 0, else
    q = rint((x - c) 2^e) with e = bits - 1 - floor(log2 m), so 2^(bits-1) <= max |q| <= 2^bits (bits = 22: the
    permutation test's e = 21 - floor(log2 m)).  Invariant to scaling a gene by a power of two (the scaling is exact)
    and, where x - c is exact, to shifting it."""
    x = np.asarray(x, dtype=np.float64)
    d = x - x.mean(axis=0)
    m = np.abs(d).max(axis=0) if x.shape[0] else np.zeros(x.shape[1])
    q = np.zeros(x.shape, dtype=np.int64)
    nz = m > 0
    _, ex = np.frexp(m[nz])                             # m = f 2^ex, 0.5 <= f < 1: floor(log2 m) = ex - 1
    e = int(bits) - ex.astype(np.int64)                 # up to 1096: scale in two exact power-of-two steps
    h = e // 2
    q[:, nz] = np.rint(d[:, nz] * np.ldexp(1.0, h) * np.ldexp(1.0, e - h))
    return q


def rho_of(N, W):
    """rho = (double) N * (double) N / W, 0 where W = 0 -- the bits g2v_perm_tally computes."""
    Nd = np.asarray(N).astype(np.float64)
    W = np.asarray(W, dtype=np.float64)
    out = np.zeros(np.broadcast(Nd, W).shape)
    np.divide(Nd * Nd, W, out=out, where=np.broadcast_to(W > 0, out.shape))
    return out


def t_of(rho, n):
    """|t| of the pooled two-sample t from rho: sqrt((n-2) rho / (1-rho)), inf where rho >= 1."""
    rho = np.asarray(rho, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.sqrt((n - 2) * rho / (1.0 - rho))
    return np.where(rho >= 1.0, np.inf, t)


def prepare(expr, label, n_perm=1):
    """Host side of perm_test up to the upload: a dict with n, n0, n1, k, obs (u8 indicator of the selected group
    over the n used samples), q, Q, W, N_obs, rho_obs and order (rank -> gene)."""
    x, lab = check_inputs(expr, label, n_perm)
    n = x.shape[0]
    n0, n1 = int((lab == 0).sum()), int((lab == 1).sum())
    sel = 1 if n1 <= n0 else 0
    obs = (lab == sel).astype(np.uint8)
    k = int(obs.sum())
    q = quantise(x)
    Q = q.sum(axis=0)
    SS = (q * q).sum(axis=0)
    W = np.array([float(n0 * n1 * (n * int(s) - int(t) * int(t))) for s, t in zip(SS, Q)], dtype=np.float64)
    N_obs = n * q[obs == 1].sum(axis=0) - k * Q
    rho_obs = rho_of(N_obs, W)
    order = np.argsort(-rho_obs, kind="stable")
    return {"n": n, "n0": n0, "n1": n1, "k": k, "obs": obs, "q": q, "Q": Q, "W": W, "N_obs": N_obs,
            "rho_obs": rho_obs, "order": order}


def planes(q, order):
    """q [n, G] -> the three byte planes of g2v_perm_sums, uint8 [3, G, S_pad] (h as its s8 bytes), genes in
    `order`, each gene's samples contiguous, zero padding up to S_pad = n rounded up to 32."""
    n, G = q.shape
    S_pad = -(-n // 32) * 32
    qt = np.zeros((G, S_pad), dtype=np.int32)          # |q| <= 2^22
    qt[:, :n] = q[:, order].T
    out = np.empty((3, G, S_pad), dtype=np.uint8)
    out[0] = (qt >> 16).astype(np.int8).view(np.uint8)
    out[1] = ((qt >> 8) & 255).astype(np.uint8)
    out[2] = (qt & 255).astype(np.uint8)
    return out


def bh(p):
    """Benjamini-Hochberg q-values: min over j >= i of m p_(j) / j along the ascending p, capped at 1."""
    p = np.asarray(p, dtype=np.float64)
    m = p.shape[0]
    o = np.argsort(p, kind="stable")
    r = np.minimum.accumulate((p[o] * m / np.arange(1, m + 1))[::-1])[::-1]
    out = np.empty(m)
    out[o] = np.minimum(r, 1.0)
    return out


def finish(prep, count_rank, count_maxt_rank, n_perm):
    """Counts in rank order -> PermResult."""
    order, B = prep["order"], int(n_perm)
    G = order.shape[0]
    count = np.empty(G, dtype=np.int64); count[order] = count_rank
    count_maxt = np.empty(G, dtype=np.int64); count_maxt[order] = count_maxt_rank
    P = (1.0 + count) / (B + 1.0)
    pm = np.empty(G); pm[order] = np.maximum.accumulate((1.0 + np.asarray(count_maxt_rank)) / (B + 1.0))
    return PermResult(T=t_of(prep["rho_obs"], prep["n"]), P=P, P_maxT=pm, Q=bh(P), count=count,
                      count_maxt=count_maxt, order=order, n_perm=B)


def chunk_rows(S_pad, G, n_perm, max_chunk_bytes):
    """Permutations per chunk: M (S_pad bytes) and A (8 G bytes) of every row within max_chunk_bytes, at least 1."""
    return int(max(1, min(int(n_perm), int(max_chunk_bytes) // (S_pad + 8 * G))))


def perm_test(expr, label, n_perm, seed=0, max_chunk_bytes=None):
    """Label-permutation test of every gene's t statistic on the GPU.

    expr: host float array [samples, genes]; label: one int per sample (0 good, 1 poor; other labels are left out).
    n_perm: B, 1 <= B <= 2^24 permutations (the observed labelling is not among them); seed: the Philox key (--seed).
    max_chunk_bytes: bound on the device memory of one chunk's indicator rows and sums (default: half the free device
    memory).  Makes 3 launches per chunk.  Returns a PermResult; ValueError (before anything is uploaded) on inputs
    check_inputs refuses."""
    prep = prepare(expr, label, n_perm)
    import torch
    from . import _capi
    lib = _capi.load()
    if not torch.cuda.is_available():
        raise RuntimeError("g2vec_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    dev = torch.device("cuda", torch.cuda.current_device())
    n, k, order, B = prep["n"], prep["k"], prep["order"], int(n_perm)
    G = order.shape[0]
    pl = planes(prep["q"], order)
    S_pad = pl.shape[2]
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    obs_d, pl_d = up(prep["obs"]), up(pl)
    Q_d, W_d = up(prep["Q"][order]), up(prep["W"][order])
    absN_d, rho_d = up(np.abs(prep["N_obs"][order])), up(prep["rho_obs"][order])
    cnt = torch.zeros(G, dtype=torch.int64, device=dev)
    cmax = torch.zeros(G, dtype=torch.int64, device=dev)
    if max_chunk_bytes is None:
        max_chunk_bytes = torch.cuda.mem_get_info(dev)[0] // 2
    rows = chunk_rows(S_pad, G, B, max_chunk_bytes)
    M = torch.empty((rows, S_pad), dtype=torch.uint8, device=dev)
    A = torch.empty((rows, G), dtype=torch.int64, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    for b0 in range(0, B, rows):
        nb = min(rows, B - b0)
        _capi.check(lib.g2v_perm_labels(obs_d.data_ptr(), n, S_pad, seed, b0, nb, M.data_ptr(), st), "g2v_perm_labels")
        _capi.check(lib.g2v_perm_sums(M.data_ptr(), pl_d.data_ptr(), nb, S_pad, G, A.data_ptr(), st), "g2v_perm_sums")
        _capi.check(lib.g2v_perm_tally(A.data_ptr(), nb, G, n, k, Q_d.data_ptr(), W_d.data_ptr(), absN_d.data_ptr(),
                                       rho_d.data_ptr(), cnt.data_ptr(), cmax.data_ptr(), st), "g2v_perm_tally")
    return finish(prep, cnt.cpu().numpy(), cmax.cpu().numpy(), B)
