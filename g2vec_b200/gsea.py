"""Phenotype-permutation gene-set enrichment of the good / poor contrast (DESIGN.md §4.28): GSEA as Subramanian et al.
(PNAS 2005) with label permutations, its normalised enrichment score NES, nominal P, FDR q and FWER p per gene set.

The ranking metric is the signed point-biserial correlation r of each gene's quantised expression with the
poor-prognosis indicator (label 1), GSEA's "Pearson" metric for a 0/1 phenotype, from the exact sums of the permutation
test (perm.py, DESIGN.md §4.24): r = (s N) / sqrt(W), quantised to rq = rint(r 2^32), weight u = |rq| (GSEA's p = 1).
Host side (NumPy): perm's checks, quantisation and byte planes (genes in their input order), the GMT file, the sets'
CSR and the final P, FDR and FWER from integer counts.  Device side (csrc/g2v_gsea.cu, csrc/g2v_perm.cu): per chunk of
permutations g2v_perm_labels, g2v_perm_sums, g2v_gsea_keys, g2v_gsea_rank and g2v_gsea_es; then g2v_gsea_norm and the
FDR / FWER counts (torch.sort and searchsorted on the device).  The permutations are those of perm_test for the same
seed and B.  Every count is an integer, so P, FDR and FWER depend only on the expression, the labels, the sets, the
seed and B.
"""
from collections import namedtuple

import numpy as np

from . import perm

MAX_GENES = 1 << 20          # G2V_GSEA_MAX_GENES: the gene index fits the low 20 bits of a sort key
MAX_PERMUTATIONS = 1 << 20   # G2V_GSEA_MAX_PERMUTATIONS
MAX_ES = 1 << 28             # G2V_GSEA_MAX_ES: B * S
MAX_SET_SIZE = 4096          # G2V_GSEA_MAX_SET_SIZE
MAX_ROWS = 65535             # G2V_GSEA_MAX_ROWS: permutations per chunk
Q_SCALE = 2.0 ** 32
FDR_CUTOFF = 0.25            # GSEA's default significance line

GseaResult = namedtuple("GseaResult", "name size members ES NES P FDR FWER leading_edge count_pos count_neg "
                                      "count_extreme count_null count_null_side count_obs count_obs_side count_fwer "
                                      "mean_pos mean_neg n_perm")
GseaResult.__doc__ = """gsea's result, one entry per kept set in input order:
name, size    the set's name and k, its number of genes in the analysis; members: their gene indices, ascending;
ES, NES       the observed enrichment score and NES = ES / mean+ (ES >= 0) or ES / mean-, NaN when that side of the
              null is empty (the set is then left out of every FDR and FWER count);
P             (1 + count_extreme) / (1 + count_pos) for ES >= 0, (1 + count_extreme) / (1 + count_neg) for ES < 0;
              1 where NES is NaN;
FDR           min(1, (count_null / count_null_side) / (count_obs / count_obs_side)), NaN where NES is NaN;
FWER          (1 + count_fwer) / (B + 1), NaN where NES is NaN;
leading_edge  the members at or before the first hit attaining D+ (ES >= 0), or at or after the first hit attaining
              D- (ES < 0), in rank order of the observed ranking; empty when ES = 0;
count_pos, count_neg   #{b: ES_b >= 0}, #{b: ES_b < 0};  count_extreme: #{b: ES_b >= ES} or #{b: ES_b <= ES};
count_null    #{(b, s'): NES_b,s' >= NES} (NES >= 0) or <= NES, over the sets whose NES is not NaN (all counts
              from here on are 0 for a set whose NES is NaN);
count_null_side  #{(b, s'): NES_b,s' >= 0} or < 0 over those sets;  count_obs, count_obs_side: the same over the
              observed NES_s';  count_fwer: #{b: the max over s' of the NES_b,s' >= 0 is >= NES} (the min of the
              NES_b,s' < 0 is <= NES for NES < 0);
mean_pos, mean_neg   mean+ and mean-;  n_perm: B."""


# ----------------------------------------------------------------------------------------------------------- GMT
def read_gmt(path):
    """GMT file -> [(name, description, genes)] in file order.  Each non-blank line is split on tabs into the name,
    the description and the genes; empty gene fields are ignored and a gene listed twice in a set counts once (first
    position kept).  ValueError on a line with fewer than 2 fields or a set name seen before."""
    sets, seen = [], {}
    with open(path) as f:
        for no, line in enumerate(f, 1):
            line = line.rstrip("\r\n")
            if not line.strip():
                continue
            fields = line.split("\t")
            if len(fields) < 2:
                raise ValueError("%s line %d: a gene set needs a name and a description separated by a tab, got %r"
                                 % (path, no, line[:80]))
            name = fields[0]
            if name in seen:
                raise ValueError("%s line %d: gene set %r is also on line %d" % (path, no, name, seen[name]))
            seen[name] = no
            genes = list(dict.fromkeys(g for g in fields[2:] if g))
            sets.append((name, fields[1], genes))
    return sets


def restrict_sets(sets, genes, min_size, max_size):
    """Keep the genes of each set that are in `genes` (the analysis' genes, in column order) and the sets with
    min_size <= k <= max_size and k < G.  sets: (name, ..., members) tuples, the members given as elements of
    `genes`.  Returns (set_ptr int32 [S + 1], set_gene int32 [nnz], names): the kept sets' gene indices ascending,
    CSR in input order."""
    index = {g: i for i, g in enumerate(genes)}
    G = len(index)
    ptr, idx, names = [0], [], []
    for entry in sets:
        m = sorted({index[g] for g in entry[-1] if g in index})
        if min_size <= len(m) <= max_size and len(m) < G:
            idx.extend(m)
            ptr.append(len(idx))
            names.append(entry[0])
    return np.array(ptr, dtype=np.int32), np.array(idx, dtype=np.int32), names


def check_inputs(expr, label, n_perm, n_sets, min_size, max_size):
    """ValueError unless the gene-set test can run: perm.check_inputs' conditions, 1 <= n_perm <= 2^20, at most 2^20
    genes, at least one set kept, n_perm * n_sets <= 2^28 and 1 <= min_size <= max_size <= 4096.  Returns (x, lab)
    as perm.check_inputs.  Needs no GPU."""
    if not (int(min_size) == min_size and int(max_size) == max_size and 1 <= min_size <= max_size <= MAX_SET_SIZE):
        raise ValueError("gene-set test: set sizes MIN,MAX must be integers with 1 <= MIN <= MAX <= %d, got %r,%r"
                         % (MAX_SET_SIZE, min_size, max_size))
    B = int(n_perm)
    if B != n_perm or not 1 <= B <= MAX_PERMUTATIONS:
        raise ValueError("gene-set test: the number of permutations must be an integer in [1, %d], got %r"
                         % (MAX_PERMUTATIONS, n_perm))
    x, lab = perm.check_inputs(expr, label, B)
    if x.shape[1] > MAX_GENES:
        raise ValueError("gene-set test: %d genes, at most %d" % (x.shape[1], MAX_GENES))
    if n_sets < 1:
        raise ValueError("gene-set test: no gene set has %d to %d genes in the analysis" % (min_size, max_size))
    if B * int(n_sets) > MAX_ES:
        raise ValueError("gene-set test: %d permutations x %d sets exceeds 2^28" % (B, n_sets))
    return x, lab


# ------------------------------------------------------------------------------------------------ host arithmetic
def sign_of(prep):
    """s = +1 if perm.prepare selected label 1, -1 if it selected label 0 (the smaller group)."""
    return 1 if prep["n1"] <= prep["n0"] else -1


def leading_edge(pos, u, members, G):
    """Leading-edge members (gene indices, rank order) of one set in one ranking: pos [G] ranks, u [G] weights."""
    members = np.asarray(members, dtype=np.int64)
    o = np.argsort(pos[members], kind="stable")
    m_sorted = members[o]
    p = pos[m_sorted].astype(np.int64)
    w = u[m_sorted].astype(np.uint64)
    k = len(m_sorted)
    S = np.cumsum(w)
    NR = int(S[-1]) if k else 0
    if NR == 0:
        return m_sorted[:0]
    m = (p - np.arange(k)).astype(np.float64) / float(G - k)
    tp = S.astype(np.float64) / float(NR) - m
    tm = (S - w).astype(np.float64) / float(NR) - m
    dp, dm = max(0.0, float(tp.max())), min(0.0, float(tm.min()))
    if dp >= -dm:
        if dp == 0.0:
            return m_sorted[:0]
        return m_sorted[:int(np.argmax(tp == dp)) + 1]
    return m_sorted[int(np.argmax(tm == dm)):]


def finish(names, set_ptr, set_gene, es_obs, nes_obs, counts, null_counts, mean_pos, mean_neg, n_perm):
    """Counts -> GseaResult.  counts [3, S] from g2v_gsea_norm; null_counts: (count_null, count_null_side,
    count_fwer) per set."""
    B = int(n_perm)
    ES, NES = np.asarray(es_obs, np.float64), np.asarray(nes_obs, np.float64)
    S = ES.shape[0]
    cpos, cneg, cext = (np.asarray(c, np.int64) for c in counts)
    valid = ~np.isnan(NES)
    up = ES >= 0
    P = np.where(up, (1.0 + cext) / (1.0 + cpos), (1.0 + cext) / (1.0 + cneg))
    P[~valid] = 1.0
    nv = NES[valid]
    obs = np.zeros(S, np.int64); obs_side = np.zeros(S, np.int64)
    pos_sorted, neg_sorted = np.sort(nv[nv >= 0]), np.sort(nv[nv < 0])
    obs[valid & up] = len(pos_sorted) - np.searchsorted(pos_sorted, NES[valid & up], side="left")
    obs[valid & ~up] = np.searchsorted(neg_sorted, NES[valid & ~up], side="right")
    obs_side[valid & up] = len(pos_sorted)
    obs_side[valid & ~up] = len(neg_sorted)
    cnull, cside, cfw = (np.where(valid, np.asarray(c, np.int64), 0) for c in null_counts)
    with np.errstate(divide="ignore", invalid="ignore"):
        FDR = np.minimum(1.0, (cnull / cside.astype(np.float64)) / (obs / obs_side.astype(np.float64)))
    FWER = (1.0 + cfw) / (B + 1.0)
    FDR[~valid] = np.nan
    FWER[~valid] = np.nan
    ptr = np.asarray(set_ptr)
    members = [np.asarray(set_gene[ptr[i]:ptr[i + 1]]) for i in range(S)]
    return GseaResult(name=list(names), size=np.diff(ptr).astype(np.int64), members=members, ES=ES, NES=NES, P=P,
                      FDR=FDR, FWER=FWER, leading_edge=None, count_pos=cpos, count_neg=cneg, count_extreme=cext,
                      count_null=cnull, count_null_side=cside, count_obs=obs, count_obs_side=obs_side,
                      count_fwer=cfw, mean_pos=np.asarray(mean_pos, np.float64),
                      mean_neg=np.asarray(mean_neg, np.float64), n_perm=B)


def summary(res):
    """The gene-set test line of the command line."""
    sig = np.nan_to_num(res.FDR, nan=2.0) <= FDR_CUTOFF
    return ("gene-set test: %d label permutations: %d of %d sets with FDR q <= %g (%d up in poor, %d up in good)"
            % (res.n_perm, int(sig.sum()), len(res.name), FDR_CUTOFF, int((sig & (res.NES > 0)).sum()),
               int((sig & (res.NES < 0)).sum())))


# ---------------------------------------------------------------------------------------------------------- device
def chunk_rows(S_pad, G, n_sets, n_perm, max_chunk_bytes):
    """Permutations per chunk: M (S_pad bytes), A, key, sorted key and u (8 G bytes each), pos (4 G bytes) and the
    CUB scratch (about 8 G bytes) of a row within max_chunk_bytes, at least 1, at most 65535 and n_b * G < 2^31."""
    per_row = S_pad + 44 * G
    rows = min(int(n_perm), int(max_chunk_bytes) // per_row, MAX_ROWS, (2 ** 31 - 1) // G)
    return int(max(1, rows))


def null_counts(nes, nes_obs):
    """The FDR and FWER counts on the device: nes [B, S] (NaN columns for the sets left out), nes_obs [S] (both torch
    float64 on the GPU) -> (count_null, count_null_side, count_fwer) as int64 torch tensors [S]."""
    import torch
    up = nes_obs >= 0
    pos_sorted = torch.sort(nes[nes >= 0]).values
    neg_sorted = torch.sort(nes[nes < 0]).values
    n_pos, n_neg = pos_sorted.numel(), neg_sorted.numel()
    cnt = torch.where(up, n_pos - torch.searchsorted(pos_sorted, nes_obs, right=False),
                      torch.searchsorted(neg_sorted, nes_obs, right=True))
    side = torch.where(up, torch.full_like(cnt, n_pos), torch.full_like(cnt, n_neg))
    inf = torch.tensor(float("inf"), dtype=torch.float64, device=nes.device)
    row_max = torch.sort(torch.where(nes >= 0, nes, -inf).amax(dim=1)).values
    row_min = torch.sort(torch.where(nes < 0, nes, inf).amin(dim=1)).values
    B = nes.shape[0]
    fw = torch.where(up, B - torch.searchsorted(row_max, nes_obs, right=False),
                     torch.searchsorted(row_min, nes_obs, right=True))
    return cnt, side, fw


def gsea(expr, label, sets, n_perm, seed=0, min_size=15, max_size=500, max_chunk_bytes=None, genes=None):
    """Phenotype-permutation GSEA of the good / poor contrast on the GPU.

    expr: host float array [samples, genes]; label: one int per sample (0 good, 1 poor; other labels are left out).
    sets: (name, ..., members) tuples in the order they are reported, e.g. read_gmt's; the members are elements of
    `genes` (default: the column indices 0 .. G-1), others are ignored.  Sets with min_size <= k <= max_size genes in
    the analysis (and k < G) are kept.  n_perm: B, 1 <= B <= 2^20 label permutations, those of perm_test for the same
    seed (the observed labelling is not among them).  max_chunk_bytes: bound on the device memory of one chunk's
    per-permutation buffers (default: half the free device memory).  Returns a GseaResult; ValueError (before anything
    is uploaded) on inputs check_inputs refuses, RuntimeError without a GPU."""
    x = np.asarray(expr)
    G = x.shape[1] if x.ndim == 2 else 0
    set_ptr, set_gene, names = restrict_sets(sets, range(G) if genes is None else genes, min_size, max_size)
    check_inputs(expr, label, n_perm, len(names), min_size, max_size)
    prep = perm.prepare(expr, label, n_perm)
    import torch
    from . import _capi
    lib = _capi.load()
    if not torch.cuda.is_available():
        raise RuntimeError("g2vec_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    dev = torch.device("cuda", torch.cuda.current_device())
    n, k, B, S = prep["n"], prep["k"], int(n_perm), len(names)
    s = sign_of(prep)
    pl = perm.planes(prep["q"], np.arange(G))
    S_pad = pl.shape[2]
    max_k = int(np.diff(set_ptr).max())
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    obs_d, pl_d, Q_d, W_d = up(prep["obs"]), up(pl), up(prep["Q"]), up(prep["W"])
    ptr_d, gene_d = up(set_ptr), up(set_gene)
    if max_chunk_bytes is None:
        max_chunk_bytes = torch.cuda.mem_get_info(dev)[0] // 2
    rows = chunk_rows(S_pad, G, S, B, max_chunk_bytes)
    M = torch.zeros((rows, S_pad), dtype=torch.uint8, device=dev)
    A = torch.empty((rows, G), dtype=torch.int64, device=dev)
    key = torch.empty((rows, G), dtype=torch.int64, device=dev)
    u = torch.empty((rows, G), dtype=torch.int64, device=dev)
    pos = torch.empty((rows, G), dtype=torch.int32, device=dev)
    ws_bytes = int(lib.g2v_gsea_rank_workspace_bytes(rows, G))
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    es = torch.empty((B, S), dtype=torch.float64, device=dev)
    es_obs = torch.empty(S, dtype=torch.float64, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream

    def rank_rows(nb, es_out):
        _capi.check(lib.g2v_perm_sums(M.data_ptr(), pl_d.data_ptr(), nb, S_pad, G, A.data_ptr(), st), "g2v_perm_sums")
        _capi.check(lib.g2v_gsea_keys(A.data_ptr(), nb, G, n, k, s, Q_d.data_ptr(), W_d.data_ptr(), key.data_ptr(),
                                      u.data_ptr(), st), "g2v_gsea_keys")
        _capi.check(lib.g2v_gsea_rank(key.data_ptr(), nb, G, pos.data_ptr(), ws.data_ptr(), ws_bytes, st),
                    "g2v_gsea_rank")
        _capi.check(lib.g2v_gsea_es(pos.data_ptr(), u.data_ptr(), nb, G, ptr_d.data_ptr(), gene_d.data_ptr(), S, max_k,
                                    es_out, st), "g2v_gsea_es")

    M[0, :n] = obs_d                                   # the observed labelling first, as row 0 of a one-row chunk
    rank_rows(1, es_obs.data_ptr())
    pos_obs, u_obs = pos[0].cpu().numpy(), u[0].cpu().numpy()
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    for b0 in range(0, B, rows):
        nb = min(rows, B - b0)
        _capi.check(lib.g2v_perm_labels(obs_d.data_ptr(), n, S_pad, seed, b0, nb, M.data_ptr(), st), "g2v_perm_labels")
        rank_rows(nb, es[b0:].data_ptr())
    del M, A, key, u, pos, ws
    nes = torch.empty((B, S), dtype=torch.float64, device=dev)
    mp, mn, nes_obs = (torch.empty(S, dtype=torch.float64, device=dev) for _ in range(3))
    counts = torch.empty((3, S), dtype=torch.int64, device=dev)
    _capi.check(lib.g2v_gsea_norm(es.data_ptr(), B, S, es_obs.data_ptr(), nes.data_ptr(), mp.data_ptr(), mn.data_ptr(),
                                  nes_obs.data_ptr(), counts.data_ptr(), st), "g2v_gsea_norm")
    del es
    nc = [c.cpu().numpy() for c in null_counts(nes, nes_obs)]
    res = finish(names, set_ptr, set_gene, es_obs.cpu().numpy(), nes_obs.cpu().numpy(), counts.cpu().numpy(), nc,
                 mp.cpu().numpy(), mn.cpu().numpy(), B)
    le = [leading_edge(pos_obs, u_obs.astype(np.uint64), m, G) for m in res.members]
    return res._replace(leading_edge=le)
