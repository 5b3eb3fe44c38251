"""NumPy restatement of the gene-set enrichment test (DESIGN.md §4.28) -- test infrastructure for
tests/test_gsea_host.py and tests/test_gpu_gsea.py, with the float64 operations of csrc/g2v_gsea.cu:

* ``keys``: rq, u and the sort keys of g2v_gsea_keys;
* ``rank``: pos of g2v_gsea_rank (the keys are unique, so any sort gives the same ranks);
* ``es``: the enrichment scores of g2v_gsea_es from sorted member positions and exact prefix sums;
* ``es_brute``: the textbook running sum of P_hit - P_miss over all G positions, its maximum deviation;
* ``norm``: g2v_gsea_norm, the sums taken one permutation at a time in b order;
* ``null_counts``: the FDR and FWER counts of gsea.null_counts;
* ``gsea``: the whole test on the host, through perm_oracle's labels and sums.
"""
import numpy as np

from g2vec_b200 import perm
from g2vec_b200.gsea import Q_SCALE, check_inputs, finish, leading_edge, restrict_sets, sign_of
from tests import perm_oracle

GENE_BITS = 20


def keys(A, n, k, s, Q, W):
    """A [n_b, G] int64 sums -> (rq, u, key), int64 [n_b, G] each."""
    A = np.atleast_2d(np.asarray(A, dtype=np.int64))
    N = n * A - k * np.asarray(Q, dtype=np.int64)[None, :]
    sN = (N if s > 0 else -N).astype(np.float64)
    W = np.broadcast_to(np.asarray(W, dtype=np.float64)[None, :], sN.shape)
    r = np.zeros(sN.shape)
    np.divide(sN, np.sqrt(W, where=W > 0, out=np.ones(sN.shape)), out=r, where=W > 0)
    rq = np.rint(r * Q_SCALE).astype(np.int64)
    g = np.arange(A.shape[1], dtype=np.int64)[None, :]
    return rq, np.abs(rq), (((1 << 32) - rq) << GENE_BITS) | g


def rank(key):
    """key [n_b, G] -> pos [n_b, G] int32."""
    key = np.atleast_2d(key)
    order = np.argsort(key, axis=1, kind="stable")
    pos = np.empty(key.shape, dtype=np.int32)
    np.put_along_axis(pos, order, np.arange(key.shape[1], dtype=np.int32)[None, :].repeat(key.shape[0], 0), axis=1)
    return pos


def es_one(pos, u, members, G):
    """ES of one set (gene indices `members`) in one ranking: pos [G], u [G]."""
    members = np.asarray(members, dtype=np.int64)
    k = len(members)
    o = np.argsort(pos[members])
    p = pos[members][o].astype(np.int64)
    w = np.asarray(u)[members][o].astype(np.int64)
    S = np.cumsum(w)
    NR = int(S[-1])
    if NR == 0:
        return 0.0
    m = (p - np.arange(k)).astype(np.float64) / float(G - k)
    dp = max(0.0, float((S.astype(np.float64) / float(NR) - m).max()))
    dm = min(0.0, float(((S - w).astype(np.float64) / float(NR) - m).min()))
    return dp if dp >= -dm else dm


def es(pos, u, set_ptr, set_gene):
    """es [n_b, S] of every set in every row of pos / u [n_b, G]."""
    pos, u = np.atleast_2d(pos), np.atleast_2d(u)
    G = pos.shape[1]
    S = len(set_ptr) - 1
    out = np.empty((pos.shape[0], S))
    for r in range(pos.shape[0]):
        for i in range(S):
            out[r, i] = es_one(pos[r], u[r], set_gene[set_ptr[i]:set_ptr[i + 1]], G)
    return out


def es_brute(weight, members):
    """Subramanian et al.'s running sum: genes ordered by `weight` (signed, any float or int) descending, ties by index;
    P_hit adds |weight| of the hits over their total, P_miss 1 / (G - k) per miss; returns the deviation of largest
    magnitude (the positive one on a tie), 0 when the hits weigh nothing.  In float64, to compare within rounding."""
    weight = np.asarray(weight)
    G = weight.shape[0]
    order = np.lexsort((np.arange(G), -weight))
    hit = np.isin(order, members)
    w = np.abs(weight[order]).astype(np.float64) * hit
    if w.sum() == 0:
        return 0.0
    d = np.cumsum(w) / w.sum() - np.cumsum(~hit) / float((~hit).sum())
    dp, dm = max(0.0, d.max()), min(0.0, d.min())
    return dp if dp >= -dm else dm


def norm(es_null, es_obs):
    """(nes [B, S], mean_pos, mean_neg, nes_obs, counts [3, S]) of g2v_gsea_norm."""
    es_null = np.asarray(es_null, dtype=np.float64)
    B, S = es_null.shape
    sp, sn = np.zeros(S), np.zeros(S)
    npos, nneg, ext = np.zeros(S, np.int64), np.zeros(S, np.int64), np.zeros(S, np.int64)
    up = es_obs >= 0
    for b in range(B):
        e = es_null[b]
        sp = np.where(e >= 0, sp + e, sp)
        sn = np.where(e < 0, sn + (-e), sn)
        npos += e >= 0
        nneg += e < 0
        ext += np.where(up, e >= es_obs, e <= es_obs)
    with np.errstate(divide="ignore", invalid="ignore"):
        mp = np.where(npos > 0, sp / np.maximum(npos, 1), np.nan)
        mn = np.where(nneg > 0, sn / np.maximum(nneg, 1), np.nan)
        nes_obs = np.where(up, np.where(npos > 0, es_obs / mp, np.nan), np.where(nneg > 0, es_obs / mn, np.nan))
        nes = np.where(es_null >= 0, es_null / mp[None, :], es_null / mn[None, :])
    nes[:, np.isnan(nes_obs)] = np.nan
    return nes, mp, mn, nes_obs, np.stack([npos, nneg, ext])


def null_counts(nes, nes_obs):
    """(count_null, count_null_side, count_fwer) straight from their definitions, one set at a time."""
    B, S = nes.shape
    cnt, side, fw = (np.zeros(S, np.int64) for _ in range(3))
    with np.errstate(invalid="ignore"):
        pos_v, neg_v = nes[nes >= 0], nes[nes < 0]
        for i in range(S):
            x = nes_obs[i]
            if x >= 0:
                cnt[i], side[i] = (pos_v >= x).sum(), pos_v.size
                fw[i] = sum(1 for b in range(B) if (nes[b] >= 0).any() and nes[b][nes[b] >= 0].max() >= x)
            else:
                cnt[i], side[i] = (neg_v <= x).sum(), neg_v.size
                fw[i] = sum(1 for b in range(B) if (nes[b] < 0).any() and nes[b][nes[b] < 0].min() <= x)
    return cnt, side, fw


def gsea(expr, label, sets, n_perm, seed=0, min_size=15, max_size=500, genes=None, chunk=None):
    """The whole test on the host: a GseaResult with the bits of gsea.gsea."""
    x = np.asarray(expr)
    G = x.shape[1]
    set_ptr, set_gene, names = restrict_sets(sets, range(G) if genes is None else genes, min_size, max_size)
    check_inputs(expr, label, n_perm, len(names), min_size, max_size)
    prep = perm.prepare(expr, label, n_perm)
    n, k, s = prep["n"], prep["k"], sign_of(prep)
    S_pad = -(-n // 32) * 32
    M_obs = np.zeros((1, S_pad), np.uint8); M_obs[0, :n] = prep["obs"]
    _, u_obs, key_obs = keys(perm_oracle.sums(M_obs, prep["q"]), n, k, s, prep["Q"], prep["W"])
    pos_obs = rank(key_obs)
    es_obs = es(pos_obs, u_obs, set_ptr, set_gene)[0]
    rows = []
    chunk = chunk or n_perm
    for b0 in range(0, n_perm, chunk):
        M = perm_oracle.labels(prep["obs"], S_pad, seed, b0, min(chunk, n_perm - b0))
        _, u, key = keys(perm_oracle.sums(M, prep["q"]), n, k, s, prep["Q"], prep["W"])
        rows.append(es(rank(key), u, set_ptr, set_gene))
    nes, mp, mn, nes_obs, counts = norm(np.concatenate(rows), es_obs)
    res = finish(names, set_ptr, set_gene, es_obs, nes_obs, counts, null_counts(nes, nes_obs), mp, mn, n_perm)
    le = [leading_edge(pos_obs[0], u_obs[0].astype(np.uint64), m, G) for m in res.members]
    return res._replace(leading_edge=le)
