"""Cross-validated survival prediction from a gene signature (DESIGN.md §4.33): ridge Cox regression (Breslow ties,
penalty 1/2 |beta|^2 on the summed partial likelihood, features standardised per training fold) on K repeats of
F-fold splits stratified by event status, for the biomarkers, for the same number of genes of largest |t| (top_t),
of largest Cox score statistic (top_z) and for R random signatures of that size.  Each fit is scored on its test
fold with Harrell's C; P_random says how often a random signature does at least as well.  The named signatures also
get pre-validated risk groups (Tibshirani & Efron 2002): each sample's out-of-fold risk averaged over the repeats,
split at the median, with a log-rank test and the hazard ratio of the high-risk group.

The biomarkers, top_t and top_z were chosen with every sample, so their C are optimistic and comparable with each
other.  Nested re-selection (steps 3-6 rerun on every training fold) is nested.nested_cv (``--nested-cv``) for the
good / poor label and nested_survival.nested_survival_cv (``--nested-survival-cv``) for survival; the latter scores
on these same splits with cox_fits.

Host side (NumPy): the checks, top_t (signature.top_t), X as float64 gene-major over the time positions, chunking over
whole signatures and the summaries.  Device side: g2v_sig_folds once (y = the event flags), g2v_surv_scores once for
the top_z ranking (survival.rank_genes), then per chunk g2v_sig_draw, g2v_cox_fit (one CTA per fit, Newton on the
device) and g2v_cox_concordance (csrc/g2v_sig.cu, csrc/g2v_surv.cu, csrc/g2v_cox.cu), in cox_fits.
"""
import math
from collections import namedtuple

import numpy as np

from . import perm, signature, survival

MAX_SIZE = signature.MAX_SIZE          # G2V_SIG_MAX_SIZE: p
MAX_FOLDS = signature.MAX_FOLDS        # G2V_SIG_MAX_FOLDS
MAX_REPEATS = signature.MAX_REPEATS    # G2V_SIG_MAX_REPEATS
MAX_RANDOM = signature.MAX_RANDOM      # G2V_SIG_MAX_RANDOM
MAX_FITS = signature.MAX_FITS          # G2V_SIG_MAX_FITS: (R + 3) K F
MAX_STAGED = 18432                     # G2V_COX_MAX_STAGED: test folds of at most this many samples use shared memory
NAMES = ("biomarkers", "top_t", "top_z")
Z95 = 1.959964

SurvivalCVResult = namedtuple("SurvivalCVResult", "names genes folds counts c n_iter converged beta scores c_mean c_sd "
                                                  "p_random risk group logrank_z logrank_p hr hr_low hr_high")
SurvivalCVResult.__doc__ = """survival_cv's result over the n samples with a record, in their input order; S = R + 3
signatures: biomarkers, top_t, top_z, random_1 .. random_R.
names     the S names;  genes: int32 [S, p], each row ascending;  folds: int8 [K, n], the test fold of every sample;
counts    int64 [S, K, F, 3]: per fit over its test fold the comparable, concordant and tied pairs;
c         float64 [S, K, F]: Harrell's C = (2 concordant + tied) / (2 comparable), NaN without a comparable pair;
n_iter    int32 [S, K, F] Newton iterations;  converged: how many of the S K F fits met the step rule within 100
          iterations (the others are reported, not hidden);
beta      float64 [3, K, F, p]: the coefficients (on the standardised genes) of the three named signatures;
scores    float64 [3, K, n]: the out-of-fold linear predictor eta of every sample, for the named signatures;
c_mean    float64 [S], the mean of c over the fits that have a comparable pair;  c_sd: SD (ddof 1) of the K per-repeat
          means, NaN at K = 1;
p_random  float64 [3]: (1 + #{r: c_mean[random_r] >= c_mean[s]}) / (R + 1) for the named signatures;
risk, group   float64 [3, n] and int8 [3, n]: the pre-validated risk (the mean out-of-fold eta over the repeats) and
          1 where it is above the median;
logrank_z, logrank_p   float64 [3]: survival.cox_score of the group and erfc(|Z| / sqrt 2);
hr, hr_low, hr_high    float64 [3]: exp(beta) of the unpenalised Breslow Cox fit of the group and its Wald 95 % CI,
          NaN when either group has no event."""


def check_inputs(expr, time, event, label, p, n_random, folds, repeats):
    """ValueError unless the test can run, before anything is uploaded.  expr [N, G] with time, event and label per
    sample; the samples with a finite time are used (survival.check_inputs: 3 to 32768 of them with at least one
    event, finite expression), and label must allow top_t (perm.check_inputs over the samples with label 0 or 1).
    1 <= R <= 65536, 2 <= F <= 100, 1 <= K <= 100, F <= the events, F <= n / 2, (R + 3) K F <= 2^24 and
    1 <= p <= min(128, G).  Returns (x float64 [n, G], time [n], event int64 [n], used bool [N]).  Needs no GPU."""
    for name, v, lo, hi in (("the number of random signatures R", n_random, 1, MAX_RANDOM),
                            ("the number of folds F", folds, 2, MAX_FOLDS),
                            ("the number of repeats K", repeats, 1, MAX_REPEATS)):
        if int(v) != v or not lo <= int(v) <= hi:
            raise ValueError("%s must be an integer in [%d, %d], got %r" % (name, lo, hi, v))
    x = np.asarray(expr)
    t = np.asarray(time, dtype=np.float64).reshape(-1)
    if x.ndim != 2 or x.shape[0] != t.shape[0]:
        raise ValueError("expression must be [samples, genes] with one time per sample, got %s and %d times"
                         % (x.shape, t.shape[0]))
    used = np.isfinite(t)
    xu, tu, eu = survival.check_inputs(x[used], t[used], np.asarray(event).reshape(-1)[used], 1)
    perm.check_inputs(x, label, 1)
    n, G = xu.shape
    n_ev = int(eu.sum())
    if folds > n_ev:
        raise ValueError("F = %d folds need at least F events, got %d" % (folds, n_ev))
    if folds > n // 2:
        raise ValueError("F = %d folds need at least 2 F samples, got %d" % (folds, n))
    fits = (int(n_random) + 3) * int(repeats) * int(folds)
    if fits > MAX_FITS:
        raise ValueError("(R + 3) x K x F = %d fits, at most 2^24" % fits)
    if int(p) != p or not 1 <= p <= min(MAX_SIZE, G):
        raise ValueError("the signature has %r genes, must be 1 to min(%d, G = %d)" % (p, MAX_SIZE, G))
    return xu, tu, eu, used


def concordance(counts):
    """Harrell's C from counts [..., 3] (comparable, concordant, tied): NaN where nothing is comparable."""
    counts = np.asarray(counts, dtype=np.int64)
    num = (2 * counts[..., 1] + counts[..., 2]).astype(np.float64)
    den = 2.0 * counts[..., 0].astype(np.float64)
    out = np.full(num.shape, np.nan)
    np.divide(num, den, out=out, where=den > 0)
    return out


def summarise(c, n_named, R):
    """(c_mean, c_sd, p_random) from the per-fit C [S, K, F]; NaN folds are left out of the means."""
    S, K, F = c.shape
    flat = c.reshape(S, K * F)
    has = ~np.isnan(flat)
    cnt = has.sum(axis=1)
    c_mean = np.where(cnt > 0, np.where(has, flat, 0.0).sum(axis=1) / np.maximum(cnt, 1), np.nan)
    with np.errstate(invalid="ignore"):
        kh = (~np.isnan(c)).sum(axis=2)
        per_repeat = np.where(kh > 0, np.where(np.isnan(c), 0.0, c).sum(axis=2) / np.maximum(kh, 1), np.nan)
        c_sd = per_repeat.std(axis=1, ddof=1) if K > 1 else np.full(S, np.nan)
    rnd = c_mean[n_named:]
    p_random = np.array([(1.0 + (rnd >= c_mean[s]).sum()) / (R + 1.0) for s in range(n_named)])
    return c_mean, c_sd, p_random


def cox_hr(x, time, event, max_iter=100):
    """(hr, lo, hi): the unpenalised Breslow Cox fit of one covariate by Newton with step halving, exp(beta) and the
    Wald 95 % interval exp(beta -+ 1.959964 / sqrt(I(beta)))."""
    x = np.asarray(x, dtype=np.float64)
    order, _, flags, _, _ = survival.time_groups(time, event)
    xs = x[order]
    ev = (flags & 1).astype(bool)
    end = (flags & 2).astype(bool)
    grp = np.cumsum(np.r_[0, end[:-1]])
    d = np.bincount(grp, weights=ev.astype(np.float64))
    e1 = np.bincount(grp, weights=np.where(ev, xs, 0.0))

    def terms(b):
        eta = b * xs
        M = np.maximum.accumulate(eta)                 # a shift per position that never overflows
        Mk = M[end]
        # risk-set sums under the group's own shift, accumulated in descending time
        s0 = np.empty(Mk.shape); s1 = np.empty(Mk.shape); s2 = np.empty(Mk.shape)
        a0 = a1 = a2 = 0.0
        prev = -np.inf
        k = 0
        for i in range(xs.shape[0]):
            if M[i] > prev:
                sc = math.exp(prev - M[i]) if prev > -np.inf else 0.0
                a0 *= sc; a1 *= sc; a2 *= sc
                prev = M[i]
            w = math.exp(eta[i] - prev)
            a0 += w; a1 += w * xs[i]; a2 += w * xs[i] * xs[i]
            if end[i]:
                s0[k], s1[k], s2[k] = a0, a1, a2
                k += 1
        m = s1 / s0
        L = float((d * (np.log(s0) + Mk)).sum() - (b * e1).sum())
        U = float((e1 - d * m).sum())
        I = float((d * (s2 / s0 - m * m)).sum())
        return L, U, I

    b = 0.0
    L, U, I = terms(b)
    for _ in range(max_iter):
        if I <= 0:
            break
        step = U / I
        t = 1.0
        while True:
            Lc, Uc, Ic = terms(b + t * step)
            if Lc <= L or t < 2.0 ** -40:
                break
            t *= 0.5
        b += t * step
        L, U, I = Lc, Uc, Ic
        if abs(t * step) <= 1e-12 * max(1.0, abs(b)):
            break
    if I <= 0:
        return math.nan, math.nan, math.nan
    se = 1.0 / math.sqrt(I)
    return math.exp(b), math.exp(b - Z95 * se), math.exp(b + Z95 * se)


def risk_groups(scores, time, event):
    """Pre-validation of one signature from its out-of-fold eta [K, n]: (risk [n], group int8 [n], Z, P, HR, lo, hi)
    with risk the mean over the repeats, group 1 where risk > median(risk), Z = survival.cox_score(group), P =
    erfc(|Z| / sqrt 2), and the hazard ratio of the group with its 95 % CI (NaN when either group has no event)."""
    risk = np.asarray(scores, dtype=np.float64).mean(axis=0)
    group = (risk > np.median(risk)).astype(np.int8)
    ev = np.asarray(event).astype(np.int64)
    z = survival.cox_score(group.astype(np.float64), time, ev)[0]
    p = math.erfc(abs(z) / math.sqrt(2.0))
    if not ((ev[group == 1] == 1).any() and (ev[group == 0] == 1).any()):
        return risk, group, z, p, math.nan, math.nan, math.nan
    hr, lo, hi = cox_hr(group, time, ev)
    return risk, group, z, p, hr, lo, hi


def summary(res):
    """The command line's line."""
    S, K, F = res.c.shape
    rnd = res.c_mean[3:]
    lo, hi = np.nanpercentile(rnd, [2.5, 97.5]) if np.isfinite(rnd).any() else (math.nan, math.nan)
    line = ("survival CV: %d-fold x %d repeats, %d genes: C %.3f (biomarkers), %.3f (top |t|), %.3f (top |Z|), random "
            "mean %.3f [%.3f, %.3f]; P_random %.3g / %.3g / %.3g; biomarker risk groups: log-rank Z = %.4f, P = %.4g, "
            "HR %.3f (%.3f, %.3f)"
            % (F, K, res.genes.shape[1], res.c_mean[0], res.c_mean[1], res.c_mean[2], np.nanmean(rnd), lo, hi,
               res.p_random[0], res.p_random[1], res.p_random[2], res.logrank_z[0], res.logrank_p[0], res.hr[0],
               res.hr_low[0], res.hr_high[0]))
    if res.converged < S * K * F:
        line += "; %d of %d fits did not converge" % (S * K * F - res.converged, S * K * F)
    return line


def chunk_signatures(S, n, p, K, F, max_chunk_bytes):
    """Signatures per chunk: scores (8 K n bytes), the fits' scratch (8 K F n), genes (4 p), counts, n_iter and
    converged (29 K F) of each within max_chunk_bytes, at least 1."""
    per_sig = 8 * K * n + 8 * K * F * n + 4 * p + 29 * K * F
    return int(max(1, min(S, int(max_chunk_bytes) // per_sig)))


def survival_cv(expr, time, event, label, signature_genes, n_random, folds=5, repeats=10, seed=0,
                max_chunk_bytes=None):
    """Cross-validated Harrell's C of the signature against top_t, top_z and n_random random signatures of its size,
    on the GPU.

    expr: host float array [N, genes] of every expression sample; time, event: per sample as survival.match_survival
    gives them (time NaN where there is no record: those samples are left out of the fits); label: per sample (0 good,
    1 poor; others are left out of top_t only).  signature_genes: distinct gene indices (columns of expr).  folds F,
    repeats K: K repeats of F-fold splits stratified by event status, the same for every signature; seed: the Philox
    key of the splits and of the random signatures (those of signature.signature_cv at the same seed and size).
    max_chunk_bytes: bound on the device memory of one chunk's per-signature buffers (default: half the free device
    memory); the result does not depend on it.  Returns a SurvivalCVResult; ValueError (before anything is uploaded)
    on inputs check_inputs refuses or a signature with repeated or out-of-range genes, RuntimeError without a GPU."""
    sig = np.asarray(signature_genes).reshape(-1)
    x, t, e, used = check_inputs(expr, time, event, label, sig.shape[0], n_random, folds, repeats)
    G = x.shape[1]
    if sig.dtype.kind not in "iu" or (sig.size and (sig.min() < 0 or sig.max() >= G)) or np.unique(sig).size != sig.size:
        raise ValueError("the signature must be distinct gene indices in [0, %d)" % G)
    p, R, K, F = int(sig.shape[0]), int(n_random), int(repeats), int(folds)
    tt = signature.top_t(expr, label, p)
    tz = np.sort(survival.rank_genes(x, t, e)[:p]).astype(np.int32)          # RuntimeError without a GPU
    head = np.stack([np.sort(sig).astype(np.int32), tt, tz])
    genes, folds_s, counts, n_iter, conv, beta, scores = cox_fits(x, t, e, head, R, K, F, seed,
                                                                  max_chunk_bytes=max_chunk_bytes)
    c = concordance(counts)
    c_mean, c_sd, p_random = summarise(c, 3, R)
    rg = [risk_groups(scores[s], t, e) for s in range(3)]
    col = lambda j: np.array([r[j] for r in rg], dtype=np.float64)
    return SurvivalCVResult(names=list(NAMES) + ["random_%d" % r for r in range(1, R + 1)], genes=genes,
                            folds=folds_s, counts=counts, c=c, n_iter=n_iter, converged=int(conv.sum()),
                            beta=beta, scores=scores, c_mean=c_mean, c_sd=c_sd, p_random=p_random,
                            risk=np.stack([r[0] for r in rg]), group=np.stack([r[1] for r in rg]),
                            logrank_z=col(2), logrank_p=col(3), hr=col(4), hr_low=col(5), hr_high=col(6))


def cox_fits(x, time, event, head, n_random, repeats, folds, seed, fold=None, cap=None, max_chunk_bytes=None):
    """The device part of survival_cv, also run by nested_survival.nested_survival_cv: the ridge Cox fits and test-fold
    concordance counts of S = H + R signatures, the H rows of head [H, p] (sorted distinct gene indices) then
    random_1 .. random_R (g2v_sig_draw, the random signatures of survival_cv at the same seed).

    x float64 [n, G], time [n] and event [n]: the samples with a record, as check_inputs returns them (not checked
    here).  fold: None to split with g2v_sig_folds (K repeats of F-fold stratified by event status at seed), or an
    int8 [K, n] array of test folds 0..F-1 over the samples to fit on instead.  cap: the largest test fold
    g2v_cox_concordance stages in shared memory (a larger fold is read from global memory, with the same counts);
    default the largest stratified fold.  Returns (genes int32 [S, p], fold int8 [K, n], counts int64 [S, K, F, 3],
    n_iter int32 [S, K, F], converged uint8 [S, K, F], beta float64 [H, K, F, p], scores float64 [H, K, n]: the
    out-of-fold eta of every sample for the head rows), every per-sample array in the samples' order."""
    n, G = x.shape
    H, p = head.shape
    R, K, F = int(n_random), int(repeats), int(folds)
    S = H + R
    import torch
    from . import _capi
    lib = _capi.load()
    if not torch.cuda.is_available():
        raise RuntimeError("g2vec_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    dev = torch.device("cuda", torch.cuda.current_device())
    st = torch.cuda.current_stream(dev).cuda_stream
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    order, _, flags, _, _ = survival.time_groups(time, event)
    end = (flags & 2).astype(bool)
    grp = np.cumsum(np.r_[0, end[:-1]]).astype(np.int32)
    n_pad = -(-n // 32) * 32
    Xt = np.zeros((G, n_pad), dtype=np.float64)
    Xt[:, :n] = x[order].T
    X_d = up(Xt)
    del Xt
    flags_d, grp_d = up(flags), up(grp)
    ev_d = up((flags & 1).astype(np.uint8))
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    if fold is None:
        fold_d = torch.empty((K, n), dtype=torch.int8, device=dev)
        _capi.check(lib.g2v_sig_folds(ev_d.data_ptr(), n, K, F, seed, fold_d.data_ptr(), st), "g2v_sig_folds")
    else:
        fold_d = up(np.asarray(fold, dtype=np.int8)[:, order])       # samples -> time positions
    if cap is None:
        n_ev = int(np.asarray(event).sum())
        cap = -(-n_ev // F) + -(-(n - n_ev) // F)      # the largest test fold
    cap = cap if cap <= MAX_STAGED else 0
    if max_chunk_bytes is None:
        max_chunk_bytes = torch.cuda.mem_get_info(dev)[0] // 2
    rows = chunk_signatures(S, n, p, K, F, max_chunk_bytes)
    genes = np.empty((S, p), dtype=np.int32)
    genes[:H] = head
    counts = np.empty((S, K, F, 3), dtype=np.int64)
    n_iter = np.empty((S, K, F), dtype=np.int32); conv = np.empty((S, K, F), dtype=np.uint8)
    beta = torch.empty((H, K, F, p), dtype=torch.float64, device=dev)
    named = np.empty((H, K, n))
    g_d = torch.empty((rows, p), dtype=torch.int32, device=dev)
    sc_d = torch.empty((rows, K, n), dtype=torch.float64, device=dev)
    ell_d = torch.empty((rows * K * F, n), dtype=torch.float64, device=dev)
    cnt_d = torch.empty((rows, K, F, 3), dtype=torch.int64, device=dev)
    it_d = torch.empty((rows, K, F), dtype=torch.int32, device=dev)
    cv_d = torch.empty((rows, K, F), dtype=torch.uint8, device=dev)
    for s0 in range(0, S, rows):
        ns = min(rows, S - s0)
        fixed = min(ns, max(0, H - s0))                # rows of this chunk that come from head
        if fixed:
            g_d[:fixed] = up(head[s0:s0 + fixed])
        if ns > fixed:
            _capi.check(lib.g2v_sig_draw(G, p, seed, s0 + fixed - H + 1, ns - fixed, g_d[fixed].data_ptr(), st),
                        "g2v_sig_draw")
        _capi.check(lib.g2v_cox_fit(X_d.data_ptr(), G, n, n_pad, flags_d.data_ptr(), fold_d.data_ptr(), K, F,
                                    g_d.data_ptr(), ns, p, ell_d.data_ptr(), sc_d.data_ptr(), it_d.data_ptr(),
                                    cv_d.data_ptr(), beta[s0].data_ptr() if fixed else None, fixed, st), "g2v_cox_fit")
        _capi.check(lib.g2v_cox_concordance(sc_d.data_ptr(), flags_d.data_ptr(), grp_d.data_ptr(), fold_d.data_ptr(),
                                            n, K, F, ns, cap, cnt_d.data_ptr(), st), "g2v_cox_concordance")
        sl = slice(s0, s0 + ns)
        genes[sl] = g_d[:ns].cpu().numpy()
        counts[sl] = cnt_d[:ns].cpu().numpy()
        n_iter[sl] = it_d[:ns].cpu().numpy(); conv[sl] = cv_d[:ns].cpu().numpy()
        if fixed:
            named[s0:s0 + fixed] = sc_d[:fixed].cpu().numpy()
    scores = np.empty_like(named)
    scores[:, :, order] = named                        # time positions -> samples
    folds_s = np.empty((K, n), dtype=np.int8)
    folds_s[:, order] = fold_d.cpu().numpy()
    return genes, folds_s, counts, n_iter, conv, beta.cpu().numpy(), scores
