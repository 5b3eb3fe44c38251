"""Cross-validated prediction of the good / poor label from a gene signature (DESIGN.md §4.29): ridge logistic
regression (scikit-learn's LogisticRegression(C=1.0) objective) on K repeats of stratified F-fold splits, for the
biomarkers, for the same number of genes of largest |t| (top_t) and for R random signatures of that size.

The biomarkers and top_t were both chosen with every sample's label, so their AUCs are optimistic and comparable with
each other (Ambroise & McLachlan 2002); the random signatures are not selected, and most random gene sets already carry
some of the outcome (Venet et al. 2011), so P_random says how often a random signature does at least as well.  The
honest AUC of the selection itself, with steps 3-6 rerun on every training fold, is nested.nested_cv
(``--nested-cv``), which scores on these same splits with cv_fits.

Host side (NumPy): the checks, top_t from perm.prepare's exact ranking, X as float64 gene-major, chunking over whole
signatures and the summaries.  Device side (csrc/g2v_sig.cu): g2v_sig_folds once, then per chunk g2v_sig_draw,
g2v_sig_fit (one CTA per fit, Newton on the device, Gram matrix on the FP64 tensor cores) and g2v_sig_auc, in
cv_fits.
"""
from collections import namedtuple

import numpy as np

from . import perm

MAX_SIZE = 128               # G2V_SIG_MAX_SIZE: p
MAX_FOLDS = 100              # G2V_SIG_MAX_FOLDS
MAX_REPEATS = 100            # G2V_SIG_MAX_REPEATS
MAX_RANDOM = 1 << 16         # G2V_SIG_MAX_RANDOM
MAX_FITS = 1 << 24           # G2V_SIG_MAX_FITS: (R + 2) K F
NAMES = ("biomarkers", "top_t")

SignatureResult = namedtuple("SignatureResult", "names genes folds auc acc n_iter converged beta auc_mean auc_sd "
                                                "acc_mean p_random")
SignatureResult.__doc__ = """signature_cv's result, S = R + 2 signatures: biomarkers, top_t, random_1 .. random_R.
names     the S names;  genes: int32 [S, p], each row ascending;  folds: int8 [K, n], the fold of every used sample;
auc, acc  float64 [S, K, F]: per fit the test fold's AUC (ties count 1/2) and accuracy (logit > 0 predicts poor);
n_iter    int32 [S, K, F] Newton iterations;  converged: how many of the S K F fits met the step rule within 100
          iterations (the others are reported, not hidden);
beta      float64 [2, K, F, p + 1]: intercept then coefficients (on the standardised genes) of biomarkers and top_t;
auc_mean, acc_mean   float64 [S], the means over the K F fits;  auc_sd: SD (ddof 1) of the K per-repeat mean AUCs,
          NaN at K = 1;
p_random  float64 [2]: (1 + #{r: auc_mean[random_r] >= auc_mean[s]}) / (R + 1) for biomarkers and top_t."""


def check_inputs(expr, label, p, n_random, folds, repeats):
    """ValueError unless the signature test can run: perm.check_inputs' conditions (labels 0 and 1 both present,
    3 <= n <= 32768 samples with label 0 or 1, finite expression), 2 <= F <= min(n0, n1) and F <= 100, 1 <= K <= 100,
    1 <= R <= 65536, 1 <= p <= min(128, G) and (R + 2) K F <= 2^24.  Returns (x, lab) as perm.check_inputs.  Needs no
    GPU."""
    for name, v, lo, hi in (("the number of random signatures R", n_random, 1, MAX_RANDOM),
                            ("the number of folds F", folds, 2, MAX_FOLDS),
                            ("the number of repeats K", repeats, 1, MAX_REPEATS)):
        if int(v) != v or not lo <= int(v) <= hi:
            raise ValueError("signature test: %s must be an integer in [%d, %d], got %r" % (name, lo, hi, v))
    x, lab = perm.check_inputs(expr, label, 1)
    n0, n1 = int((lab == 0).sum()), int((lab == 1).sum())
    if folds > min(n0, n1):
        raise ValueError("signature test: F = %d folds need at least F samples of each label, got %d and %d"
                         % (folds, n0, n1))
    G = x.shape[1]
    if int(p) != p or not 1 <= p <= min(MAX_SIZE, G):
        raise ValueError("signature test: the signature has %r genes, must be 1 to min(%d, G = %d)" % (p, MAX_SIZE, G))
    fits = (int(n_random) + 2) * int(repeats) * int(folds)
    if fits > MAX_FITS:
        raise ValueError("signature test: (R + 2) x K x F = %d fits, at most 2^24" % fits)
    return x, lab


def top_t(expr, label, p):
    """The p genes of largest |t| (perm.prepare's exact point-biserial ranking, ties by gene index), ascending."""
    return np.sort(perm.prepare(expr, label)["order"][:p]).astype(np.int32)


def summarise(auc, acc, R):
    """(auc_mean, auc_sd, acc_mean, p_random) from the per-fit auc and acc [S, K, F]."""
    S, K, F = auc.shape
    auc_mean = auc.reshape(S, K * F).mean(axis=1)
    acc_mean = acc.reshape(S, K * F).mean(axis=1)
    per_repeat = auc.mean(axis=2)
    auc_sd = per_repeat.std(axis=1, ddof=1) if K > 1 else np.full(S, np.nan)
    rnd = auc_mean[2:]
    p_random = np.array([(1.0 + (rnd >= auc_mean[s]).sum()) / (R + 1.0) for s in (0, 1)])
    return auc_mean, auc_sd, acc_mean, p_random


def summary(res):
    """The signature line of the command line."""
    S, K, F = res.auc.shape
    rnd = res.auc_mean[2:]
    lo, hi = np.percentile(rnd, [2.5, 97.5])
    line = ("signature CV: %d-fold x %d repeats, %d genes: AUC %.3f (biomarkers), %.3f (top |t|), random mean %.3f "
            "[%.3f, %.3f]; P_random %.3g / %.3g" % (F, K, res.genes.shape[1], res.auc_mean[0], res.auc_mean[1],
                                                     rnd.mean(), lo, hi, res.p_random[0], res.p_random[1]))
    if res.converged < S * K * F:
        line += "; %d of %d fits did not converge" % (S * K * F - res.converged, S * K * F)
    return line


def chunk_signatures(S, n, p, K, F, max_chunk_bytes):
    """Signatures per chunk: scores (8 K n bytes), genes (4 p), auc, acc, n_iter, converged (21 K F) of each within
    max_chunk_bytes, at least 1."""
    per_sig = 8 * K * n + 4 * p + 21 * K * F
    return int(max(1, min(S, int(max_chunk_bytes) // per_sig)))


def signature_cv(expr, label, signature, n_random, folds=5, repeats=10, seed=0, max_chunk_bytes=None):
    """Cross-validated AUC of the signature against top_t and n_random random signatures of its size, on the GPU.

    expr: host float array [samples, genes]; label: one int per sample (0 good, 1 poor; other labels are left out);
    signature: distinct gene indices (columns of expr).  folds F, repeats K: K repeats of stratified F-fold splits,
    the same for every signature; seed: the Philox key of the splits and the random signatures.  max_chunk_bytes:
    bound on the device memory of one chunk's per-signature buffers (default: half the free device memory); the
    result does not depend on it.  Returns a SignatureResult; ValueError (before anything is uploaded) on inputs
    check_inputs refuses or a signature with repeated or out-of-range genes, RuntimeError without a GPU."""
    sig = np.asarray(signature).reshape(-1)
    x, lab = check_inputs(expr, label, sig.shape[0], n_random, folds, repeats)
    G = x.shape[1]
    if sig.dtype.kind not in "iu" or (sig.size and (sig.min() < 0 or sig.max() >= G)) or np.unique(sig).size != sig.size:
        raise ValueError("signature test: the signature must be distinct gene indices in [0, %d)" % G)
    p, R, K, F = int(sig.shape[0]), int(n_random), int(repeats), int(folds)
    head = np.stack([np.sort(sig).astype(np.int32), top_t(expr, label, p)])
    genes, fold, auc, acc, n_iter, conv, beta = cv_fits(x, lab, head, R, K, F, seed, max_chunk_bytes=max_chunk_bytes)
    auc_mean, auc_sd, acc_mean, p_random = summarise(auc, acc, R)
    return SignatureResult(names=list(NAMES) + ["random_%d" % r for r in range(1, R + 1)], genes=genes, folds=fold,
                           auc=auc, acc=acc, n_iter=n_iter, converged=int(conv.sum()), beta=beta, auc_mean=auc_mean,
                           auc_sd=auc_sd, acc_mean=acc_mean, p_random=p_random)


def cv_fits(x, lab, head, n_random, repeats, folds, seed, fold=None, cap=None, max_chunk_bytes=None):
    """The device part of signature_cv, also run by nested.nested_cv: the fits and test-fold scores of S = H + R
    signatures, the H rows of head [H, p] (sorted distinct gene indices) then random_1 .. random_R (g2v_sig_draw).

    x float64 [n, G] and lab [n] in {0, 1}: the used samples, as check_inputs returns them (not checked here).  fold:
    None to split with g2v_sig_folds (K repeats of stratified F-fold at seed), or an int8 [K, n] array of test folds
    0..F-1 to fit on instead.  cap: the largest test fold g2v_sig_auc scores (a larger fold gets NaN); default the
    largest stratified fold.  Returns (genes int32 [S, p], fold int8 [K, n], auc, acc float64 [S, K, F], n_iter int32
    [S, K, F], converged uint8 [S, K, F], beta float64 [H, K, F, p + 1])."""
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
    n_pad = -(-n // 32) * 32
    Xt = np.zeros((G, n_pad), dtype=np.float64)
    Xt[:, :n] = x.T
    X_d = torch.from_numpy(Xt).to(dev)
    del Xt
    y_d = torch.from_numpy(lab.astype(np.uint8)).to(dev)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    if fold is None:
        fold_d = torch.empty((K, n), dtype=torch.int8, device=dev)
        _capi.check(lib.g2v_sig_folds(y_d.data_ptr(), n, K, F, seed, fold_d.data_ptr(), st), "g2v_sig_folds")
    else:
        fold_d = torch.from_numpy(np.ascontiguousarray(fold, dtype=np.int8)).to(dev)
    if cap is None:
        n0, n1 = int((lab == 0).sum()), int((lab == 1).sum())
        cap = -(-n0 // F) + -(-n1 // F)                # the largest test fold
    if max_chunk_bytes is None:
        max_chunk_bytes = torch.cuda.mem_get_info(dev)[0] // 2
    rows = chunk_signatures(S, n, p, K, F, max_chunk_bytes)
    genes = np.empty((S, p), dtype=np.int32)
    genes[:H] = head
    auc = np.empty((S, K, F)); acc = np.empty((S, K, F))
    n_iter = np.empty((S, K, F), dtype=np.int32); conv = np.empty((S, K, F), dtype=np.uint8)
    beta = torch.empty((H, K, F, p + 1), dtype=torch.float64, device=dev)
    g_d = torch.empty((rows, p), dtype=torch.int32, device=dev)
    sc_d = torch.empty((rows, K, n), dtype=torch.float64, device=dev)
    auc_d, acc_d = (torch.empty((rows, K, F), dtype=torch.float64, device=dev) for _ in range(2))
    it_d = torch.empty((rows, K, F), dtype=torch.int32, device=dev)
    cv_d = torch.empty((rows, K, F), dtype=torch.uint8, device=dev)
    for s0 in range(0, S, rows):
        ns = min(rows, S - s0)
        fixed = min(ns, max(0, H - s0))                # rows of this chunk that come from head
        if fixed:
            g_d[:fixed] = torch.from_numpy(head[s0:s0 + fixed]).to(dev)
        if ns > fixed:
            _capi.check(lib.g2v_sig_draw(G, p, seed, s0 + fixed - H + 1, ns - fixed, g_d[fixed].data_ptr(), st),
                        "g2v_sig_draw")
        _capi.check(lib.g2v_sig_fit(X_d.data_ptr(), G, n, n_pad, y_d.data_ptr(), fold_d.data_ptr(), K, F,
                                    g_d.data_ptr(), ns, p, sc_d.data_ptr(), it_d.data_ptr(), cv_d.data_ptr(),
                                    beta[s0].data_ptr() if fixed else None, fixed, st), "g2v_sig_fit")
        _capi.check(lib.g2v_sig_auc(sc_d.data_ptr(), y_d.data_ptr(), fold_d.data_ptr(), n, K, F, ns, cap,
                                    auc_d.data_ptr(), acc_d.data_ptr(), st), "g2v_sig_auc")
        sl = slice(s0, s0 + ns)
        genes[sl] = g_d[:ns].cpu().numpy()
        auc[sl] = auc_d[:ns].cpu().numpy(); acc[sl] = acc_d[:ns].cpu().numpy()
        n_iter[sl] = it_d[:ns].cpu().numpy(); conv[sl] = cv_d[:ns].cpu().numpy()
    return genes, fold_d.cpu().numpy(), auc, acc, n_iter, conv, beta.cpu().numpy()
