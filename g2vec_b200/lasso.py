"""Cross-validated lasso / elastic-net logistic regression of the good / poor label on every gene (DESIGN.md §4.37):
glmnet's path (Friedman, Hastie & Tibshirani 2010) on the full cohort and on every training fold of the splits
``--signature-cv`` uses, cv.glmnet's deviance rule for lambda_min and lambda_1se, and top_lasso, the genes in the order
they enter the path: the standard supervised sparse baseline beside the biomarkers.

Host side (NumPy): the checks, the lambda sequence from the device's lambda_max, the round loop, chunking over whole
fits and the summaries.  Device side (csrc/g2v_lasso.cu): g2v_lasso_standardise, then per lambda g2v_lasso_grad and
g2v_lasso_cd in rounds until every fit is certified (or out of Newton steps), and g2v_lasso_score; the held-out AUCs
are g2v_sig_auc's.
"""
from collections import namedtuple

import numpy as np

from . import perm, signature

N_LAMBDA = 100               # G2V_LASSO_N_LAMBDA
MAX_ACTIVE = 512             # G2V_LASSO_MAX_ACTIVE
MAX_GENES = 1 << 20          # G2V_LASSO_MAX_GENES
EPS = 1e-7                   # G2V_LASSO_EPS: the certificate's tolerance
MAX_FOLDS = signature.MAX_FOLDS
MAX_REPEATS = signature.MAX_REPEATS

LassoResult = namedtuple("LassoResult", "alpha lambdas n_lambda a0 beta df dev_ratio cvm cvsd auc auc_mean i_min i_1se "
                                        "folds entry entry_abs n_iter kkt converged fits scores")
LassoResult.__doc__ = """lasso_cv's result over the L' lambdas of the path (fit 0 decides L'), K repeats of F folds.
alpha      the elastic-net mixing;  lambdas: float64 [L'];  n_lambda: L' (at most 100);
a0, beta   float64 [L'] and [L', G]: fit 0's intercept and coefficients on the standardised genes;
df, dev_ratio   int32 / float64 [L']: fit 0's nonzero genes and deviance ratio 1 - dev / dev_null;
cvm, cvsd  float64 [L']: cv.glmnet's fold-size-weighted mean held-out binomial deviance and its standard error over
           the K F folds;  auc: float64 [L', K, F], each fold's held-out AUC (g2v_sig_auc);  auc_mean: [L'];
i_min, i_1se    the indices of lambda_min (argmin cvm) and lambda_1se (the largest lambda with cvm <= cvm[i_min] +
           cvsd[i_min]);  folds: int8 [K, n], the fold of every used sample;
entry      int16 [1 + K F, G]: per fit, the first lambda index at which the gene is nonzero (-1: never);
entry_abs  float64 [1 + K F, G]: |beta| at that index;
n_iter     int32 [1 + K F, L']: Newton steps;  kkt: float64 [1 + K F, L']: the largest KKT violation of each reported
           solution (checked on the device in float64);  converged: how many of the (1 + K F) L' solutions certified
           (kkt <= 1e-7; the others are reported, not hidden);  fits: 1 + K F;
scores     float64 [L', K, n]: each sample's held-out linear predictor in repeat k, per lambda."""


def check_inputs(expr, label, folds, repeats, alpha):
    """ValueError unless the lasso path can run: perm.check_inputs' conditions (labels 0 and 1 both present, 3 <= n <=
    32768 samples with label 0 or 1, finite expression), 2 <= F <= min(n0, n1) and F <= 100, 1 <= K <= 100 and a
    finite alpha in (0, 1], at most 2^20 genes.  Returns (x, lab) as perm.check_inputs.  Needs no GPU."""
    for name, v, lo, hi in (("the number of folds F", folds, 2, MAX_FOLDS),
                            ("the number of repeats K", repeats, 1, MAX_REPEATS)):
        if int(v) != v or not lo <= int(v) <= hi:
            raise ValueError("lasso: %s must be an integer in [%d, %d], got %r" % (name, lo, hi, v))
    a = float(alpha)
    if not np.isfinite(a) or not 0.0 < a <= 1.0:
        raise ValueError("lasso: alpha must be finite and in (0, 1], got %r" % (alpha,))
    x, lab = perm.check_inputs(expr, label, 1)
    if x.shape[1] > MAX_GENES:
        raise ValueError("lasso: %d genes, at most %d" % (x.shape[1], MAX_GENES))
    n0, n1 = int((lab == 0).sum()), int((lab == 1).sum())
    if folds > min(n0, n1):
        raise ValueError("lasso: F = %d folds need at least F samples of each label, got %d and %d" % (folds, n0, n1))
    return x, lab


def lambda_path(lam_max, n, G):
    """glmnet's 100 lambdas: geometric from lam_max down to ratio lam_max, ratio 0.01 when n < G, else 1e-4."""
    ratio = 0.01 if n < G else 1e-4
    return lam_max * ratio ** (np.arange(N_LAMBDA) / (N_LAMBDA - 1.0))


def top_lasso(entry, entry_abs, p):
    """The first p genes to enter one fit's path: by entry index, then |beta| at entry descending, then gene index.
    Fewer than p when fewer entered."""
    entry = np.asarray(entry).astype(np.int64)
    j = np.nonzero(entry >= 0)[0]
    order = np.lexsort((j, -np.asarray(entry_abs)[j], entry[j]))
    return j[order][:int(p)].astype(np.int32)


def cv_summary(dev, fold, F):
    """(cvm, cvsd, i_min, i_1se) from the held-out deviance terms dev [L, K, n] and the folds [K, n]: cv.glmnet's
    grouped rule with the K F folds as one set of folds."""
    L, K, n = dev.shape
    means, sizes = [], []
    for k in range(K):
        for f in range(F):
            m = fold[k] == f
            sizes.append(m.sum())
            means.append(dev[:, k, m].mean(axis=1))
    means = np.stack(means, axis=1)                    # [L, K F]
    w = np.asarray(sizes, dtype=np.float64)
    cvm = (means * w).sum(axis=1) / w.sum()
    cvsd = np.sqrt(((means - cvm[:, None]) ** 2 * w).sum(axis=1) / w.sum() / (K * F - 1))
    i_min, i_1se = pick(cvm, cvsd)
    return cvm, cvsd, i_min, i_1se


def pick(cvm, cvsd):
    """(i_min, i_1se): the first argmin of cvm, and the smallest index (largest lambda) within one SE of it."""
    i_min = int(np.argmin(cvm))
    i_1se = int(np.nonzero(cvm <= cvm[i_min] + cvsd[i_min])[0][0])
    return i_min, i_1se


def fold_top(res, k, f, p):
    """top_lasso of fold fit (k, f) (global fit 1 + k F + f) at size p, sorted ascending."""
    F = res.auc.shape[2]
    return np.sort(top_lasso(res.entry[1 + k * F + f], res.entry_abs[1 + k * F + f], p))


def nested_lasso(x, lab, res, lists, seed):
    """nested_lasso's held-out AUC [K, F]: for every outer fit (k, f) of --nested-cv on the same splits, top_lasso of
    fold fit (k, f) at the size of that fit's nested list lists[k][f], refit and scored by nested.score_fit.  A fold
    fit in which no gene entered scores NaN."""
    from . import nested
    K, F = res.auc.shape[1:]
    auc = np.full((K, F), np.nan)
    for k in range(K):
        for f in range(F):
            top = fold_top(res, k, f, len(lists[k][f]))
            if top.size:
                auc[k, f] = nested.score_fit(x, lab, res.folds, k, f, top[None, :], seed=seed)[0][0]
    return auc


def summary(res, biomarkers=None, extra=""):
    """The lasso line of the command line."""
    K, F = res.auc.shape[1:]
    line = ("lasso: alpha %g, %d-fold x %d repeats, %d of %d lambdas; lambda_min %.4g (%d genes, CV deviance %.4f, "
            "AUC %.3f), lambda_1se %.4g (%d genes, CV deviance %.4f, AUC %.3f)"
            % (res.alpha, F, K, res.n_lambda, N_LAMBDA, res.lambdas[res.i_min], res.df[res.i_min], res.cvm[res.i_min],
               res.auc_mean[res.i_min], res.lambdas[res.i_1se], res.df[res.i_1se], res.cvm[res.i_1se],
               res.auc_mean[res.i_1se]))
    if biomarkers is not None and len(biomarkers):
        bm = np.asarray(biomarkers)
        top = top_lasso(res.entry[0], res.entry_abs[0], bm.size)
        inter = np.intersect1d(top, bm).size
        jac = inter / float(np.union1d(top, bm).size)
        nz = int((res.beta[res.i_1se][bm] != 0).sum())
        line += "; top_lasso(%d) Jaccard %.3f with the biomarkers; %d biomarkers nonzero at lambda_1se" % (
            top.size, jac, nz)
    line += extra
    total = res.fits * res.n_lambda
    if res.converged < total:
        line += "; %d of %d fits did not certify" % (total - res.converged, total)
    return line


def lasso_cv(expr, label, folds=5, repeats=1, alpha=1.0, seed=0, max_chunk_bytes=None):
    """The lasso / elastic-net path of the label on every gene, cross-validated, on the GPU.

    expr: host float array [samples, genes]; label: one int per sample (0 good, 1 poor; other labels are left out).
    folds F, repeats K: the stratified splits of g2v_sig_folds at seed, the ones signature_cv uses for the same F, K
    and seed.  alpha: the elastic-net mixing in (0, 1] (1 = the lasso).  max_chunk_bytes: bound on the device memory
    of one chunk of fits (default: half the free device memory); the result does not depend on it.  Returns a
    LassoResult; ValueError (before anything is uploaded) on inputs check_inputs refuses, RuntimeError without a
    GPU."""
    x, lab = check_inputs(expr, label, folds, repeats, alpha)
    K, F, alpha = int(repeats), int(folds), float(alpha)
    n, G = x.shape
    fits = 1 + K * F
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
    fold_d = torch.empty((K, n), dtype=torch.int8, device=dev)
    _capi.check(lib.g2v_sig_folds(y_d.data_ptr(), n, K, F, seed, fold_d.data_ptr(), st), "g2v_sig_folds")
    if max_chunk_bytes is None:
        max_chunk_bytes = torch.cuda.mem_get_info(dev)[0] // 2
    # per fit of a chunk: its workspace, entries (10 G bytes) and per-lambda records (24 per lambda)
    per_fit = int(lib.g2v_lasso_workspace_bytes(G, n_pad, 1)) + 10 * G + 24 * N_LAMBDA
    rows = int(max(1, min(fits, int(max_chunk_bytes) // per_fit)))
    ws = torch.empty(int(lib.g2v_lasso_workspace_bytes(G, n_pad, rows)), dtype=torch.uint8, device=dev)
    entry = torch.empty((rows, G), dtype=torch.int16, device=dev)
    entry_abs = torch.empty((rows, G), dtype=torch.float64, device=dev)
    rec = [torch.zeros((rows, N_LAMBDA), dtype=t, device=dev)
           for t in (torch.int32, torch.int32, torch.float64, torch.float64)]          # df, n_iter, dev_ratio, kkt
    path = torch.zeros((N_LAMBDA, G + 1), dtype=torch.float64, device=dev)
    sc_d = torch.zeros((K, n), dtype=torch.float64, device=dev)                   # one lambda's held-out scores
    dv_d = torch.zeros((K, n), dtype=torch.float64, device=dev)
    ctl = torch.zeros(2, dtype=torch.int32, device=dev)
    lam_d = torch.zeros(1, dtype=torch.float64, device=dev)
    ent, ent_abs = np.empty((fits, G), dtype=np.int16), np.empty((fits, G))
    df, n_iter = np.zeros((fits, N_LAMBDA), dtype=np.int32), np.zeros((fits, N_LAMBDA), dtype=np.int32)
    devr, kkt = np.zeros((fits, N_LAMBDA)), np.zeros((fits, N_LAMBDA))
    scores, devi = np.zeros((N_LAMBDA, K, n)), np.zeros((N_LAMBDA, K, n))
    fold = fold_d.cpu().numpy()
    owner = 1 + np.arange(K)[:, None] * F + fold.astype(np.int64)                   # the fold fit holding sample out
    ws_p, X_p, y_p, f_p = ws.data_ptr(), X_d.data_ptr(), y_d.data_ptr(), fold_d.data_ptr()
    lambdas, L = None, N_LAMBDA
    for c0 in range(0, fits, rows):
        nf = min(rows, fits - c0)
        mine = (owner >= c0) & (owner < c0 + nf)
        _capi.check(lib.g2v_lasso_standardise(X_p, G, n, n_pad, y_p, f_p, K, F, c0, nf, ws_p, entry.data_ptr(),
                                              entry_abs.data_ptr(), st), "g2v_lasso_standardise")
        if lambdas is None:                            # the first chunk holds fit 0, which sets the lambdas
            _capi.check(lib.g2v_lasso_grad(X_p, G, n, n_pad, nf, ws_p, 0.0, alpha, st), "g2v_lasso_grad")
            _capi.check(lib.g2v_lasso_lambda_max(G, n_pad, nf, ws_p, alpha, lam_d.data_ptr(), st),
                        "g2v_lasso_lambda_max")
            lambdas = lambda_path(float(lam_d.item()), n, G)
        for k in range(L):
            lam, lam_prev = float(lambdas[k]), float(lambdas[max(k - 1, 0)])
            r = 0
            while True:
                _capi.check(lib.g2v_lasso_grad(X_p, G, n, n_pad, nf, ws_p, lam, alpha, st), "g2v_lasso_grad")
                _capi.check(lib.g2v_lasso_cd(X_p, G, n, n_pad, y_p, nf, ws_p, k, lam, lam_prev, alpha, r,
                                             rec[0].data_ptr(), rec[2].data_ptr(), rec[1].data_ptr(),
                                             rec[3].data_ptr(), entry.data_ptr(), entry_abs.data_ptr(),
                                             path.data_ptr() if c0 == 0 else None, ctl.data_ptr(), st),
                            "g2v_lasso_cd")
                pending, stop0 = (int(v) for v in ctl.cpu().numpy())
                if pending == 0:
                    break
                r += 1
            # the buffers hold one lambda: the kernel writes its row 0, the host keeps this chunk's samples
            _capi.check(lib.g2v_lasso_score(y_p, f_p, n, n_pad, K, F, c0, nf, ws_p, G, 0, sc_d.data_ptr(),
                                            dv_d.data_ptr(), st), "g2v_lasso_score")
            scores[k][mine] = sc_d.cpu().numpy()[mine]
            devi[k][mine] = dv_d.cpu().numpy()[mine]
            if c0 == 0 and stop0 >= 0:                 # fit 0 stopped: the path has stop0 lambdas
                L = stop0
                break
        sl = slice(c0, c0 + nf)
        ent[sl], ent_abs[sl] = entry[:nf].cpu().numpy(), entry_abs[:nf].cpu().numpy()
        df[sl], n_iter[sl] = rec[0][:nf].cpu().numpy(), rec[1][:nf].cpu().numpy()
        devr[sl], kkt[sl] = rec[2][:nf].cpu().numpy(), rec[3][:nf].cpu().numpy()
    del ws
    late = ent >= L                                    # fold fits of the first chunk may have run one lambda more
    ent[late] = -1
    ent_abs[late] = 0.0
    scores, devi = np.ascontiguousarray(scores[:L]), devi[:L]
    s_d = torch.from_numpy(scores).to(dev)
    auc_d = torch.empty((L, K, F), dtype=torch.float64, device=dev)
    acc_d = torch.empty((L, K, F), dtype=torch.float64, device=dev)
    n0, n1 = int((lab == 0).sum()), int((lab == 1).sum())
    cap = -(-n0 // F) + -(-n1 // F)
    _capi.check(lib.g2v_sig_auc(s_d.data_ptr(), y_p, f_p, n, K, F, L, cap, auc_d.data_ptr(), acc_d.data_ptr(), st),
                "g2v_sig_auc")
    auc = auc_d.cpu().numpy()
    cvm, cvsd, i_min, i_1se = cv_summary(devi, fold, F)
    kk = kkt[:, :L]
    return LassoResult(alpha=alpha, lambdas=lambdas[:L].copy(), n_lambda=L, a0=path[:L, 0].cpu().numpy(),
                       beta=path[:L, 1:].cpu().numpy(), df=df[0, :L], dev_ratio=devr[0, :L], cvm=cvm, cvsd=cvsd,
                       auc=auc, auc_mean=auc.reshape(L, K * F).mean(axis=1), i_min=i_min, i_1se=i_1se, folds=fold,
                       entry=ent, entry_abs=ent_abs, n_iter=n_iter[:, :L], kkt=kk, converged=int((kk <= EPS).sum()),
                       fits=fits, scores=scores)
