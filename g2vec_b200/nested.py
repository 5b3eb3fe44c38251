"""Nested cross-validation of the biomarker selection (DESIGN.md §4.34): steps 3-6 rerun on every outer training
fold, the selected list scored on the held-out fold by ridge logistic regression's AUC (Ambroise & McLachlan 2002).

The biomarkers of a run are chosen with every sample's label -- the groups' edge weights, the walks and windows on
those graphs, the CBOW training on the window labels and the t half of the gene score all see it -- so the AUC
``--signature-cv`` reports for them is optimistic.  Here each outer fit (k, f) runs pipeline.select on the training
samples of fold f of repeat k only, with every option of the run, and fits its list (``nested_biomarkers``) and the
top-|t| genes of the same training samples at the same size (``nested_top_t``) on exactly that split.  The test fold's
expression and labels reach neither the selection nor the fit.  The full run's ``biomarkers`` and ``top_t`` are scored
on the same splits, as ``--signature-cv`` scores them: optimism = AUC(biomarkers) - AUC(nested_biomarkers).

Splits: K repeats of stratified F-fold from g2v_sig_folds at the run's seed, the splits of ``--signature-cv`` for the
same F and seed; repeat k's split depends only on (labels, F, seed, k).  Fits and AUC: signature.cv_fits, the device
part of signature.signature_cv, unchanged.  An outer fit is scored as a two-fold row (its test fold 0, the rest 1):
fold 0's fit trains on the same samples in the same order as fit (k, f) of a K x F call, so it gives the same bits;
fold 1's fit is discarded.
"""
from collections import namedtuple

import numpy as np

from . import perm, signature

MAX_FOLDS = signature.MAX_FOLDS        # G2V_SIG_MAX_FOLDS
MAX_REPEATS = signature.MAX_REPEATS    # G2V_SIG_MAX_REPEATS
MAX_SIZE = signature.MAX_SIZE          # G2V_SIG_MAX_SIZE: at most 2 n biomarkers
ROWS = ("nested_biomarkers", "nested_top_t", "biomarkers", "top_t")

NestedResult = namedtuple("NestedResult", "folds n_train n_test n_windows stop_epoch biomarkers auc acc jaccard "
                                          "selected selected_good selected_poor frequency auc_mean auc_sd acc_mean "
                                          "optimism p_random converged n_fits")
NestedResult.__doc__ = """nested_cv's result over the n samples with label 0 or 1; K repeats of F folds.
folds       int8 [K, n]: the test fold of every sample;
n_train, n_test, n_windows, stop_epoch   int64 [K, F]: per outer fit its sample counts, the windows its trainer got
            and the epoch whose vectors it kept (-1 when no epoch ran);
biomarkers  [K][F] lists: each outer fit's sorted gene indices (at most 2 n);
auc, acc    float64 [4, K, F]: per fit the test fold's AUC and accuracy of the rows ROWS: nested_biomarkers,
            nested_top_t (top_t of the training samples at the fit's size), biomarkers and top_t (the full run's);
jaccard     float64 [K, F]: |A & B| / |A | B| of each fit's list A and the full run's B;
selected, selected_good, selected_poor   int64 [G]: per gene, how many outer fits selected it, and from the good and
            from the poor L-group;  frequency: selected / (K F);
auc_mean, acc_mean   float64 [4]: the means over the K F fits;  auc_sd: SD (ddof 1) of the K per-repeat mean AUCs, NaN
            at K = 1;
optimism    auc_mean[biomarkers] - auc_mean[nested_biomarkers];
p_random    (1 + #{random AUC >= nested AUC}) / (R + 1) against the R random rows of --signature-cv on the same
            splits, NaN without them;
converged, n_fits   how many of the n_fits logistic fits met the step rule."""


def check_inputs(expr, label, folds, repeats, p=None):
    """ValueError unless the nested loop can run, before anything is uploaded: perm.check_inputs' conditions (labels 0
    and 1 both present, 3 <= n <= 32768 samples with label 0 or 1, finite expression), 2 <= F <= min(100, n0, n1),
    1 <= K <= 100 and, when given, the largest list 1 <= p <= 128.  Returns (x float64 [n, G], lab [n], used bool [N]).
    Needs no GPU."""
    for name, v, lo, hi in (("the number of folds F", folds, 2, MAX_FOLDS),
                            ("the number of repeats K", repeats, 1, MAX_REPEATS)):
        if int(v) != v or not lo <= int(v) <= hi:
            raise ValueError("%s must be an integer in [%d, %d], got %r" % (name, lo, hi, v))
    x, lab = perm.check_inputs(expr, label, 1)
    n0, n1 = int((lab == 0).sum()), int((lab == 1).sum())
    if folds > min(n0, n1):
        raise ValueError("F = %d folds need at least F samples of each label, got %d and %d" % (folds, n0, n1))
    if p is not None and not 1 <= p <= MAX_SIZE:
        raise ValueError("a signature of %d genes, must be 1 to %d" % (p, MAX_SIZE))
    used = np.isin(np.asarray(label).reshape(-1), (0, 1))
    return x, lab, used


def two_fold_row(fold, k, f):
    """int8 [1, n]: 0 on the samples of test fold f of repeat k, 1 on the others."""
    return np.where(np.asarray(fold)[k] == f, 0, 1).astype(np.int8)[None, :]


def jaccard(a, b):
    """|A & B| / |A | B| of two gene collections (1 for two empty ones)."""
    a, b = set(a), set(b)
    return len(a & b) / len(a | b) if a or b else 1.0


def selection_counts(lists, lgroups, G):
    """Per gene (selected, selected_good, selected_poor) over the outer fits: lists of selected gene indices with the
    fit's L-group array each (a selected gene is in L-group 0 or 1)."""
    sel, good, poor = (np.zeros(G, dtype=np.int64) for _ in range(3))
    for genes, lg in zip(lists, lgroups):
        g = np.asarray(genes, dtype=np.int64)
        sel[g] += 1
        good[g[lg[g] == 0]] += 1
        poor[g[lg[g] == 1]] += 1
    return sel, good, poor


def summarise(auc, acc, random_auc=None):
    """(auc_mean, auc_sd, acc_mean, optimism, p_random) from the per-fit auc and acc [4, K, F] of ROWS; random_auc:
    the mean AUCs of --signature-cv's random rows on the same splits, or None (p_random NaN)."""
    S, K, F = auc.shape
    auc_mean = auc.reshape(S, K * F).mean(axis=1)
    acc_mean = acc.reshape(S, K * F).mean(axis=1)
    auc_sd = auc.mean(axis=2).std(axis=1, ddof=1) if K > 1 else np.full(S, np.nan)
    optimism = float(auc_mean[2] - auc_mean[0])
    p_random = float("nan")
    if random_auc is not None and len(random_auc):
        rnd = np.asarray(random_auc, dtype=np.float64)
        p_random = (1.0 + float((rnd >= auc_mean[0]).sum())) / (rnd.shape[0] + 1.0)
    return auc_mean, auc_sd, acc_mean, optimism, p_random


def fit_line(k, f, K, F, n_train, n_windows, stop_epoch, size, auc_nested, auc_top_t):
    """The progress line of outer fit (k, f), 1-based in the text."""
    return ("nested CV: repeat %d/%d, fold %d/%d: %d training samples, %d windows, stop epoch %d, %d genes: AUC %.3f "
            "(nested biomarkers), %.3f (nested top |t|)" % (k + 1, K, f + 1, F, n_train, n_windows, stop_epoch, size,
                                                            auc_nested, auc_top_t))


def summary(res):
    """The command line's ``nested CV:`` line."""
    K, F = res.n_train.shape
    m = res.auc_mean
    line = ("nested CV: %d-fold x %d repeats, %.1f genes per fit: AUC %.3f (nested biomarkers), %.3f (nested top |t|), "
            "%.3f (biomarkers), %.3f (top |t|); optimism %.3f; mean Jaccard with the biomarkers %.3f"
            % (F, K, float(np.mean([len(b) for row in res.biomarkers for b in row])), m[0], m[1], m[2], m[3],
               res.optimism, float(res.jaccard.mean())))
    if not np.isnan(res.p_random):
        line += "; P_random %.3g" % res.p_random
    if res.converged < res.n_fits:
        line += "; %d of %d fits did not converge" % (res.n_fits - res.converged, res.n_fits)
    return line


def score_fit(x, lab, fold, k, f, head, seed=0):
    """Fit and score the rows of head [H, p] on outer fit (k, f) as a two-fold row: (auc [H], acc [H], converged [H])
    of fold 0.  Only the head's genes are uploaded."""
    cols = np.unique(head)
    row = two_fold_row(fold, k, f)
    n_test = int((row == 0).sum())
    _, _, auc, acc, _, conv, _ = signature.cv_fits(np.ascontiguousarray(x[:, cols]), lab,
                                                   np.searchsorted(cols, head).astype(np.int32), 0, 1, 2, seed,
                                                   fold=row, cap=n_test)
    return auc[:, 0, 0], acc[:, 0, 0], conv[:, 0, 0]


def run_list(genes, biomarkers):
    """The full run's list (gene names) as sorted int32 indices into genes; ValueError unless it holds 1 to 128."""
    pos = {g: i for i, g in enumerate(genes)}
    bm = np.array(sorted(pos[g] for g in biomarkers), dtype=np.int32)
    if not 1 <= bm.shape[0] <= MAX_SIZE:
        raise ValueError("the run selected %d biomarkers, must be 1 to %d" % (bm.shape[0], MAX_SIZE))
    return bm


def select_fit(expr, label, rows, src, dst, genes, args, k, f, on_fit=None):
    """Steps 3-6 of outer fit (k, f) on the expression rows `rows` alone (pipeline.select with every option of args):
    (its pipeline.Selection, its list as sorted int32 indices into genes).  on_fit(k, f, selection) is called before
    the list is checked.  ValueError naming the fit when it cannot train or selects no biomarkers."""
    from . import pipeline
    try:
        sel = pipeline.select(expr[rows], label[rows], src, dst, genes, args)
    except ValueError as e:
        raise ValueError("outer fit repeat %d fold %d (%d training samples): %s"
                         % (k + 1, f + 1, rows.shape[0], e)) from e
    if on_fit is not None:
        on_fit(k, f, sel)
    pos = {g: i for i, g in enumerate(genes)}
    mine = np.array(sorted(pos[g] for g in sel.biomarkers), dtype=np.int32)
    if mine.shape[0] == 0:
        raise ValueError("outer fit repeat %d fold %d selected no biomarkers" % (k + 1, f + 1))
    return sel, mine


def nested_cv(expr, label, src, dst, genes, args, biomarkers, random_auc=None, fold=None, log=None, on_fit=None):
    """Nested cross-validation of the selection, on one GPU.

    expr [N, G] (host, as step 2 leaves it), label per sample (samples with other labels are left out), the step-2
    edges as int32 indices into genes, args: the run's options (cli.parse_arguments; ``--nested-cv`` F,
    ``--nested-cv-repeats`` K, ``--seed`` and every option of steps 3-6).  biomarkers: the full run's list (gene
    names).  random_auc: the mean AUCs of --signature-cv's random rows on the same splits, for P_random.  fold: the
    outer splits int8 [K, n] over the used samples (default: g2v_sig_folds at the seed).  log(line): the progress line
    of every outer fit.  on_fit(k, f, selection): called with each outer fit's pipeline.Selection.  Returns a
    NestedResult; ValueError naming (k, f) when an outer fit cannot train."""
    F, K = int(args.nested_cv), int(args.nested_cv_repeats)
    x, lab, used = check_inputs(expr, label, F, K)
    genes = np.asarray(genes)
    G = len(genes)
    bm = run_list(genes, biomarkers)
    p = len(bm)
    head = np.stack([bm, signature.top_t(x, lab, p)])
    cap = None
    if fold is not None:
        fold = np.ascontiguousarray(fold, dtype=np.int8)
        cap = max(int((fold[k] == f).sum()) for k in range(K) for f in range(F))
    _, fold, auc_full, acc_full, _, conv_full, _ = signature.cv_fits(x, lab, head, 0, K, F, args.seed, fold=fold,
                                                                     cap=cap)
    idx = np.flatnonzero(used)
    expr = np.asarray(expr)
    lab_all = np.asarray(label).reshape(-1)
    auc = np.empty((4, K, F)); acc = np.empty((4, K, F))
    auc[2:], acc[2:] = auc_full, acc_full
    shape = (K, F)
    n_train, n_test, n_windows, stop_epoch = (np.zeros(shape, dtype=np.int64) for _ in range(4))
    jac = np.empty(shape)
    lists, lgroups = [[None] * F for _ in range(K)], []
    converged = int(conv_full.sum())
    for k in range(K):
        for f in range(F):
            train = fold[k] != f
            sel, mine = select_fit(expr, lab_all, idx[train], src, dst, genes, args, k, f, on_fit)
            pair = np.stack([mine, signature.top_t(x[train], lab[train], mine.shape[0])])
            a, c, cv = score_fit(x, lab, fold, k, f, pair, seed=args.seed)
            auc[:2, k, f], acc[:2, k, f] = a, c
            converged += int(cv.sum())
            best = sel.info.get("best_step")
            n_train[k, f], n_test[k, f] = int(train.sum()), int((~train).sum())
            n_windows[k, f], stop_epoch[k, f] = sel.n_windows, -1 if best is None else int(best)
            lists[k][f] = [int(g) for g in mine]
            lgroups.append(np.asarray(sel.lgroup))
            jac[k, f] = jaccard(mine, bm)
            if log is not None:
                log(fit_line(k, f, K, F, n_train[k, f], n_windows[k, f], stop_epoch[k, f], mine.shape[0],
                             auc[0, k, f], auc[1, k, f]))
    sel_n, sel_good, sel_poor = selection_counts([g for row in lists for g in row], lgroups, G)
    auc_mean, auc_sd, acc_mean, optimism, p_random = summarise(auc, acc, random_auc)
    return NestedResult(folds=fold, n_train=n_train, n_test=n_test, n_windows=n_windows, stop_epoch=stop_epoch,
                        biomarkers=lists, auc=auc, acc=acc, jaccard=jac, selected=sel_n, selected_good=sel_good,
                        selected_poor=sel_poor, frequency=sel_n / float(K * F), auc_mean=auc_mean, auc_sd=auc_sd,
                        acc_mean=acc_mean, optimism=optimism, p_random=p_random, converged=converged,
                        n_fits=4 * K * F)
