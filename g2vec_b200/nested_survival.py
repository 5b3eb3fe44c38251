"""Nested cross-validation of the biomarker selection against survival (DESIGN.md §4.36): steps 3-6 rerun without
each event-stratified test fold of the samples with a survival record, the selected list scored on the held-out fold
by ridge Cox regression's Harrell's C (Ambroise & McLachlan 2002; pre-validation, Tibshirani & Efron 2002).

The biomarkers of a run are chosen with every sample -- the groups' edge weights, the walks and windows, the CBOW
training and the t half of the gene score -- so the C ``--survival-cv`` reports for them, and the Kaplan-Meier split
of its _risk.txt, are optimistic.  Here each outer fit (k, f) runs pipeline.select on every expression sample outside
the test fold T (the samples without a record and those of other labels included, as the main run passes them), with
every option of the run, and fits three lists of the fit's size on the survival samples outside T: the selected list
(``nested_biomarkers``), the top-|t| genes of the training samples (``nested_top_t``) and their top Cox-score genes
(``nested_top_z``).  Nothing of T -- expression, label or record -- reaches the selection or the fit.  The full run's
``biomarkers``, ``top_t`` and ``top_z`` are scored on the same splits, as ``--survival-cv`` scores them: optimism =
C(biomarkers) - C(nested_biomarkers).  Each survival sample's out-of-fold eta of the nested biomarkers, averaged over
the repeats, gives the pre-validated nested risk groups (survival_cv.risk_groups).

Splits: K repeats of F-fold stratified by event status, g2v_sig_folds on the event flags in time order at the run's
seed: the splits of ``--survival-cv`` for the same F, K and seed; repeat k's split depends only on (records, F, seed,
k).  Fits and C: survival_cv.cox_fits, unchanged.  An outer fit is scored as a two-fold row over the time order (its
test fold 0, the rest 1): fold 0's fit trains on the same samples in the same order as fit (k, f) of a K x F call, so
it gives the same bits; fold 1's fit is discarded.
"""
from collections import namedtuple

import numpy as np

from . import nested, signature, survival, survival_cv

MAX_FOLDS = survival_cv.MAX_FOLDS        # G2V_SIG_MAX_FOLDS
MAX_REPEATS = survival_cv.MAX_REPEATS    # G2V_SIG_MAX_REPEATS
MAX_SIZE = survival_cv.MAX_SIZE          # G2V_SIG_MAX_SIZE: at most 2 n biomarkers
ROWS = ("nested_biomarkers", "nested_top_t", "nested_top_z", "biomarkers", "top_t", "top_z")

NestedSurvivalResult = namedtuple("NestedSurvivalResult", "folds n_train n_test n_test_events n_windows stop_epoch "
                                                          "biomarkers counts c jaccard selected selected_good "
                                                          "selected_poor frequency c_mean c_sd optimism p_random "
                                                          "converged n_fits scores risk group logrank_z logrank_p hr "
                                                          "hr_low hr_high")
NestedSurvivalResult.__doc__ = """nested_survival_cv's result over the n samples with a survival record, in their input
order; K repeats of F folds.
folds       int8 [K, n]: the test fold of every survival sample;
n_train, n_test, n_test_events, n_windows, stop_epoch   int64 [K, F]: per outer fit the expression samples its
            selection saw, the samples and the events of its test fold, the windows its trainer got and the epoch whose
            vectors it kept (-1 when no epoch ran);  n_train + n_test is every expression sample;
biomarkers  [K][F] lists: each outer fit's sorted gene indices (at most 2 n);
counts      int64 [6, K, F, 3]: per fit of the rows ROWS the test fold's comparable, concordant and tied pairs;
c           float64 [6, K, F]: their Harrell's C (NaN without a comparable pair): nested_biomarkers, nested_top_t
            (top_t of the training samples at the fit's size), nested_top_z (survival.rank_genes of the training
            survival samples at that size), then the full run's biomarkers, top_t and top_z;
jaccard     float64 [K, F]: |A & B| / |A | B| of each fit's list A and the full run's B;
selected, selected_good, selected_poor   int64 [G]: per gene, how many outer fits selected it, and from the good and
            from the poor L-group;  frequency: selected / (K F);
c_mean      float64 [6]: the mean over the fits that have a comparable pair;  c_sd: SD (ddof 1) of the K per-repeat
            means, NaN at K = 1 (survival_cv.summarise);
optimism    c_mean[biomarkers] - c_mean[nested_biomarkers];
p_random    (1 + #{random C >= nested C}) / (R + 1) against the R random rows of --survival-cv on the same splits, NaN
            without them;
converged, n_fits   how many of the n_fits = 6 K F Cox fits met the step rule;
scores      float64 [K, n]: the out-of-fold eta of every survival sample from the nested_biomarkers fit whose test fold
            holds it;
risk, group, logrank_z, logrank_p, hr, hr_low, hr_high   as SurvivalCVResult's, with one row: the pre-validated risk
            of the nested biomarkers (the mean of scores over the repeats), its median split, log-rank test and hazard
            ratio."""


def check_inputs(expr, time, event, label, folds, repeats, p=None):
    """ValueError unless the nested loop can run, before anything is uploaded: survival_cv.check_inputs' conditions
    (3 to 32768 samples with a finite time and at least one event, finite expression, labels that allow top_t,
    2 <= F <= 100, 1 <= K <= 100, F at most the events and at most half the survival samples) and, when given, the
    largest list 1 <= p <= min(128, G).  Returns (x float64 [n, G], time [n], event int64 [n], used bool [N]).  Needs
    no GPU."""
    return survival_cv.check_inputs(expr, time, event, label, 1 if p is None else p, 1, folds, repeats)


def score_fit(x, time, event, fold, k, f, head, seed=0):
    """Fit and score the rows of head [H, p] on outer fit (k, f) as a two-fold row: (counts int64 [H, 3], eta [H,
    n_test] of the test samples in their order, converged [H]) of fold 0.  Only the head's genes are uploaded."""
    cols = np.unique(head)
    row = nested.two_fold_row(fold, k, f)
    test = row[0] == 0
    _, _, counts, _, conv, _, scores = survival_cv.cox_fits(np.ascontiguousarray(x[:, cols]), time, event,
                                                            np.searchsorted(cols, head).astype(np.int32), 0, 1, 2,
                                                            seed, fold=row, cap=int(test.sum()))
    return counts[:, 0, 0], scores[:, 0, test], conv[:, 0, 0]


def summarise(c, random_c=None):
    """(c_mean, c_sd, optimism, p_random) from the per-fit C [6, K, F] of ROWS; random_c: the mean C of --survival-cv's
    random rows on the same splits, or None (p_random NaN)."""
    c_mean, c_sd, _ = survival_cv.summarise(c, c.shape[0], 0)
    optimism = float(c_mean[3] - c_mean[0])
    p_random = float("nan")
    if random_c is not None and len(random_c):
        rnd = np.asarray(random_c, dtype=np.float64)
        p_random = (1.0 + float((rnd >= c_mean[0]).sum())) / (rnd.shape[0] + 1.0)
    return c_mean, c_sd, optimism, p_random


def fit_line(k, f, K, F, n_train, n_test, n_test_events, n_windows, stop_epoch, size, c):
    """The progress line of outer fit (k, f), 1-based in the text; c: its three nested C."""
    return ("nested survival CV: repeat %d/%d, fold %d/%d: %d training samples, %d test samples (%d events), %d "
            "windows, stop epoch %d, %d genes: C %.3f (nested biomarkers), %.3f (nested top |t|), %.3f (nested top "
            "|Z|)" % (k + 1, K, f + 1, F, n_train, n_test, n_test_events, n_windows, stop_epoch, size, c[0], c[1],
                      c[2]))


def summary(res):
    """The command line's ``nested survival CV:`` line."""
    K, F = res.n_train.shape
    m = res.c_mean
    line = ("nested survival CV: %d-fold x %d repeats, %.1f genes per fit: C %.3f (nested biomarkers), %.3f (nested "
            "top |t|), %.3f (nested top |Z|), %.3f (biomarkers), %.3f (top |t|), %.3f (top |Z|); optimism %.3f; mean "
            "Jaccard with the biomarkers %.3f; nested risk groups: log-rank Z = %.4f, P = %.4g, HR %.3f (%.3f, %.3f)"
            % (F, K, float(np.mean([len(b) for row in res.biomarkers for b in row])), m[0], m[1], m[2], m[3], m[4],
               m[5], res.optimism, float(res.jaccard.mean()), res.logrank_z[0], res.logrank_p[0], res.hr[0],
               res.hr_low[0], res.hr_high[0]))
    if not np.isnan(res.p_random):
        line += "; P_random %.3g" % res.p_random
    if res.converged < res.n_fits:
        line += "; %d of %d fits did not converge" % (res.n_fits - res.converged, res.n_fits)
    return line


def nested_survival_cv(expr, label, time, event, src, dst, genes, args, biomarkers, random_c=None, fold=None, log=None,
                       on_fit=None):
    """Nested cross-validation of the selection against survival, on one GPU.

    expr [N, G] (host, as step 2 leaves it), label per sample, time and event per sample as survival.match_survival
    gives them (time NaN where there is no record), the step-2 edges as int32 indices into genes, args: the run's
    options (cli.parse_arguments; ``--nested-survival-cv`` F, ``--nested-survival-cv-repeats`` K, ``--seed`` and every
    option of steps 3-6).  biomarkers: the full run's list (gene names).  random_c: the mean C of --survival-cv's
    random rows on the same splits, for P_random.  fold: the outer splits int8 [K, n] over the survival samples
    (default: g2v_sig_folds on the event flags at the seed).  log(line): the progress line of every outer fit.
    on_fit(k, f, selection): called with each outer fit's pipeline.Selection.  Returns a NestedSurvivalResult;
    ValueError naming (k, f) when an outer fit cannot train."""
    F, K = int(args.nested_survival_cv), int(args.nested_survival_cv_repeats)
    x, t, e, used = check_inputs(expr, time, event, label, F, K)
    genes = np.asarray(genes)
    G = len(genes)
    bm = nested.run_list(genes, biomarkers)
    p = len(bm)
    expr = np.asarray(expr)
    lab_all = np.asarray(label).reshape(-1)
    tz = np.sort(survival.rank_genes(x, t, e)[:p]).astype(np.int32)
    head = np.stack([bm, signature.top_t(expr, lab_all, p), tz])
    cap = None
    if fold is not None:
        fold = np.ascontiguousarray(fold, dtype=np.int8)
        cap = max(int((fold[k] == f).sum()) for k in range(K) for f in range(F))
    _, fold, counts_full, _, conv_full, _, _ = survival_cv.cox_fits(x, t, e, head, 0, K, F, args.seed, fold=fold,
                                                                    cap=cap)
    idx = np.flatnonzero(used)
    N, n = expr.shape[0], x.shape[0]
    counts = np.empty((len(ROWS), K, F, 3), dtype=np.int64)
    counts[3:] = counts_full
    c = np.empty((len(ROWS), K, F))
    c[3:] = survival_cv.concordance(counts_full)
    shape = (K, F)
    n_train, n_test, n_test_events, n_windows, stop_epoch = (np.zeros(shape, dtype=np.int64) for _ in range(5))
    jac = np.empty(shape)
    scores = np.empty((K, n))
    lists, lgroups = [[None] * F for _ in range(K)], []
    converged = int(conv_full.sum())
    for k in range(K):
        for f in range(F):
            test = fold[k] == f                        # over the survival samples
            in_test = np.zeros(N, dtype=bool)
            in_test[idx[test]] = True
            rows = np.flatnonzero(~in_test)            # every expression sample outside T
            sel, mine = nested.select_fit(expr, lab_all, rows, src, dst, genes, args, k, f, on_fit)
            q = mine.shape[0]
            tr = ~test
            three = np.stack([mine, signature.top_t(expr[rows], lab_all[rows], q),
                              np.sort(survival.rank_genes(x[tr], t[tr], e[tr])[:q]).astype(np.int32)])
            counts[:3, k, f], eta, cv = score_fit(x, t, e, fold, k, f, three, seed=args.seed)
            c[:3, k, f] = survival_cv.concordance(counts[:3, k, f])
            scores[k, test] = eta[0]
            converged += int(cv.sum())
            best = sel.info.get("best_step")
            n_train[k, f], n_test[k, f], n_test_events[k, f] = rows.shape[0], int(test.sum()), int(e[test].sum())
            n_windows[k, f], stop_epoch[k, f] = sel.n_windows, -1 if best is None else int(best)
            lists[k][f] = [int(g) for g in mine]
            lgroups.append(np.asarray(sel.lgroup))
            jac[k, f] = nested.jaccard(mine, bm)
            if log is not None:
                log(fit_line(k, f, K, F, n_train[k, f], n_test[k, f], n_test_events[k, f], n_windows[k, f],
                             stop_epoch[k, f], q, c[:3, k, f]))
    sel_n, sel_good, sel_poor = nested.selection_counts([g for row in lists for g in row], lgroups, G)
    c_mean, c_sd, optimism, p_random = summarise(c, random_c)
    risk, group, z, pz, hr, lo, hi = survival_cv.risk_groups(scores, t, e)
    one = lambda v: np.array([v], dtype=np.float64)
    return NestedSurvivalResult(folds=fold, n_train=n_train, n_test=n_test, n_test_events=n_test_events,
                                n_windows=n_windows, stop_epoch=stop_epoch, biomarkers=lists, counts=counts, c=c,
                                jaccard=jac, selected=sel_n, selected_good=sel_good, selected_poor=sel_poor,
                                frequency=sel_n / float(K * F), c_mean=c_mean, c_sd=c_sd, optimism=optimism,
                                p_random=p_random, converged=converged, n_fits=len(ROWS) * K * F, scores=scores,
                                risk=risk[None, :], group=group[None, :], logrank_z=one(z), logrank_p=one(pz),
                                hr=one(hr), hr_low=one(lo), hr_high=one(hi))
