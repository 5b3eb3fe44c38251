"""The G2Vec command line, kept as the drop-in shell around the two H100 hot paths.

Same positionals, options, progress banners and output files as /root/reference/G2Vec.py
(parse_arguments :505-518, main :11-119, writers :127-131,159-165,203-215).  Steps 1, 2, 5, 6, 7 are
plain Python/NumPy/scikit-learn as in the reference (step 5 runs on the GPU with ``--kmeans-restarts``);
step 3 runs g2vec_b200.walks on the GPU and step 4 g2vec_b200.cbow.  Two documented differences: ``--epoch`` is honoured as the cap on optimizer
steps (the reference parses it, :515, and then loops ``range(500)``, :262 -- the default 500 is the
reference behaviour), and ``--seed`` (default 0) seeds the walk sampler, the path glue, the split and the
initial vectors (the reference is unseeded).

``--patience K`` (default 1, the reference's rule) keeps training through up to K-1 epochs in a row whose validation
accuracy is below the best so far, stops at the K-th, and writes the vectors of the best epoch (ties: the later one);
the ``Epoch(stop)`` line then names the best epoch, and a run that reaches ``--epoch`` with a better earlier epoch
prints an ``Epoch(best)`` line (DESIGN.md §4.15).

``--lr-patience K`` (default 0: a fixed learning rate) multiplies the learning rate by ``--lr-factor`` (default 0.1), but
not below ``--min-lr`` (default 0), after K epochs in a row whose validation accuracy is not above the best so far (a
tie does not count as better), and prints a ``learning rate ->`` line among the epoch lines for every cut (Keras
ReduceLROnPlateau; DESIGN.md §4.17).  It works with the Adam optimizers only, and is independent of ``--patience``.

``--weight-decay λ`` (default 0: off; finite, 0 <= λ < 1) is decoupled weight decay, AdamW / SGDW: every optimizer
step first shrinks each weight it updates to w - λ·w, then takes the usual step (DESIGN.md §4.18).  It acts per
optimizer step (once per batch with ``--batch``), is not scaled by the learning rate or ``--lr-patience``, and adds
nothing to the logged loss.  ``adam``, ``sgd`` and ``--algo rank1`` decay every gene vector every step; ``lazy_adam``
decays only the vectors of the genes a batch gathered.

``--monitor val_loss`` (default ``val_acc``) makes ``--patience`` and ``--lr-patience`` decide on the validation loss
instead of the validation accuracy: an epoch whose loss is not above the best so far is the new best (ties: the later
one), and only a loss below the best counts as an improvement for the learning rate.  The loss is the mean sigmoid
cross-entropy of the validation windows, each term capped at 64, summed exactly in fixed point (2^-24), so for given
vectors it does not depend on how the windows are split over the GPUs; the epoch lines then show it as ``LOSS[val]`` after ``ACC[tr]`` (DESIGN.md §4.19).

``--class-weight balanced`` or ``--class-weight W0,W1`` (default off) weights the training loss per label, Keras
``fit(class_weight=...)``: a window of label y counts W_y times in the step's mean (DESIGN.md §4.20).  ``balanced`` is
sklearn's rule, W_y = n / (2 n_y) over the training windows, so each label carries half of the loss however the paths
fall between the groups; a training split with one label only is an error.  The weights must be finite and > 0.  The
run prints a ``class weights:`` line after ``Start training``; the accuracies, ``LOSS[val]``, ``--patience`` and
``--lr-patience`` keep their meanings, and the logged training loss is the weighted one.

``--correlation {pearson,spearman,bicor}`` (default ``pearson``, the reference's) chooses the coefficient of step 3's
edge weights, and ``--min-corr T`` (default 0.5, finite, 0 <= T < 1) the cutoff: an edge is kept in a group's graph iff
its |coefficient| over that group's samples is > T (DESIGN.md §4.22).  ``spearman`` is Pearson's coefficient of the
average ranks (ties share the mean of their positions); ``bicor`` is the biweight midcorrelation of WGCNA
(Langfelder & Horvath 2012), falling back to Pearson for a gene whose median absolute deviation is 0.  Both need
finite expression values and at most 32768 samples per group.  A run with either option off its default prints a
``correlation:`` line under the step-3 banner.

``--permutations B`` (default 0: off) adds a label-permutation test of every gene's t statistic (DESIGN.md §4.24):
B permutations of the good / poor labels (Fisher-Yates, seeded by ``--seed``; the observed labelling is not among
them) give each gene a raw p-value P = (1 + #{|t_b| >= |t|}) / (B + 1), Westfall & Young's step-down maxT adjusted
p-value P_maxT (Ge, Dudoit & Speed 2003, as multtest's mt.maxT) and the Benjamini-Hochberg q-value Q of P.  The
family is every gene of the analysis.  The inputs are checked before step 3 (labels 0 and 1 both present, 3 to 32768
samples with label 0 or 1, finite expression values, 1 <= B <= 2^24), the test runs on the GPU after step 6 (on rank 0
only under torchrun) and prints a ``permutation test:`` line, and step 7 also writes RESULT_NAME_pvalues.txt: per gene,
in the order of _lgroups.txt, its L-group, T (the observed |t|, ``inf`` at perfect separation, where step 6's t-score
is 0), P, P_maxT, Q and whether it is a biomarker.  P, P_maxT and Q do not depend on training.

``--neighbors K`` (default 0: off; 0 <= K <= 64) adds the K nearest genes of every gene in the learned embedding, by
exact cosine on the GPU (DESIGN.md §4.25).  The searched genes are those in at least one good or poor random path (the
``n_genes`` count of step 3): the others keep their random initial vectors.  A run whose paths hold K genes or fewer
stops with an ``ERROR`` after step 3, before training.  After step 6 (on rank 0 only under torchrun) the run prints a
``neighbors:`` line with the share of (gene, neighbour) pairs in the same L-group, and step 7 also writes
RESULT_NAME_neighbors.txt: per searched gene, in the order of _lgroups.txt, K rows of its L-group, the rank 1..K, the
neighbour, its L-group and the cosine, nearest first (equal cosines by the neighbour's position in _lgroups.txt).

``--kmeans-restarts R`` (default 0: off, step 5 is scikit-learn's ``KMeans(3, random_state=0)`` as in the reference;
0 <= R <= 1024) finds the L-groups on the GPU with the best of R k-means++ restarts instead (DESIGN.md §4.26): restart r
is seeded by ``--seed`` and r, every restart runs Lloyd's iterations (at most 300) in exact float64, and the one of
lowest inertia names the L-groups by the same rule.  Each gene's agreement is the share of restarts that put it in the
best restart's cluster, after matching every restart's cluster labels to the best one's.  A run with fewer than 3
common genes stops with an ``ERROR`` before step 3.  Step 5 (on rank 0 only under torchrun) prints a ``k-means:`` line,
and step 7 also writes RESULT_NAME_kmeans.txt: per gene, in the order of _lgroups.txt, its L-group and agreement,
followed by the same line.  Steps 6 and 7, ``--permutations`` and ``--neighbors`` use these L-groups.

``--tsne P`` (default 0: off; otherwise a finite perplexity, 1 <= P <= 1000) adds an exact 2-D t-SNE map of the genes in
paths (the same genes as ``--neighbors``) from their learned vectors, on the GPU in float64 (DESIGN.md §4.27):
scikit-learn's exact method with its defaults (early exaggeration 12 for 250 iterations, learning rate
max(n / 48, 50), PCA initialisation), always 1000 iterations, the same bits for the same vectors.  A run whose paths hold
P genes or fewer, or more than 32768, stops with an ``ERROR`` after step 3, before training.  After step 6 (on rank 0
only under torchrun) the run prints a ``t-SNE:`` line with the final KL divergence, and step 7 also writes
RESULT_NAME_tsne.txt: per gene in paths, in the order of _lgroups.txt, its L-group and its X and Y in the map.

``--gene-sets FILE`` (default off) adds gene-set enrichment of the good / poor contrast, phenotype-permutation GSEA
(Subramanian et al. 2005) on the GPU (DESIGN.md §4.28), for the sets of the GMT file FILE (one set per line: name,
description, genes, tab-separated).  The ranking metric is each gene's point-biserial correlation with the poor label
(label 1), the weight its absolute value; ``--gene-set-permutations B`` (default 1000, 1 <= B <= 2^20) label
permutations, seeded by ``--seed`` and the same as ``--permutations`` makes for the same B, give each set its ES, NES,
nominal P, FDR q and FWER p.  ``--gene-set-size MIN,MAX`` (default 15,500; 1 <= MIN <= MAX <= 4096) keeps the sets
with MIN to MAX genes in the analysis (the common genes of step 2).  The file and the inputs are checked after step 2,
where the run prints a ``gene sets:`` line or stops with an ``ERROR``; after step 6 (on rank 0 only under torchrun) it
prints a ``gene-set test:`` line, and step 7 also writes RESULT_NAME_gsea.txt: per kept set, in the file's order, its
size, ES, NES, P, FDR_Q, FWER_P (``nan`` when the needed side of the null is empty), how many of its genes are
biomarkers, and its leading-edge genes in rank order.  None of these depend on training.

``--signature-cv R`` (default 0: off; 0 <= R <= 65536) adds a cross-validated test of whether the biomarkers predict
the good / poor label, on the GPU (DESIGN.md §4.29): ridge logistic regression (scikit-learn's
``LogisticRegression(C=1.0)`` objective, features standardised on each training fold) over ``--signature-repeats K``
(default 10, 1 <= K <= 100) repeats of stratified ``--signature-folds F``-fold splits (default 5, 2 <= F <= 100, and F
at most the number of samples of either label), the same splits for every signature.  The biomarkers are compared with
the same number of genes of largest |t| (``top_t``) and with R random signatures of that size (Floyd's sampling, seeded
by ``--seed``).  The biomarkers and ``top_t`` were both chosen with every sample's label, so their AUCs are optimistic
and comparable with each other; the random signatures are not selected, and P_random = (1 + #{random AUC >= AUC}) /
(R + 1) says how often one does at least as well.  For the AUC of the selection itself, rerun inside every fold, see
``--nested-cv``, which scores on the same splits for the same F, K and ``--seed``.  It needs ``-n`` <= 64 (at most 128 biomarkers).  The inputs are checked after step 2, where the run
stops with an ``ERROR`` if they are refused; after step 6 (on rank 0 only under torchrun) it prints a ``signature CV:``
line, and step 7 also writes RESULT_NAME_signature.txt: per signature (biomarkers, top_t, random_1 .. random_R) its
size, mean AUC over the K F fits, the SD of the K per-repeat AUCs, mean accuracy, P_random (``nan`` on random rows)
and how many of its genes are biomarkers.

``--diff-coexpression B`` (default 0: off; 1 <= B <= 2^20) adds a label-permutation test of differential co-expression
for every pair of genes joined in the network, on the GPU (DESIGN.md §4.30): the pairs are the distinct unordered
gene pairs of step 2's edges (self-loops dropped, direction and duplicates collapsed), and each pair's Pearson
correlations over the good and the poor samples are compared by Fisher's z.  The test is always Pearson, whatever
``--correlation`` chose for step 3's graphs.  B label permutations, seeded by ``--seed`` and the same as
``--permutations`` makes for the same B, give each pair a raw P, Westfall & Young's step-down maxT P_maxT over the
pairs and the Benjamini-Hochberg Q.  The inputs are checked after step 2 (at least 4 samples of each label, at most
32768 in all, finite expression values, 1 to 2^26 pairs), where the run stops with an ``ERROR`` if they are refused;
after step 6 (on rank 0 only under torchrun) it prints a ``differential co-expression:`` line (the last two counts are
over the pairs with Q <= 0.05), and step 7 also writes RESULT_NAME_diffcoex.txt: per pair, ordered by the two genes'
positions in _lgroups.txt, R_good, R_poor, Z, P, P_maxT, Q, whether step 3 kept the pair in the good and in the poor
graph (either direction), and how many of its two genes are biomarkers.  None of these depend on training.

``--survival FILE`` (default off) adds a permutation Cox score test of every gene against patient survival, on the GPU
(DESIGN.md §4.31).  FILE is tab-delimited with a header line and the columns SAMPLE, TIME (a finite number >= 0, any
unit) and EVENT (1 for death or relapse, 0 for censored); further columns are ignored, rows of samples not in the
expression file are ignored, and a sample whose TIME or EVENT is NA or empty is left out of the test.  Each gene's
statistic is the Cox partial-likelihood score test at beta = 0 with Breslow ties (the log-rank test for a 0/1
covariate without tied event times); Z > 0 means higher expression goes with higher hazard.
``--survival-permutations B`` (default 1000, 1 <= B <= 2^20) permutations of the expression against the records, seeded
by ``--seed`` and drawn as ``--permutations`` draws its rows, give each gene a raw P, Westfall & Young's step-down maxT
P_maxT over the genes and the Benjamini-Hochberg Q.  The file and the inputs are checked after step 2 (every
expression sample has exactly one row, at least 3 and at most 32768 samples used, at least one event), where the run
prints a ``survival:`` line or stops with an ``ERROR``; after step 6 (on rank 0 only under torchrun) it prints a
``survival:`` line that also gives the score test of the good / poor label itself, and step 7 also writes
RESULT_NAME_survival.txt: per gene, in the order of _lgroups.txt, its L-group, Z, P_score (the asymptotic
erfc(|Z| / sqrt(2))), P, P_maxT, Q and whether it is a biomarker.  None of these depend on training.

``--survival-cv R`` (default 0: off; 0 <= R <= 65536, needs ``--survival``) adds a cross-validated test of whether the
biomarkers predict survival, on the GPU (DESIGN.md §4.33), over the samples ``--survival`` uses: ridge Cox regression
(Breslow ties, penalty |beta|^2 / 2 on the summed partial likelihood, features standardised on each training fold)
over ``--survival-cv-repeats K`` (default 10, 1 <= K <= 100) repeats of ``--survival-cv-folds F``-fold splits (default
5, 2 <= F <= 100, F at most the number of events and at most half the samples) stratified by event status, scored on
each test fold with Harrell's C.  The biomarkers are compared with the same number of genes of largest |t| (``top_t``,
as ``--signature-cv`` picks them), of largest Cox score statistic (``top_z``, the ranking of ``--survival``) and with
R random signatures of that size (the random signatures of ``--signature-cv`` for the same ``--seed``); P_random =
(1 + #{random C >= C}) / (R + 1).  Each sample's out-of-fold risk, averaged over the repeats, splits the samples at the
median into a high- and a low-risk group (pre-validation), with a log-rank test and the hazard ratio of the high-risk
group.  It needs ``-n`` <= 64.  The inputs are checked after step 2, where the run stops with an ``ERROR`` if they are
refused; after step 6 (on rank 0 only under torchrun) it prints a ``survival CV:`` line, and step 7 also writes
RESULT_NAME_survival_cv.txt: per signature (biomarkers, top_t, top_z, random_1 .. random_R) its size, mean C over the
fits, the SD of the K per-repeat means, P_random, the log-rank Z and P and the hazard ratio with its 95 % CI of the
risk groups (``nan`` on random rows) and how many of its genes are biomarkers; and RESULT_NAME_risk.txt: per sample
used, in the expression file's order, its time, event, the biomarkers' pre-validated risk and group (1 = high risk),
ready for a Kaplan-Meier plot.  The biomarkers were chosen with every sample's label, so their C is optimistic;
nested re-selection is ``--nested-cv`` for the good / poor label and ``--nested-survival-cv`` for survival.

``--nested-cv F`` (default 0: off; 2 <= F <= 100, F at most the number of samples of either label) adds nested
cross-validation of the selection itself, on one GPU (DESIGN.md §4.34): over ``--nested-cv-repeats K`` (default 1,
1 <= K <= 100) repeats of stratified F-fold splits of the samples with label 0 or 1 -- the splits ``--signature-cv``
uses for the same F, K and ``--seed``; repeat k's split depends only on the labels, F, the seed and k -- steps 3 to 6
run again on every outer training fold alone, with every option of the run, and the fit's list (``nested
biomarkers``, at most 2 ``-n`` genes) and the same number of genes of largest |t| over those training samples
(``nested top_t``) are scored on the held-out fold by ``--signature-cv``'s ridge logistic regression.  The test fold's
expression and labels reach neither the selection nor the fit, so the nested AUC is the honest estimate of how well
the selection generalises (Ambroise & McLachlan 2002); the run's own biomarkers and ``top_t`` are scored on the same
splits, and the optimism is AUC(biomarkers) - AUC(nested biomarkers).  With ``--signature-cv R`` at the same F and K,
P_random = (1 + #{random AUC >= nested AUC}) / (R + 1).  It needs ``-n`` <= 64 and refuses torchrun.  The inputs are
checked after step 2, where the run stops with an ``ERROR`` if they are refused; after step 6 every outer fit prints
one line (repeat, fold, training samples, windows, stop epoch, its two AUCs; its steps 3 and 4 print nothing), an
outer fit that cannot train stops the run with an ``ERROR`` naming it, and the run prints a ``nested CV:`` line.  Step
7 also writes RESULT_NAME_nested_cv.txt: per outer fit its repeat, fold, N_train, N_test, N_windows, Stop_epoch,
Size, AUC and accuracy of the nested biomarkers and of nested top_t, the AUC of the biomarkers and of top_t, the
Jaccard overlap with the biomarkers and its list, then the ``nested CV:`` line; and RESULT_NAME_nested_selection.txt:
per gene, in the order of _lgroups.txt, its L-group, whether it is a biomarker, how many outer fits selected it, that
count's share of the K F fits, and how many selected it from the good and from the poor L-group.

``--nested-survival-cv F`` (default 0: off; 2 <= F <= 100, F at most the number of events and at most half the samples
with a record; needs ``--survival``) is the same nested cross-validation against survival, on one GPU (DESIGN.md
§4.36): over ``--nested-survival-cv-repeats K`` (default 1, 1 <= K <= 100) repeats of F-fold splits of the samples
``--survival`` uses, stratified by event status -- the splits ``--survival-cv`` uses for the same F, K and ``--seed`` --
steps 3 to 6 run again, with every option of the run, on every expression sample outside the test fold (samples
without a record and of other labels included, as the main run takes them), and the fit's list, the same number of
genes of largest |t| (``nested top_t``) and of largest Cox score statistic (``nested top_z``) over those training
samples are scored on the held-out fold by ``--survival-cv``'s ridge Cox regression and Harrell's C.  The test fold's
expression, labels and records reach neither the selection nor the fit.  The run's own biomarkers, ``top_t`` and
``top_z`` are scored on the same splits, and the optimism is C(biomarkers) - C(nested biomarkers); with
``--survival-cv R`` at the same F and K, P_random = (1 + #{random C >= nested C}) / (R + 1).  Each sample's
out-of-fold risk from the nested biomarkers, averaged over the repeats, splits the samples at the median into
pre-validated risk groups, with a log-rank test and a hazard ratio: the Kaplan-Meier split to report.  It needs ``-n``
<= 64 and refuses torchrun.  The inputs are checked after step 2, where the run stops with an ``ERROR`` if they are
refused; after step 6 (and after ``--nested-cv``'s lines) every outer fit prints one line, an outer fit that cannot
train stops the run with an ``ERROR`` naming it, and the run prints a ``nested survival CV:`` line.  Step 7 also writes
RESULT_NAME_nested_survival_cv.txt: per outer fit its repeat, fold, N_train, N_test, N_test_events, N_windows,
Stop_epoch, Size, the C of the nested biomarkers, nested top_t and nested top_z, the C of the biomarkers, top_t and
top_z, the Jaccard overlap with the biomarkers and its list, then the ``nested survival CV:`` line;
RESULT_NAME_nested_survival_risk.txt, laid out as _risk.txt, with the nested biomarkers' pre-validated risk; and
RESULT_NAME_nested_survival_selection.txt, laid out as _nested_selection.txt.

``--netrank B`` (default 0: off; 1 <= B <= 2^20) adds network-propagated gene scores, NetRank (Winter et al. 2012;
GeneRank, Morrison et al. 2005), with a label-permutation test, on the GPU (DESIGN.md §4.35).  The network is the
distinct unordered gene pairs of step 2's edges, as ``--diff-coexpression`` takes them, unweighted; each gene's seed is
its |point-biserial r| with the good / poor label (the |t| of ``--permutations`` on another scale), and the score is
personalised PageRank of the seeds, x_j = (1 - d) s_j + d sum over the neighbours i of x_i / deg_i, iterated from
x = s until d^T <= 1e-12, with ``--netrank-damping d`` (default 0.5; finite, 0 <= d <= 0.95; 0 gives the seeds
themselves).  A gene with little difference of its own can rank high when its neighbourhood differs.  B label
permutations, seeded by ``--seed`` and the same as ``--permutations`` makes for the same B, give each gene a raw P and
the Benjamini-Hochberg Q (no maxT: the null spread of a score grows with the gene's degree).  ``top_netrank`` is the
genes of highest score (ties by position), as many as there are biomarkers.  The inputs are checked after step 2
(labels 0 and 1 both present, 3 to 32768 samples with label 0 or 1, finite expression values, 1 to 2^26 pairs), where
the run stops with an ``ERROR`` if they are refused; after step 6 (on rank 0 only under torchrun) it prints a
``netrank:`` line (how many genes have Q <= 0.05 and how many of those are biomarkers, and the Jaccard overlap of
``top_netrank`` with the biomarkers; with ``--signature-cv`` also the cross-validated AUC of ``top_netrank`` on the same
splits, beside the biomarkers'), and step 7 also writes RESULT_NAME_netrank.txt: per gene, in the order of _lgroups.txt, its L-group, degree, seed S, score,
rank (1 = highest score), P, Q and whether it is a biomarker, followed by the same line.  None of these depend on
training.

``--lasso F`` (default 0: off; 2 <= F <= 100, F at most the number of samples of either label) adds the lasso /
elastic-net logistic baseline on the GPU (DESIGN.md §4.37): glmnet's path of the good / poor label on every gene (the
samples with label 0 or 1, the matrix ``top_t`` uses), each gene standardised over the fit's training samples, with
mixing ``--lasso-alpha α`` (default 1 = the lasso; finite, 0 < α <= 1), on the full cohort and on every training fold
of ``--lasso-repeats K`` (default 1, 1 <= K <= 100) repeats of stratified F-fold splits (``--signature-cv``'s splits
for the same F, K and ``--seed``).  The 100 lambdas are glmnet's; the path stops at a deviance ratio of 0.999, a rise
below 1e-5 of it, or 512 genes entered.  Every solution is checked against the KKT conditions in float64.  The
held-out binomial deviance gives cv.glmnet's lambda_min and lambda_1se; ``top_lasso`` is the genes in the order they
enter the full-cohort path.  The inputs are checked after step 2, where the run stops with an ``ERROR`` if they are
refused.  After step 6 (and after ``--nested-cv``'s lines) it prints a ``lasso:`` line: α, F x K, the path length,
lambda_min and lambda_1se with their gene counts, CV deviance and CV AUC, the Jaccard overlap of ``top_lasso`` at the
biomarkers' size with the biomarkers, how many biomarkers are nonzero at lambda_1se; with ``--signature-cv`` the AUC
of ``top_lasso`` on its splits beside the biomarkers'; with ``--nested-cv`` at the same F and K the mean AUC of
``nested_lasso`` (``top_lasso`` of each training fold at the size of that fold's nested list, scored as the nested
lists are) beside ``nested_biomarkers``; and how many solutions did not certify.  Step 7 also writes
RESULT_NAME_lasso.txt: per gene, in the order of _lgroups.txt, its L-group, entry index on the full-cohort path (-1 if
never), beta at lambda_min and at lambda_1se, the fraction of fold fits in which it had entered by lambda_1se's index
and whether it is a biomarker, followed by the line; and RESULT_NAME_lasso_path.txt: per lambda index its lambda, df,
deviance ratio, CV deviance and SE, mean CV AUC and the marks of lambda_min and lambda_1se.

Which runs are bit-reproducible (same input, same seed, one GPU: the same three output files):
- ``--deterministic`` with ``--algo rows``: every optimizer, full batch or ``--batch``, with or without
  ``--reshuffle`` or ``--class-weight``, at every table size (DESIGN.md §4.13); ``--class-weight 1,1`` writes the
  files of the same run without it;
- ``--algo rank1`` with a full batch.
Without ``--deterministic`` the rows trainer adds some floating-point values in an order the GPU picks (the
output-layer gradient every step; the gradient rows with ``--batch`` and adam/sgd, or on tables larger than the
L2), so two runs can differ in the last bits of the vectors, and rarely in the stop step or the biomarkers.
Runs on several GPUs are not bit-reproducible.
"""
import argparse
import sys
from math import sqrt

import numpy as np


def parse_arguments(argv=None):
    p = argparse.ArgumentParser(
        description="G2Vec (H100-native hot paths): network-based identification of prognostic gene "
                    "signatures. Same interface as mathcom/G2Vec G2Vec.py.")
    p.add_argument('EXPRESSION_FILE', type=str, help="Tab-delimited file for gene expression profiles.")
    p.add_argument('CLINICAL_FILE', type=str, help="Tab-delimited clinical file. LABEL=0: good prognosis, 1: poor.")
    p.add_argument('NETWORK_FILE', type=str, help="Tab-delimited file for the gene interaction network.")
    p.add_argument('RESULT_NAME', type=str, help="Prefix of *_biomarkers.txt, *_lgroups.txt and *_vectors.txt")
    p.add_argument('-p', '--lenPath', type=int, default=80, help='')
    p.add_argument('-r', '--numRepetition', type=int, default=10, help='')
    p.add_argument('-s', '--sizeHiddenlayer', type=int, default=128, help='')
    p.add_argument('-e', '--epoch', type=int, default=500, help='')
    p.add_argument('-l', '--learningRate', type=float, default=0.005, help='')
    p.add_argument('-n', '--numBiomarker', type=int, default=50, help='')
    p.add_argument('--seed', type=int, default=0, help='seed of the walk sampler, the split and the init')
    p.add_argument('--walk-q', type=float, default=1.0, metavar='Q',
                   help="node2vec's in-out parameter of the random walks, in [1/256, 256]: Q > 1 keeps a walk near the "
                        "previous gene's neighbours (BFS-like), Q < 1 moves it away (DFS-like); 1 (default) = the "
                        "reference's first-order walk.  There is no return parameter: the walks never revisit a gene")
    p.add_argument('--correlation', choices=['pearson', 'spearman', 'bicor'], default='pearson',
                   help="coefficient of the edge weights: 'pearson' (default, the reference's), 'spearman' (Pearson "
                        "on average ranks) or 'bicor' (biweight midcorrelation); spearman and bicor take at most "
                        "32768 samples per group and finite expression values")
    p.add_argument('--min-corr', type=float, default=0.5, metavar='T',
                   help="an edge is kept iff its |coefficient| over the group's samples is > T, 0 <= T < 1 "
                        "(default 0.5, the reference's cutoff)")
    p.add_argument('--algo', choices=['rows', 'rank1'], default='rows',
                   help="CBOW kernels: 'rows' = embedding-row gather/scatter (default), 'rank1' = collapsed, "
                        "bit-reproducible trainer; same results to fp32 rounding")
    p.add_argument('--batch', type=int, default=0,
                   help="windows per optimizer step; 0 (default) = full batch, one step per epoch as the reference")
    p.add_argument('--optimizer', choices=['adam', 'sgd', 'lazy_adam'], default='adam',
                   help="'adam' = TF1 AdamOptimizer (the reference's), 'sgd', or 'lazy_adam' = TF1 LazyAdam: a step "
                        "updates only the rows of the genes its batch gathered (rows, one GPU)")
    p.add_argument('--reshuffle', action='store_true',
                   help="with --batch: train every epoch after the first on a new pseudo-random order of the training "
                        "windows (seeded by --seed and the epoch) instead of the same batches every epoch")
    p.add_argument('--deterministic', action='store_true',
                   help="bit-reproducible training on one GPU: every floating-point sum of a step in a fixed order "
                        "(rows: any optimizer and batch size; rank1: full batch only); somewhat slower")
    p.add_argument('--patience', type=int, default=1,
                   help="early stopping: stop after this many epochs in a row whose validation accuracy is below the "
                        "best so far, and write the vectors of the best epoch; 1 (default) = the reference's rule, "
                        "stop at the first drop")
    p.add_argument('--lr-patience', type=int, default=0,
                   help="reduce the learning rate on a plateau: after this many epochs in a row without a validation "
                        "accuracy above the best so far, multiply it by --lr-factor; 0 (default) = a fixed rate")
    p.add_argument('--lr-factor', type=float, default=0.1,
                   help="with --lr-patience: the factor in (0, 1) the learning rate is multiplied by (default 0.1)")
    p.add_argument('--min-lr', type=float, default=0.0,
                   help="with --lr-patience: the learning rate is never cut below this (default 0)")
    p.add_argument('--weight-decay', type=float, default=0.0,
                   help="decoupled weight decay (AdamW / SGDW): every optimizer step first shrinks each weight it "
                        "updates by this fraction, in [0, 1); 0 (default) = off")
    p.add_argument('--monitor', choices=['val_acc', 'val_loss'], default='val_acc',
                   help="what --patience and --lr-patience decide on: 'val_acc' (default) = the validation accuracy, "
                        "'val_loss' = the validation loss (lower is better), also printed as LOSS[val] on the epoch "
                        "lines")
    p.add_argument('--class-weight', type=str, default=None, metavar='{balanced | W0,W1}',
                   help="weights of the label-0 and label-1 windows in the training loss: 'balanced' = n / (2 n_y) "
                        "from the training windows, or two finite numbers > 0; default off")
    p.add_argument('--permutations', type=int, default=0, metavar='B',
                   help="label-permutation test of every gene's t statistic with B permutations (1 <= B <= 2^24): "
                        "raw, step-down maxT and Benjamini-Hochberg p-values in RESULT_NAME_pvalues.txt; 0 (default) "
                        "= off")
    p.add_argument('--neighbors', type=int, default=0, metavar='K',
                   help="the K nearest genes (0 <= K <= 64) of every gene in the random paths by cosine of the "
                        "learned vectors, in RESULT_NAME_neighbors.txt; 0 (default) = off")
    p.add_argument('--kmeans-restarts', type=int, default=0, metavar='R',
                   help="find the L-groups with the best of R k-means++ restarts on the GPU (0 <= R <= 1024, seeded "
                        "by --seed) and write each gene's agreement across them to RESULT_NAME_kmeans.txt; 0 (default) "
                        "= scikit-learn's KMeans(3, random_state=0)")
    p.add_argument('--tsne', type=float, default=0.0, metavar='P',
                   help="an exact 2-D t-SNE map on the GPU of the genes in the random paths with perplexity P "
                        "(1 <= P <= 1000), in RESULT_NAME_tsne.txt; 0 (default) = off")
    p.add_argument('--gene-sets', type=str, default=None, metavar='FILE',
                   help="gene-set enrichment (phenotype-permutation GSEA) of the good / poor contrast for the sets "
                        "of the GMT file FILE, in RESULT_NAME_gsea.txt; default off")
    p.add_argument('--gene-set-permutations', type=int, default=1000, metavar='B',
                   help="with --gene-sets: label permutations of the gene-set test, 1 <= B <= 2^20 (default 1000)")
    p.add_argument('--gene-set-size', type=str, default='15,500', metavar='MIN,MAX',
                   help="with --gene-sets: keep the sets with MIN to MAX genes in the analysis, 1 <= MIN <= MAX <= "
                        "4096 (default 15,500)")
    p.add_argument('--signature-cv', type=int, default=0, metavar='R',
                   help="cross-validated AUC of the biomarkers against the top-|t| genes and R random signatures of "
                        "the same size (0 <= R <= 65536), in RESULT_NAME_signature.txt; 0 (default) = off")
    p.add_argument('--signature-folds', type=int, default=5, metavar='F',
                   help="with --signature-cv: stratified folds per repeat, 2 <= F <= 100 (default 5)")
    p.add_argument('--signature-repeats', type=int, default=10, metavar='K',
                   help="with --signature-cv: repeats of the fold split, 1 <= K <= 100 (default 10)")
    p.add_argument('--diff-coexpression', type=int, default=0, metavar='B',
                   help="label-permutation test of differential co-expression (Pearson, Fisher's z) of every gene pair "
                        "of the network with B permutations (1 <= B <= 2^20): raw, step-down maxT and "
                        "Benjamini-Hochberg p-values in RESULT_NAME_diffcoex.txt; 0 (default) = off")
    p.add_argument('--survival', type=str, default=None, metavar='FILE',
                   help="permutation Cox score test (Breslow ties) of every gene against the survival times of FILE "
                        "(tab-delimited SAMPLE, TIME, EVENT with a header line), in RESULT_NAME_survival.txt; default "
                        "off")
    p.add_argument('--survival-permutations', type=int, default=1000, metavar='B',
                   help="with --survival: permutations of the expression against the records, 1 <= B <= 2^20 "
                        "(default 1000)")
    p.add_argument('--survival-cv', type=int, default=0, metavar='R',
                   help="with --survival: cross-validated Harrell's C of ridge Cox fits of the biomarkers against the "
                        "top-|t| genes, the top-|Z| genes and R random signatures of the same size (0 <= R <= 65536), "
                        "in RESULT_NAME_survival_cv.txt, and the biomarkers' pre-validated risk groups in "
                        "RESULT_NAME_risk.txt; 0 (default) = off")
    p.add_argument('--survival-cv-folds', type=int, default=5, metavar='F',
                   help="with --survival-cv: folds per repeat, stratified by event, 2 <= F <= 100 (default 5)")
    p.add_argument('--survival-cv-repeats', type=int, default=10, metavar='K',
                   help="with --survival-cv: repeats of the fold split, 1 <= K <= 100 (default 10)")
    p.add_argument('--nested-cv', type=int, default=0, metavar='F',
                   help="nested cross-validation of the selection: steps 3-6 rerun on every training fold of "
                        "stratified F-fold splits (2 <= F <= 100) and the list's ridge logistic AUC on the held-out "
                        "fold, in RESULT_NAME_nested_cv.txt and RESULT_NAME_nested_selection.txt; 0 (default) = off")
    p.add_argument('--nested-cv-repeats', type=int, default=1, metavar='K',
                   help="with --nested-cv: repeats of the fold split, 1 <= K <= 100 (default 1)")
    p.add_argument('--nested-survival-cv', type=int, default=0, metavar='F',
                   help="with --survival: nested cross-validation of the selection against survival: steps 3-6 rerun "
                        "without every test fold of F-fold splits stratified by event (2 <= F <= 100) and the list's "
                        "ridge Cox C on the held-out fold, in RESULT_NAME_nested_survival_cv.txt, "
                        "RESULT_NAME_nested_survival_risk.txt and RESULT_NAME_nested_survival_selection.txt; 0 "
                        "(default) = off")
    p.add_argument('--nested-survival-cv-repeats', type=int, default=1, metavar='K',
                   help="with --nested-survival-cv: repeats of the fold split, 1 <= K <= 100 (default 1)")
    p.add_argument('--netrank', type=int, default=0, metavar='B',
                   help="network-propagated gene scores (NetRank: personalised PageRank of each gene's |r| with the "
                        "label over the network) with a label-permutation test of B permutations (1 <= B <= 2^20): P "
                        "and Benjamini-Hochberg Q in RESULT_NAME_netrank.txt; 0 (default) = off")
    p.add_argument('--netrank-damping', type=float, default=0.5, metavar='d',
                   help="with --netrank: the damping d, a finite number in [0, 0.95] (default 0.5; 0 = no propagation)")
    p.add_argument('--lasso', type=int, default=0, metavar='F',
                   help="lasso / elastic-net logistic baseline on every gene: glmnet's path on the cohort and on every "
                        "training fold of F-fold splits (2 <= F <= 100), lambda_min and lambda_1se by CV deviance, in "
                        "RESULT_NAME_lasso.txt and RESULT_NAME_lasso_path.txt; 0 (default) = off")
    p.add_argument('--lasso-repeats', type=int, default=1, metavar='K',
                   help="with --lasso: repeats of the fold split, 1 <= K <= 100 (default 1)")
    p.add_argument('--lasso-alpha', type=float, default=1.0, metavar='ALPHA',
                   help="with --lasso: the elastic-net mixing, a finite number in (0, 1] (default 1 = the lasso)")
    args = p.parse_args(argv)
    if not (np.isfinite(args.walk_q) and 1.0 / 256.0 <= args.walk_q <= 256.0):
        p.error("--walk-q must be a finite number in [1/256, 256]")
    if not (np.isfinite(args.min_corr) and 0.0 <= args.min_corr < 1.0):
        p.error("--min-corr must be a finite number with 0 <= T < 1")
    if args.class_weight is not None:
        args.class_weight = _parse_class_weight(args.class_weight, p)
    if not 0.0 <= float(np.float32(args.weight_decay)) < 1.0:
        p.error("--weight-decay must be a finite number with 0 <= weight-decay < 1")
    if not 0 <= args.permutations <= 1 << 24:
        p.error("--permutations must be an integer in [0, 2^24]")
    if not 1 <= args.gene_set_permutations <= 1 << 20:
        p.error("--gene-set-permutations must be an integer in [1, 2^20]")
    args.gene_set_size = _parse_gene_set_size(args.gene_set_size, p)
    if not 0 <= args.diff_coexpression <= 1 << 20:
        p.error("--diff-coexpression must be an integer in [0, 2^20]")
    if not 1 <= args.survival_permutations <= 1 << 20:
        p.error("--survival-permutations must be an integer in [1, 2^20]")
    if not 0 <= args.signature_cv <= 1 << 16:
        p.error("--signature-cv must be an integer in [0, 65536]")
    if not 2 <= args.signature_folds <= 100:
        p.error("--signature-folds must be an integer in [2, 100]")
    if not 1 <= args.signature_repeats <= 100:
        p.error("--signature-repeats must be an integer in [1, 100]")
    if args.signature_cv and args.numBiomarker > 64:
        p.error("--signature-cv needs -n <= 64: a signature has at most 128 genes")
    if not 0 <= args.survival_cv <= 1 << 16:
        p.error("--survival-cv must be an integer in [0, 65536]")
    if not 2 <= args.survival_cv_folds <= 100:
        p.error("--survival-cv-folds must be an integer in [2, 100]")
    if not 1 <= args.survival_cv_repeats <= 100:
        p.error("--survival-cv-repeats must be an integer in [1, 100]")
    if args.survival_cv and args.survival is None:
        p.error("--survival-cv needs --survival FILE")
    if args.survival_cv and args.numBiomarker > 64:
        p.error("--survival-cv needs -n <= 64: a signature has at most 128 genes")
    if not (args.nested_cv == 0 or 2 <= args.nested_cv <= 100):
        p.error("--nested-cv must be 0 (off) or an integer in [2, 100]")
    if not 1 <= args.nested_cv_repeats <= 100:
        p.error("--nested-cv-repeats must be an integer in [1, 100]")
    if args.nested_cv and args.numBiomarker > 64:
        p.error("--nested-cv needs -n <= 64: a signature has at most 128 genes")
    if not (args.nested_survival_cv == 0 or 2 <= args.nested_survival_cv <= 100):
        p.error("--nested-survival-cv must be 0 (off) or an integer in [2, 100]")
    if not 1 <= args.nested_survival_cv_repeats <= 100:
        p.error("--nested-survival-cv-repeats must be an integer in [1, 100]")
    if args.nested_survival_cv and args.survival is None:
        p.error("--nested-survival-cv needs --survival FILE")
    if args.nested_survival_cv and args.numBiomarker > 64:
        p.error("--nested-survival-cv needs -n <= 64: a signature has at most 128 genes")
    if not (args.lasso == 0 or 2 <= args.lasso <= 100):
        p.error("--lasso must be 0 (off) or an integer in [2, 100]")
    if not 1 <= args.lasso_repeats <= 100:
        p.error("--lasso-repeats must be an integer in [1, 100]")
    if not (np.isfinite(args.lasso_alpha) and 0.0 < args.lasso_alpha <= 1.0):
        p.error("--lasso-alpha must be a finite number in (0, 1]")
    if not 0 <= args.netrank <= 1 << 20:
        p.error("--netrank must be an integer in [0, 2^20]")
    if not (np.isfinite(args.netrank_damping) and 0.0 <= args.netrank_damping <= 0.95):
        p.error("--netrank-damping must be a finite number in [0, 0.95]")
    if not 0 <= args.neighbors <= 64:
        p.error("--neighbors must be an integer in [0, 64]")
    if not 0 <= args.kmeans_restarts <= 1024:
        p.error("--kmeans-restarts must be an integer in [0, 1024]")
    if not (args.tsne == 0 or (np.isfinite(args.tsne) and 1.0 <= args.tsne <= 1000.0)):
        p.error("--tsne must be 0 (off) or a finite perplexity in [1, 1000]")
    if args.patience < 1:
        p.error("--patience must be an integer >= 1")
    if args.lr_patience < 0:
        p.error("--lr-patience must be an integer >= 0")
    if not 0.0 < float(np.float32(args.lr_factor)) < 1.0:
        p.error("--lr-factor must be in (0, 1)")
    if not 0.0 <= args.min_lr < float("inf"):
        p.error("--min-lr must be a finite number >= 0")
    if args.lr_patience > 0 and args.optimizer == 'sgd':
        p.error("--lr-patience needs --optimizer adam or lazy_adam")
    if args.reshuffle and args.batch <= 0:
        p.error("--reshuffle needs mini-batches (--batch B with B > 0)")
    if args.deterministic and args.algo == 'rank1' and args.batch > 0:
        p.error("--deterministic with --algo rank1 needs a full batch (--batch 0)")
    return args


def _parse_class_weight(text, p):
    """'balanced', or 'W0,W1' as the pair of float32 weights (finite, > 0 in float32); anything else is p.error."""
    if text == 'balanced':
        return text
    parts = text.split(',')
    try:
        if len(parts) != 2:
            raise ValueError
        with np.errstate(over='ignore', under='ignore'):
            w = tuple(np.float32(float(x)) for x in parts)
    except ValueError:
        w = None
    if w is None or not all(np.isfinite(x) and x > 0 for x in w):
        p.error("--class-weight must be 'balanced' or W0,W1: two numbers that are finite and > 0 in float32")
    return tuple(float(x) for x in w)


def _parse_gene_set_size(text, p):
    """'MIN,MAX' -> (MIN, MAX), two integers with 1 <= MIN <= MAX <= 4096; anything else is p.error."""
    try:
        lo, hi = (int(x) for x in text.split(','))
    except ValueError:
        lo = hi = 0
    if not 1 <= lo <= hi <= 4096:
        p.error("--gene-set-size must be MIN,MAX: two integers with 1 <= MIN <= MAX <= 4096")
    return lo, hi


# ----------------------------------------------------------------------------------- step 1: I/O
def _rows(path):
    with open(path) as f:
        return [ln.rstrip().split('\t') for ln in f]


def load_data(path):
    """Expression TSV: header = samples, rows = genes -> expr float32 [samples, genes] (G2Vec.py:478-503)."""
    rows = _rows(path)
    sample = np.array(rows[0][1:])
    gene = np.array([r[0] for r in rows[1:]])
    expr = np.array([r[1:] for r in rows[1:]], dtype=np.float32).T
    return {'sample': sample, 'expr': expr, 'gene': gene}


def load_clinical(path):
    """sample -> int label, header skipped (G2Vec.py:436-453)."""
    return {r[0]: int(r[1]) for r in _rows(path)[1:]}


def load_network(path):
    """Directed edge list [src, dest] and the gene set, header skipped (G2Vec.py:455-476)."""
    edges = _rows(path)[1:]
    genes = set()
    for e in edges:
        genes.add(e[0]); genes.add(e[1])
    return {'edge': edges, 'gene': genes}


# ------------------------------------------------------------------------- step 2: preprocessing
def match_labels(clinical, samples):
    try:
        return np.array([clinical[s] for s in samples])
    except KeyError:
        print('ERROR: There is a mismatched sample between expression data and clinical data. '
              'Please check sample names')
        sys.exit(1)


def restrict(data, network):
    """Sorted common gene list; edges with both ends in it; expression columns (G2Vec.py:393-426)."""
    common = sorted(set(network['gene']) & set(data['gene']))
    cs = set(common)
    edges = [e for e in network['edge'] if e[0] in cs and e[1] in cs]
    pos = {g: i for i, g in enumerate(data['gene'])}
    cols = [pos[g] for g in common]
    data = dict(data, expr=data['expr'][:, cols], gene=np.array(common))
    return data, {'edge': edges, 'gene': cs}


# ------------------------------------------------------------------------------ step 5: L-groups
def find_lgroups(mat, gene_names, geneFreq):
    """KMeans(3, random_state=0) on the vectors, named by kmeans.name_lgroups: largest cluster -> 2 (other); of the
    remaining two clusters the reference compares good/poor gene-frequency votes (G2Vec.py:167-200).  In the reference
    ``freqIdx`` is a Python list, so ``freqIdx==0`` is the scalar False and both votes are always 0
    (:172,186-187): the outcome is therefore always good = second remaining cluster, poor = first.  That
    behaviour is reproduced here so the output files match."""
    from sklearn.cluster import KMeans
    from .kmeans import name_lgroups
    return name_lgroups(KMeans(n_clusters=3, random_state=0).fit(mat).labels_)


# ------------------------------------------------------------------------------- step 6: scoring
def minmax(x, lo=0., hi=1.):
    return (hi - lo) / (x.max() - x.min()) * (x - x.min()) + lo


def tscore(a, b):
    """abs pooled-variance t statistic between two samples (G2Vec.py:138-149)."""
    na, nb = len(a), len(b)
    sa, sb = a.std(ddof=1), b.std(ddof=1)
    d1 = sqrt(((float(na) - 1.) * sa * sa + (float(nb) - 1.) * sb * sb) / float(na + nb - 2))
    d2 = sqrt(1. / float(na) + 1. / float(nb))
    if d1 > 0. and d2 > 0.:
        return abs((a.mean() - b.mean()) / d1 / d2)
    return 0.


def tscores(expr, label):
    out = np.zeros(expr.shape[1], dtype=np.float32)
    g, p = label == 0, label == 1
    for i in range(expr.shape[1]):
        out[i] = tscore(expr[g, i], expr[p, i])
    return out


# ------------------------------------------------------------------------------- step 7: writers
def write_biomarkers(prefix, genes):
    with open(prefix + "_biomarkers.txt", 'w') as f:
        f.write("GeneSymbol\n")
        f.writelines('%s\n' % g for g in genes)


def write_lgroups(prefix, lgroup, genes):
    with open(prefix + "_lgroups.txt", 'w') as f:
        f.write('GeneSymbol\tLgroup(0:good,1:poor,2:other)\n')
        f.writelines('%s\t%d\n' % (g, k) for g, k in zip(genes, lgroup))


def write_pvalues(prefix, genes, lgroup, res, biomarkers):
    """One row per gene in the order of _lgroups.txt: L-group, T, P, P_maxT, Q of a perm.PermResult, biomarker 0/1."""
    bm = set(biomarkers)
    with open(prefix + "_pvalues.txt", 'w') as f:
        f.write('GeneSymbol\tLgroup(0:good,1:poor,2:other)\tT\tP\tP_maxT\tQ\tBiomarker\n')
        f.writelines('%s\t%d\t%.6f\t%.6g\t%.6g\t%.6g\t%d\n' % (g, k, t, pv, pm, qv, g in bm)
                     for g, k, t, pv, pm, qv in zip(genes, lgroup, res.T, res.P, res.P_maxT, res.Q))


def write_neighbors(prefix, genes, lgroup, sub, idx, sim):
    """K rows per searched gene (sub: their indices in genes, ascending): L-group, rank 1..K, the neighbour (idx holds
    positions in sub), its L-group and the cosine."""
    with open(prefix + "_neighbors.txt", 'w') as f:
        f.write('GeneSymbol\tLgroup(0:good,1:poor,2:other)\tRank\tNeighbor\tNeighborLgroup\tCosine\n')
        for g, row, srow in zip(sub, idx, sim):
            f.writelines('%s\t%d\t%d\t%s\t%d\t%.6f\n' % (genes[g], lgroup[g], r + 1, genes[sub[j]], lgroup[sub[j]], s)
                         for r, (j, s) in enumerate(zip(row, srow)))


def write_kmeans(prefix, genes, res):
    """One row per gene in the order of _lgroups.txt: its L-group and agreement (a kmeans.KMeansResult), then the
    k-means line."""
    from .kmeans import summary
    with open(prefix + "_kmeans.txt", 'w') as f:
        f.write('GeneSymbol\tLgroup(0:good,1:poor,2:other)\tAgreement\n')
        f.writelines('%s\t%d\t%.6f\n' % (g, k, a) for g, k, a in zip(genes, res.lgroups, res.agreement))
        f.write(summary(res) + '\n')


def write_tsne(prefix, genes, lgroup, sub, Y):
    """One row per gene in paths (sub: their indices in genes, ascending): its L-group and its map coordinates."""
    with open(prefix + "_tsne.txt", 'w') as f:
        f.write('GeneSymbol\tLgroup(0:good,1:poor,2:other)\tX\tY\n')
        f.writelines('%s\t%d\t%.6f\t%.6f\n' % (genes[g], lgroup[g], x, y) for g, (x, y) in zip(sub, Y))


def write_gsea(prefix, genes, res, biomarkers):
    """One row per kept gene set (a gsea.GseaResult): size, ES, NES, P, FDR_Q, FWER_P, how many of its genes are
    biomarkers, and its leading-edge genes in rank order, comma-separated."""
    bm = set(biomarkers)
    with open(prefix + "_gsea.txt", 'w') as f:
        f.write('GeneSet\tSize\tES\tNES\tP\tFDR_Q\tFWER_P\tBiomarkers\tLeadingEdge\n')
        for i, name in enumerate(res.name):
            f.write('%s\t%d\t%.6f\t%.6f\t%.6g\t%.6g\t%.6g\t%d\t%s\n'
                    % (name, res.size[i], res.ES[i], res.NES[i], res.P[i], res.FDR[i], res.FWER[i],
                       sum(genes[g] in bm for g in res.members[i]), ','.join(genes[g] for g in res.leading_edge[i])))


def write_signature(prefix, genes, res, biomarkers):
    """One row per signature of a signature.SignatureResult: size, AUC, AUC_SD, accuracy, P_random (nan on the random
    rows) and how many of its genes are biomarkers."""
    bm = set(biomarkers)
    p_random = list(res.p_random) + [float("nan")] * (len(res.names) - 2)
    with open(prefix + "_signature.txt", 'w') as f:
        f.write('Signature\tSize\tAUC\tAUC_SD\tAccuracy\tP_random\tBiomarkers\n')
        for i, name in enumerate(res.names):
            f.write('%s\t%d\t%.6f\t%.6f\t%.6f\t%.6g\t%d\n'
                    % (name, res.genes.shape[1], res.auc_mean[i], res.auc_sd[i], res.acc_mean[i], p_random[i],
                       sum(genes[g] in bm for g in res.genes[i])))


def write_diffcoex(prefix, genes, res, in_good, in_poor, biomarkers):
    """One row per pair of a diffcoex.DiffCoexResult in pair order: R_good, R_poor, Z, P, P_maxT, Q, whether the pair is
    in step 3's good and poor graphs (0/1), and how many of its genes are biomarkers (0..2)."""
    with open(prefix + "_diffcoex.txt", 'w') as f:
        f.write('Gene1\tGene2\tR_good\tR_poor\tZ\tP\tP_maxT\tQ\tInGood\tInPoor\tBiomarkers\n')
        f.writelines('%s\t%s\t%.6f\t%.6f\t%.6f\t%.6g\t%.6g\t%.6g\t%d\t%d\t%d\n'
                     % (genes[i], genes[j], rg, rp, z, pv, pm, qv, a, b, c)
                     for (i, j), rg, rp, z, pv, pm, qv, a, b, c
                     in zip(res.pairs, res.R_good, res.R_poor, res.Z, res.P, res.P_maxT, res.Q, in_good, in_poor,
                            biomarkers))


def write_survival(prefix, genes, lgroup, res, biomarkers):
    """One row per gene in the order of _lgroups.txt: L-group, Z, P_score, P, P_maxT, Q of a survival.SurvivalResult,
    biomarker 0/1."""
    bm = set(biomarkers)
    with open(prefix + "_survival.txt", 'w') as f:
        f.write('GeneSymbol\tLgroup(0:good,1:poor,2:other)\tZ\tP_score\tP\tP_maxT\tQ\tBiomarker\n')
        f.writelines('%s\t%d\t%.6f\t%.6g\t%.6g\t%.6g\t%.6g\t%d\n' % (g, k, z, ps, pv, pm, qv, g in bm)
                     for g, k, z, ps, pv, pm, qv in zip(genes, lgroup, res.Z, res.P_score, res.P, res.P_maxT, res.Q))


def write_survival_cv(prefix, genes, res, biomarkers):
    """One row per signature of a survival_cv.SurvivalCVResult: size, C, C_SD, P_random, the log-rank Z and P and the
    hazard ratio with its 95 % CI of the risk groups (nan on the random rows), and how many of its genes are
    biomarkers."""
    bm = set(biomarkers)
    nan = [float("nan")] * (len(res.names) - 3)
    cols = [list(a) + nan for a in (res.p_random, res.logrank_z, res.logrank_p, res.hr, res.hr_low, res.hr_high)]
    with open(prefix + "_survival_cv.txt", 'w') as f:
        f.write('Signature\tSize\tC\tC_SD\tP_random\tLogRank_Z\tLogRank_P\tHR\tHR_Low\tHR_High\tBiomarkers\n')
        for i, name in enumerate(res.names):
            f.write('%s\t%d\t%.6f\t%.6f\t%.6g\t%.6f\t%.6g\t%.6g\t%.6g\t%.6g\t%d\n'
                    % ((name, res.genes.shape[1], res.c_mean[i], res.c_sd[i]) + tuple(c[i] for c in cols)
                       + (sum(genes[g] in bm for g in res.genes[i]),)))


def write_risk(prefix, samples, time, event, res, suffix="_risk.txt"):
    """One row per sample of the survival CV, in expression order: time, event, the pre-validated risk and risk group
    (1 = high) of res's first row (the biomarkers of a survival_cv.SurvivalCVResult, the nested biomarkers of a
    nested_survival.NestedSurvivalResult)."""
    with open(prefix + suffix, 'w') as f:
        f.write('SAMPLE\tTIME\tEVENT\tRISK\tGROUP\n')
        f.writelines('%s\t%.10g\t%d\t%.6f\t%d\n' % (s, t, e, r, g)
                     for s, t, e, r, g in zip(samples, time, event, res.risk[0], res.group[0]))


def write_nested_cv(prefix, genes, res):
    """One row per outer fit of a nested.NestedResult (repeat-major, 1-based): its sizes, windows, stop epoch, list
    size, the AUC and accuracy of its list and of top_t at that size, the full run's biomarkers' and top_t's AUC on
    the same fold, the Jaccard overlap with the full run's list and the list itself; then the nested CV line."""
    from .nested import summary
    K, F = res.n_train.shape
    with open(prefix + "_nested_cv.txt", 'w') as f:
        f.write('Repeat\tFold\tN_train\tN_test\tN_windows\tStop_epoch\tSize\tAUC_nested\tACC_nested\tAUC_nested_top_t\t'
                'ACC_nested_top_t\tAUC_biomarkers\tAUC_top_t\tJaccard\tBiomarkers\n')
        for k in range(K):
            for j in range(F):
                bm = res.biomarkers[k][j]
                f.write('%d\t%d\t%d\t%d\t%d\t%d\t%d\t%.6f\t%.6f\t%.6f\t%.6f\t%.6f\t%.6f\t%.6f\t%s\n'
                        % (k + 1, j + 1, res.n_train[k, j], res.n_test[k, j], res.n_windows[k, j], res.stop_epoch[k, j],
                           len(bm), res.auc[0, k, j], res.acc[0, k, j], res.auc[1, k, j], res.acc[1, k, j],
                           res.auc[2, k, j], res.auc[3, k, j], res.jaccard[k, j], ','.join(genes[g] for g in bm)))
        f.write(summary(res) + '\n')


def write_nested_selection(prefix, genes, lgroup, res, biomarkers, suffix="_nested_selection.txt"):
    """One row per gene in the order of _lgroups.txt: L-group, biomarker 0/1, how many outer fits selected it, that
    count over the fits, and how many selected it from the good and from the poor L-group (a nested.NestedResult or a
    nested_survival.NestedSurvivalResult)."""
    bm = set(biomarkers)
    with open(prefix + suffix, 'w') as f:
        f.write('GeneSymbol\tLgroup(0:good,1:poor,2:other)\tBiomarker\tSelected\tFrequency\tSelectedGood\tSelectedPoor\n')
        f.writelines('%s\t%d\t%d\t%d\t%.6f\t%d\t%d\n' % (g, k, g in bm, n, q, a, b)
                     for g, k, n, q, a, b in zip(genes, lgroup, res.selected, res.frequency, res.selected_good,
                                                 res.selected_poor))


def write_nested_survival_cv(prefix, genes, res):
    """One row per outer fit of a nested_survival.NestedSurvivalResult (repeat-major, 1-based): its sample counts, test
    events, windows, stop epoch, list size, the C of its list and of top_t and top_z at that size, the full run's
    biomarkers', top_t's and top_z's C on the same fold, the Jaccard overlap with the full run's list and the list
    itself; then the nested survival CV line."""
    from .nested_survival import summary
    K, F = res.n_train.shape
    with open(prefix + "_nested_survival_cv.txt", 'w') as f:
        f.write('Repeat\tFold\tN_train\tN_test\tN_test_events\tN_windows\tStop_epoch\tSize\tC_nested\t'
                'C_nested_top_t\tC_nested_top_z\tC_biomarkers\tC_top_t\tC_top_z\tJaccard\tBiomarkers\n')
        for k in range(K):
            for j in range(F):
                bm = res.biomarkers[k][j]
                f.write('%d\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%.6f\t%.6f\t%.6f\t%.6f\t%.6f\t%.6f\t%.6f\t%s\n'
                        % ((k + 1, j + 1, res.n_train[k, j], res.n_test[k, j], res.n_test_events[k, j],
                            res.n_windows[k, j], res.stop_epoch[k, j], len(bm)) + tuple(res.c[:, k, j])
                           + (res.jaccard[k, j], ','.join(genes[g] for g in bm))))
        f.write(summary(res) + '\n')


def write_netrank(prefix, genes, lgroup, res, biomarkers, line):
    """One row per gene in the order of _lgroups.txt: L-group, degree, seed S, score, rank (1 = highest score), P and Q
    of a netrank.NetRankResult, biomarker 0/1; then the netrank line."""
    bm = set(biomarkers)
    rank = np.empty(res.order.shape[0], dtype=np.int64)
    rank[res.order] = np.arange(1, res.order.shape[0] + 1)
    with open(prefix + "_netrank.txt", 'w') as f:
        f.write('GeneSymbol\tLgroup(0:good,1:poor,2:other)\tDegree\tS\tScore\tRank\tP\tQ\tBiomarker\n')
        f.writelines('%s\t%d\t%d\t%.6f\t%.6f\t%d\t%.6g\t%.6g\t%d\n' % (g, k, dg, sv, sc, r, pv, qv, g in bm)
                     for g, k, dg, sv, sc, r, pv, qv in zip(genes, lgroup, res.degree, res.S, res.score, rank, res.P,
                                                          res.Q))
        f.write(line + '\n')


def write_lasso(prefix, genes, lgroup, res, biomarkers, line):
    """One row per gene in the order of _lgroups.txt: L-group, entry index on fit 0's path (-1 never), beta at
    lambda_min and lambda_1se, the fraction of fold fits in which the gene had entered by lambda_1se's index, biomarker
    0/1 (a lasso.LassoResult); then the lasso line."""
    bm = set(biomarkers)
    ent = res.entry[1:].astype(np.int64)
    frac = ((ent >= 0) & (ent <= res.i_1se)).mean(axis=0)
    with open(prefix + "_lasso.txt", 'w') as f:
        f.write('GeneSymbol\tLgroup(0:good,1:poor,2:other)\tEntry\tBeta_min\tBeta_1se\tFold_entered\tBiomarker\n')
        f.writelines('%s\t%d\t%d\t%.6g\t%.6g\t%.6f\t%d\n' % (g, k, e, b0, b1, fr, g in bm)
                     for g, k, e, b0, b1, fr in zip(genes, lgroup, res.entry[0], res.beta[res.i_min],
                                                  res.beta[res.i_1se], frac))
        f.write(line + '\n')


def write_lasso_path(prefix, res):
    """One row per lambda index of a lasso.LassoResult: lambda, df and deviance ratio of fit 0, CV deviance and its SE,
    mean CV AUC, and the marks of lambda_min and lambda_1se."""
    with open(prefix + "_lasso_path.txt", 'w') as f:
        f.write('Index\tLambda\tDf\tDev_ratio\tCV_deviance\tCV_SE\tCV_AUC\tMark\n')
        for k in range(res.n_lambda):
            mark = ','.join(m for m, i in (("min", res.i_min), ("1se", res.i_1se)) if i == k)
            f.write('%d\t%.6g\t%d\t%.6f\t%.6f\t%.6f\t%.6f\t%s\n' % (k, res.lambdas[k], res.df[k], res.dev_ratio[k],
                                                                      res.cvm[k], res.cvsd[k], res.auc_mean[k], mark))


def write_vectors(prefix, genes, mat):
    with open(prefix + "_vectors.txt", 'w') as f:
        f.write('GeneSymbol' + ''.join('\tV%d' % i for i in range(mat.shape[1])) + '\n')
        for g, vec in zip(genes, mat):
            f.write(g + ''.join("\t%.6f" % v for v in vec) + "\n")


# ------------------------------------------------------------------------------------------ main
def _distributed():
    """One process per GPU under torchrun (RANK / WORLD_SIZE / LOCAL_RANK in the environment): NCCL group,
    device = LOCAL_RANK.  Returns (rank, world, dist or None)."""
    import os
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1:
        return 0, 1, None
    import torch
    import torch.distributed as dist
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if not dist.is_initialized():
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    return dist.get_rank(), world, dist


def main(argv=None):
    args = parse_arguments(argv)
    nested_flag = '--nested-cv' if args.nested_cv else '--nested-survival-cv' if args.nested_survival_cv else None
    if nested_flag:
        import os
        if int(os.environ.get("WORLD_SIZE", "1")) > 1:            # before any process group or device
            sys.stdout.write('ERROR: %s: the nested loop runs on one GPU; run without torchrun\n' % nested_flag)
            sys.exit(1)
    rank, world, dist = _distributed()
    import builtins
    print = builtins.print if rank == 0 else (lambda *a, **k: None)   # noqa: A001  every rank computes, rank 0 talks
    print('>>> 0. Arguments')
    print(args)

    print('>>> 1. Load data')
    data = load_data(args.EXPRESSION_FILE)
    clinical = load_clinical(args.CLINICAL_FILE)
    network = load_network(args.NETWORK_FILE)

    print('>>> 2. Preprocess data')
    data['label'] = match_labels(clinical, data['sample'])
    data, network = restrict(data, network)
    n_samples, n_genes = data['expr'].shape
    print('    n_samples: %d' % n_samples)
    print('    n_genes  : %d\t(common genes in both EXPRESSION and NETWORK)' % n_genes)
    print('    n_edges  : %d\t(edges with the common genes)' % len(network['edge']))
    if args.permutations:
        from . import perm
        try:                                           # fail now rather than after training
            perm.check_inputs(data['expr'], data['label'], args.permutations)
        except ValueError as e:
            print('ERROR: %s' % e)
            sys.exit(1)
    if args.gene_sets is not None:
        from .gsea import check_inputs as gsea_check, read_gmt, restrict_sets
        try:                                           # fail now rather than after training
            gmt = read_gmt(args.gene_sets)
            set_ptr, _, set_names = restrict_sets(gmt, data['gene'], *args.gene_set_size)
            gsea_check(data['expr'], data['label'], args.gene_set_permutations, len(set_names), *args.gene_set_size)
        except (OSError, ValueError) as e:
            print('ERROR: --gene-sets: %s' % e)
            sys.exit(1)
        print('    gene sets: %d of %d in %s with %d..%d genes in the analysis'
              % (len(set_names), len(gmt), args.gene_sets, args.gene_set_size[0], args.gene_set_size[1]))
    if args.signature_cv:
        from . import signature
        try:                                           # fail now rather than after training
            signature.check_inputs(data['expr'], data['label'], min(2 * args.numBiomarker, n_genes), args.signature_cv,
                                   args.signature_folds, args.signature_repeats)
        except ValueError as e:
            print('ERROR: --signature-cv: %s' % e)
            sys.exit(1)
    if args.diff_coexpression:
        from . import diffcoex
        try:                                           # fail now rather than after training
            gi = {g: i for i, g in enumerate(data['gene'])}
            dcx_pairs = diffcoex.pairs_from_edges([gi[e[0]] for e in network['edge']],
                                                  [gi[e[1]] for e in network['edge']])
            diffcoex.check_inputs(data['expr'], data['label'], dcx_pairs, args.diff_coexpression)
        except ValueError as e:
            print('ERROR: --diff-coexpression: %s' % e)
            sys.exit(1)
        dcx_in_graph = []
    if args.netrank:
        from . import diffcoex, netrank
        try:                                           # fail now rather than after training
            gi = {g: i for i, g in enumerate(data['gene'])}
            nr_pairs = diffcoex.pairs_from_edges([gi[e[0]] for e in network['edge']],
                                                 [gi[e[1]] for e in network['edge']])
            netrank.check_inputs(data['expr'], data['label'], nr_pairs, args.netrank, args.netrank_damping)
        except ValueError as e:
            print('ERROR: --netrank: %s' % e)
            sys.exit(1)
    if args.survival is not None:
        from . import survival
        try:                                           # fail now rather than after training
            surv_time, surv_event, surv_used = survival.match_survival(survival.read_survival(args.survival),
                                                                       data['sample'])
            survival.check_inputs(data['expr'][surv_used], surv_time[surv_used], surv_event[surv_used],
                                  args.survival_permutations)
        except (OSError, ValueError) as e:
            print('ERROR: --survival: %s' % e)
            sys.exit(1)
        print('    survival: %d of %d samples with a record, %d events, in %s'
              % (int(surv_used.sum()), n_samples, int(surv_event[surv_used].sum()), args.survival))
        if args.survival_cv:
            from . import survival_cv
            try:
                survival_cv.check_inputs(data['expr'], surv_time, surv_event, data['label'],
                                         min(2 * args.numBiomarker, n_genes), args.survival_cv,
                                         args.survival_cv_folds, args.survival_cv_repeats)
            except ValueError as e:
                print('ERROR: --survival-cv: %s' % e)
                sys.exit(1)
    if args.nested_cv:
        from . import nested
        try:                                           # fail now rather than after training
            nested.check_inputs(data['expr'], data['label'], args.nested_cv, args.nested_cv_repeats,
                                min(2 * args.numBiomarker, n_genes))
        except ValueError as e:
            print('ERROR: --nested-cv: %s' % e)
            sys.exit(1)
    if args.nested_survival_cv:
        from . import nested_survival
        try:                                           # fail now rather than after training
            nested_survival.check_inputs(data['expr'], surv_time, surv_event, data['label'], args.nested_survival_cv,
                                         args.nested_survival_cv_repeats, min(2 * args.numBiomarker, n_genes))
        except ValueError as e:
            print('ERROR: --nested-survival-cv: %s' % e)
            sys.exit(1)
    if args.lasso:
        from . import lasso
        try:
            lasso.check_inputs(data['expr'], data['label'], args.lasso, args.lasso_repeats, args.lasso_alpha)
        except ValueError as e:
            print('ERROR: --lasso: %s' % e)
            sys.exit(1)
    if args.kmeans_restarts and n_genes < 3:
        print('ERROR: --kmeans-restarts needs at least 3 common genes, found %d' % n_genes)
        sys.exit(1)

    print('>>> 3. Generate random paths from each group')
    print('    *** most time consuming step ***')
    from . import paths, pipeline, walks              # needs the GPU from here on
    if args.walk_q != 1.0:
        a_near, a_far = walks.walk_bias(args.walk_q)
        print('    walk q  : %g\t(in-out multipliers %d near, %d far: effective q = %.6g)'
              % (args.walk_q, a_near, a_far, walks.effective_q(args.walk_q)))
    if args.correlation != 'pearson' or args.min_corr != 0.5:
        print('    correlation: %s (|r| > %g)' % (args.correlation, args.min_corr))
    src, dst = pipeline.edge_arrays(data['gene'], network['edge'])
    on_graph = None
    if args.diff_coexpression:                         # which pairs each group's graph kept, either direction
        on_graph = lambda i, rp, col: dcx_in_graph.append(diffcoex.graph_pairs(dcx_pairs, n_genes, rp.cpu().numpy(),
                                                                                col.cpu().numpy()))
    windows = pipeline.walk_windows(data['expr'], data['label'], src, dst, n_genes, args, dist=dist, rank=rank,
                                    world=world, on_graph=on_graph)
    code = windows[3]
    geneFreq = paths.gene_freq_dict(code, data['gene'])
    print("    n_paths : %d" % int(windows[2].shape[0]))
    print("    n_genes : %d\t(genes in good or poor random paths)" % len(geneFreq))
    if args.neighbors or args.tsne:
        from . import neighbors
        in_paths = neighbors.genes_in_paths(code)     # the same on every rank: each holds the 1-GPU windows
    if args.neighbors:
        if args.neighbors >= len(in_paths):
            print('ERROR: --neighbors %d needs more than %d genes in the random paths, found %d'
                  % (args.neighbors, args.neighbors, len(in_paths)))
            sys.exit(1)
    if args.tsne:
        from . import tsne
        if not args.tsne < len(in_paths) <= tsne.MAX_GENES:
            print('ERROR: --tsne %g needs more than %g and at most %d genes in the random paths, found %d'
                  % (args.tsne, args.tsne, tsne.MAX_GENES, len(in_paths)))
            sys.exit(1)

    print(">>> 4. Compute distributed representations using modified CBOW")
    mat = pipeline.train(windows, n_genes, args, log=print)   # print is silent off rank 0
    del windows
    genes = data['gene']
    if rank != 0:
        dist.barrier()
        dist.destroy_process_group()
        return

    print('>>> 5. Find L-groups')
    lgroup, km = pipeline.find_lgroups(mat, args)
    if args.kmeans_restarts:
        from . import kmeans
        print('    ' + kmeans.summary(km))

    print(">>> 6. Select biomarkers with gene scores")
    biomarkers = pipeline.select_biomarkers(mat, lgroup, data['expr'], data['label'], genes, args.numBiomarker)
    if args.permutations:
        res = perm.perm_test(data['expr'], data['label'], args.permutations, seed=args.seed)
        sig = res.P_maxT <= 0.05
        print('    permutation test: %d label permutations: %d genes with P_maxT <= 0.05 (%d of the biomarkers)'
              % (args.permutations, int(sig.sum()), len(set(genes[sig]) & set(biomarkers))))
    if args.neighbors:
        nbr_idx, nbr_sim = neighbors.nearest_genes(mat[in_paths], args.neighbors)
        print("    neighbors: %d nearest genes by cosine for each of %d genes in paths; %.1f %% of the pairs share the "
              "gene's L-group" % (args.neighbors, len(in_paths),
                                  100.0 * neighbors.same_lgroup_share(lgroup[in_paths], nbr_idx)))
    if args.tsne:
        tsne_res = tsne.tsne_map(mat[in_paths], args.tsne, n_iter=tsne.N_ITER, seed=args.seed)
        print('    ' + tsne.summary(len(in_paths), args.tsne, tsne.N_ITER, tsne_res.kl))

    if args.gene_sets is not None:
        from .gsea import gsea as gsea_test, summary as gsea_summary
        gsea_res = gsea_test(data['expr'], data['label'], gmt, args.gene_set_permutations, seed=args.seed,
                             min_size=args.gene_set_size[0], max_size=args.gene_set_size[1], genes=genes)
        print('    ' + gsea_summary(gsea_res))

    if args.signature_cv:
        pos = {g: i for i, g in enumerate(genes)}
        sig_res = signature.signature_cv(data['expr'], data['label'], np.array([pos[g] for g in biomarkers]),
                                         args.signature_cv, folds=args.signature_folds,
                                         repeats=args.signature_repeats, seed=args.seed)
        print('    ' + signature.summary(sig_res))

    if args.diff_coexpression:
        dcx_res = diffcoex.diffcoex_test(data['expr'], data['label'], dcx_pairs, args.diff_coexpression, seed=args.seed)
        bm = set(biomarkers)
        is_bm = np.array([g in bm for g in genes], dtype=np.int64)
        dcx_bm = is_bm[dcx_pairs[:, 0]] + is_bm[dcx_pairs[:, 1]]
        print('    ' + diffcoex.summary(dcx_res, dcx_in_graph[0], dcx_in_graph[1], dcx_bm))

    if args.netrank:
        nr_res = netrank.netrank_test(data['expr'], data['label'], nr_pairs, args.netrank, damping=args.netrank_damping,
                                      seed=args.seed)
        bm = set(biomarkers)
        nr_bm = np.array([g in bm for g in genes])
        nr_auc = None
        if args.signature_cv:                          # top_netrank on --signature-cv's splits, beside the biomarkers
            from .perm import check_inputs as used_samples
            head = netrank.top_netrank(nr_res, len(biomarkers))[None, :]
            auc = signature.cv_fits(*used_samples(data['expr'], data['label'], 1), head, 0, args.signature_repeats,
                                    args.signature_folds, args.seed)[2]
            nr_auc = (float(auc[0].reshape(-1).mean()), float(sig_res.auc_mean[0]))
        nr_line = netrank.summary(nr_res, args.netrank_damping, nr_pairs.shape[0], nr_bm, nr_auc)
        print('    ' + nr_line)

    if args.survival is not None:
        surv_res = survival.survival_test(data['expr'][surv_used], surv_time[surv_used], surv_event[surv_used],
                                          args.survival_permutations, seed=args.seed)
        bm = set(biomarkers)
        label_z, label_p = survival.label_score(data['label'][surv_used], surv_time[surv_used],
                                                surv_event[surv_used])
        print('    ' + survival.summary(surv_res, np.array([g in bm for g in genes]), label_z, label_p))

    if args.survival_cv:
        pos = {g: i for i, g in enumerate(genes)}
        scv_res = survival_cv.survival_cv(data['expr'], surv_time, surv_event, data['label'],
                                          np.array([pos[g] for g in biomarkers]), args.survival_cv,
                                          folds=args.survival_cv_folds, repeats=args.survival_cv_repeats,
                                          seed=args.seed)
        print('    ' + survival_cv.summary(scv_res))

    if args.nested_cv:
        same_splits = (args.signature_cv and args.signature_folds == args.nested_cv
                       and args.signature_repeats == args.nested_cv_repeats)
        try:
            ncv_res = nested.nested_cv(data['expr'], data['label'], src, dst, genes, args, biomarkers,
                                       random_auc=sig_res.auc_mean[2:] if same_splits else None,
                                       log=lambda line: print('    ' + line))
        except ValueError as e:
            print('ERROR: --nested-cv: %s' % e)
            sys.exit(1)
        print('    ' + nested.summary(ncv_res))

    if args.nested_survival_cv:
        same_splits = (args.survival_cv and args.survival_cv_folds == args.nested_survival_cv
                       and args.survival_cv_repeats == args.nested_survival_cv_repeats)
        try:
            nscv_res = nested_survival.nested_survival_cv(data['expr'], data['label'], surv_time, surv_event, src, dst,
                                                          genes, args, biomarkers,
                                                          random_c=scv_res.c_mean[3:] if same_splits else None,
                                                          log=lambda line: print('    ' + line))
        except ValueError as e:
            print('ERROR: --nested-survival-cv: %s' % e)
            sys.exit(1)
        print('    ' + nested_survival.summary(nscv_res))

    if args.lasso:
        ls_res = lasso.lasso_cv(data['expr'], data['label'], folds=args.lasso, repeats=args.lasso_repeats,
                                alpha=args.lasso_alpha, seed=args.seed)
        pos = {g: i for i, g in enumerate(genes)}
        bm_idx = np.array(sorted(pos[g] for g in biomarkers), dtype=np.int64)
        ls_x, ls_lab = lasso.check_inputs(data['expr'], data['label'], args.lasso, args.lasso_repeats,
                                          args.lasso_alpha)
        extra = ""
        top = np.sort(lasso.top_lasso(ls_res.entry[0], ls_res.entry_abs[0], len(biomarkers)))
        if args.signature_cv and top.size:             # top_lasso on --signature-cv's splits, beside the biomarkers
            auc = signature.cv_fits(ls_x, ls_lab, top[None, :].astype(np.int32), 0, args.signature_repeats,
                                    args.signature_folds, args.seed)[2]
            extra += "; top_lasso AUC %.3f vs biomarkers %.3f on the signature splits" % (
                float(auc[0].reshape(-1).mean()), float(sig_res.auc_mean[0]))
        if args.nested_cv == args.lasso and args.nested_cv_repeats == args.lasso_repeats:
            nl = lasso.nested_lasso(ls_x, ls_lab, ls_res, ncv_res.biomarkers, args.seed)
            extra += "; nested_lasso AUC %.3f vs nested_biomarkers %.3f" % (float(np.nanmean(nl)),
                                                                            float(ncv_res.auc_mean[0]))
        ls_line = lasso.summary(ls_res, bm_idx, extra)
        print('    ' + ls_line)

    print(">>> 7. Save results")
    write_biomarkers(args.RESULT_NAME, biomarkers)
    print('    %s_biomarkers.txt' % args.RESULT_NAME)
    write_lgroups(args.RESULT_NAME, lgroup, genes)
    print('    %s_lgroups.txt' % args.RESULT_NAME)
    write_vectors(args.RESULT_NAME, genes, mat)
    print('    %s_vectors.txt' % args.RESULT_NAME)
    if args.permutations:
        write_pvalues(args.RESULT_NAME, genes, lgroup, res, biomarkers)
        print('    %s_pvalues.txt' % args.RESULT_NAME)
    if args.neighbors:
        write_neighbors(args.RESULT_NAME, genes, lgroup, in_paths, nbr_idx, nbr_sim)
        print('    %s_neighbors.txt' % args.RESULT_NAME)
    if args.kmeans_restarts:
        write_kmeans(args.RESULT_NAME, genes, km)
        print('    %s_kmeans.txt' % args.RESULT_NAME)
    if args.tsne:
        write_tsne(args.RESULT_NAME, genes, lgroup, in_paths, tsne_res.Y)
        print('    %s_tsne.txt' % args.RESULT_NAME)
    if args.gene_sets is not None:
        write_gsea(args.RESULT_NAME, genes, gsea_res, biomarkers)
        print('    %s_gsea.txt' % args.RESULT_NAME)
    if args.signature_cv:
        write_signature(args.RESULT_NAME, genes, sig_res, biomarkers)
        print('    %s_signature.txt' % args.RESULT_NAME)
    if args.diff_coexpression:
        write_diffcoex(args.RESULT_NAME, genes, dcx_res, dcx_in_graph[0], dcx_in_graph[1], dcx_bm)
        print('    %s_diffcoex.txt' % args.RESULT_NAME)
    if args.netrank:
        write_netrank(args.RESULT_NAME, genes, lgroup, nr_res, biomarkers, nr_line)
        print('    %s_netrank.txt' % args.RESULT_NAME)
    if args.survival is not None:
        write_survival(args.RESULT_NAME, genes, lgroup, surv_res, biomarkers)
        print('    %s_survival.txt' % args.RESULT_NAME)
    if args.survival_cv:
        write_survival_cv(args.RESULT_NAME, genes, scv_res, biomarkers)
        print('    %s_survival_cv.txt' % args.RESULT_NAME)
        write_risk(args.RESULT_NAME, [s for s, u in zip(data['sample'], surv_used) if u], surv_time[surv_used],
                   surv_event[surv_used], scv_res)
        print('    %s_risk.txt' % args.RESULT_NAME)
    if args.nested_cv:
        write_nested_cv(args.RESULT_NAME, genes, ncv_res)
        print('    %s_nested_cv.txt' % args.RESULT_NAME)
        write_nested_selection(args.RESULT_NAME, genes, lgroup, ncv_res, biomarkers)
        print('    %s_nested_selection.txt' % args.RESULT_NAME)
    if args.nested_survival_cv:
        write_nested_survival_cv(args.RESULT_NAME, genes, nscv_res)
        print('    %s_nested_survival_cv.txt' % args.RESULT_NAME)
        write_risk(args.RESULT_NAME, [s for s, u in zip(data['sample'], surv_used) if u], surv_time[surv_used],
                   surv_event[surv_used], nscv_res, suffix="_nested_survival_risk.txt")
        print('    %s_nested_survival_risk.txt' % args.RESULT_NAME)
        write_nested_selection(args.RESULT_NAME, genes, lgroup, nscv_res, biomarkers,
                               suffix="_nested_survival_selection.txt")
        print('    %s_nested_survival_selection.txt' % args.RESULT_NAME)
    if args.lasso:
        write_lasso(args.RESULT_NAME, genes, lgroup, ls_res, biomarkers, ls_line)
        print('    %s_lasso.txt' % args.RESULT_NAME)
        write_lasso_path(args.RESULT_NAME, ls_res)
        print('    %s_lasso_path.txt' % args.RESULT_NAME)
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
