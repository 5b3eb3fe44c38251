"""The G2Vec command line, kept as the drop-in shell around the two H100 hot paths.

Same positionals, options, progress banners and output files as /root/reference/G2Vec.py
(parse_arguments :505-518, main :11-119, writers :127-131,159-165,203-215).  Steps 1, 2, 5, 6, 7 are
plain Python/NumPy/scikit-learn as in the reference; step 3 runs g2vec_b200.walks on the GPU and
step 4 g2vec_b200.cbow.  Two documented differences: ``--epoch`` is honoured as the cap on optimizer
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
    args = p.parse_args(argv)
    if not (np.isfinite(args.walk_q) and 1.0 / 256.0 <= args.walk_q <= 256.0):
        p.error("--walk-q must be a finite number in [1/256, 256]")
    if not (np.isfinite(args.min_corr) and 0.0 <= args.min_corr < 1.0):
        p.error("--min-corr must be a finite number with 0 <= T < 1")
    if args.class_weight is not None:
        args.class_weight = _parse_class_weight(args.class_weight, p)
    if not 0.0 <= float(np.float32(args.weight_decay)) < 1.0:
        p.error("--weight-decay must be a finite number with 0 <= weight-decay < 1")
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
    """KMeans(3, random_state=0) on the vectors; largest cluster -> 2 (other); of the remaining two
    clusters the reference compares good/poor gene-frequency votes (G2Vec.py:167-200).  In the reference
    ``freqIdx`` is a Python list, so ``freqIdx==0`` is the scalar False and both votes are always 0
    (:172,186-187): the outcome is therefore always good = second remaining cluster, poor = first.  That
    behaviour is reproduced here so the output files match."""
    from sklearn.cluster import KMeans
    km = KMeans(n_clusters=3, random_state=0).fit(mat).labels_
    sizes = [int(np.count_nonzero(km == k)) for k in range(3)]
    largest = 0
    for k in (1, 2):
        if sizes[k] > sizes[largest]:
            largest = k
    rest = [k for k in (0, 1, 2) if k != largest]
    poor_c, good_c = rest[0], rest[1]
    out = np.zeros(mat.shape[0], dtype=np.int32)
    out[km == good_c] = 0
    out[km == poor_c] = 1
    out[km == largest] = 2
    return out


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

    print('>>> 3. Generate random paths from each group')
    print('    *** most time consuming step ***')
    from . import graph, paths, walks, cbow           # needs the GPU from here on
    if args.walk_q != 1.0:
        a_near, a_far = walks.walk_bias(args.walk_q)
        print('    walk q  : %g\t(in-out multipliers %d near, %d far: effective q = %.6g)'
              % (args.walk_q, a_near, a_far, walks.effective_q(args.walk_q)))
    if args.correlation != 'pearson' or args.min_corr != 0.5:
        print('    correlation: %s (|r| > %g)' % (args.correlation, args.min_corr))
    idx = {g: i for i, g in enumerate(data['gene'])}
    src = np.fromiter((idx[e[0]] for e in network['edge']), dtype=np.int32, count=len(network['edge']))
    dst = np.fromiter((idx[e[1]] for e in network['edge']), dtype=np.int32, count=len(network['edge']))
    import torch
    n_total = n_genes * args.numRepetition                     # walkers per group: w = repetition * n_genes + start gene
    L = args.lenPath
    dev = torch.device("cuda", torch.cuda.current_device())
    rows = torch.empty((2 * n_total, L), dtype=torch.int32, device=dev)
    lens = torch.empty(2 * n_total, dtype=torch.int32, device=dev)
    key = torch.empty(2 * n_total, dtype=torch.int64, device=dev)
    for i, _group in enumerate(['g', 'p']):
        rp, col, w = graph.group_csr_gpu(data['expr'], data['label'], i, src, dst, threshold=args.min_corr,
                                         method=args.correlation)
        wg = walks.WalkGraph(rp, col, weights=w)
        sl = slice(i * n_total, (i + 1) * n_total)
        if dist is None:
            # tuple(sorted(path)) is fused into the sampler: sorted rows + their 64-bit keys come back
            walks.generate_paths(wg, L, args.numRepetition, seed=args.seed, group=i, canonical=True,
                                 out=(rows[sl], lens[sl], key[sl]), q=args.walk_q)
        else:
            # walkers rank, rank+world, ...: no collective during the walk (counter-based RNG); one all_gather after,
            # rows put back at their walker index so that every rank holds the 1-GPU arrays (same window order,
            # hence the same --seed split, whatever the number of GPUs)
            r_, l_, k_ = walks.generate_paths(wg, L, args.numRepetition, seed=args.seed, group=i, canonical=True,
                                              walker_begin=rank, walker_stride=world, q=args.walk_q)
            rows[sl], lens[sl], key[sl] = paths.gather_walker_shards(dist, world, n_total, r_, l_, k_)
    group = torch.cat([torch.zeros(n_total, dtype=torch.uint8, device=dev), torch.ones(n_total, dtype=torch.uint8, device=dev)])
    w_rowptr, w_gene, w_label, code = paths.build_windows(rows, lens, key, group, n_genes)
    del rows, lens, key, group
    geneFreq = paths.gene_freq_dict(code, data['gene'])
    print("    n_paths : %d" % int(w_label.shape[0]))
    print("    n_genes : %d\t(genes in good or poor random paths)" % len(geneFreq))

    print(">>> 4. Compute distributed representations using modified CBOW")
    mat = cbow.train_cbow(w_rowptr, w_gene, w_label, n_genes, args.sizeHiddenlayer, args.learningRate,
                          max_epoch=args.epoch, seed=args.seed, log=print, algo=args.algo,   # print is silent off rank 0
                          batch=args.batch, optimizer=args.optimizer, reshuffle=args.reshuffle,
                          deterministic=args.deterministic, patience=args.patience, lr_patience=args.lr_patience,
                          lr_factor=args.lr_factor, min_lr=args.min_lr, weight_decay=args.weight_decay,
                          monitor=args.monitor, class_weight=args.class_weight)
    genes = data['gene']
    if rank != 0:
        dist.barrier()
        dist.destroy_process_group()
        return

    print('>>> 5. Find L-groups')
    lgroup = find_lgroups(mat, genes, geneFreq)

    print(">>> 6. Select biomarkers with gene scores")
    biomarkers = []
    for i in (0, 1):
        sel = lgroup == i
        d = minmax(np.linalg.norm(mat[sel], axis=1))
        t = minmax(tscores(data['expr'][:, sel], data['label']))
        score = 0.5 * (d + t)
        ranked = sorted(zip(genes[sel], score), key=lambda gs: gs[1], reverse=True)
        biomarkers += sorted(g for g, _ in ranked[:args.numBiomarker])
    biomarkers = sorted(biomarkers)

    print(">>> 7. Save results")
    write_biomarkers(args.RESULT_NAME, biomarkers)
    print('    %s_biomarkers.txt' % args.RESULT_NAME)
    write_lgroups(args.RESULT_NAME, lgroup, genes)
    print('    %s_lgroups.txt' % args.RESULT_NAME)
    write_vectors(args.RESULT_NAME, genes, mat)
    print('    %s_vectors.txt' % args.RESULT_NAME)
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
