"""Steps 3-6 of a G2Vec run, the selection of the biomarkers, in one implementation: cli.main runs them on every
sample, nested.nested_cv on every outer training fold (DESIGN.md §4.34).

Each step takes the run's options as the namespace cli.parse_arguments returns (or any object with the same
attributes) and is silent unless given a ``log``.  What only the command line's own run needs stays with the caller:
cli.main passes the torchrun process group to walk_windows and collects ``--diff-coexpression``'s per-group graphs
through ``on_graph``, and it checks ``--neighbors`` / ``--tsne`` against the windows' genes itself.
"""
from collections import namedtuple

import numpy as np

Selection = namedtuple("Selection", "vectors lgroup biomarkers gene_freq n_windows info kmeans")
Selection.__doc__ = """select's result.
vectors     float32 [G, D]: the trained W_ih (step 4);  lgroup: int [G], 0 good, 1 poor, 2 other (step 5);
biomarkers  the sorted gene names of step 6 (at most 2 n);  gene_freq: {gene name: 0 good, 1 poor, 2 tie} over the
            genes in the windows (step 3's vote);  n_windows: the number of windows the trainer got;
info        the trainer's return_info dict without its device objects ("history", "stop_step", "best_step", ...);
kmeans      the kmeans.KMeansResult of step 5 with ``--kmeans-restarts``, else None."""


def edge_arrays(genes, edges):
    """The edge list of step 2 (pairs of gene names) as int32 (src, dst) indices into genes."""
    idx = {g: i for i, g in enumerate(genes)}
    src = np.fromiter((idx[e[0]] for e in edges), dtype=np.int32, count=len(edges))
    dst = np.fromiter((idx[e[1]] for e in edges), dtype=np.int32, count=len(edges))
    return src, dst


def walk_windows(expr, label, src, dst, n_genes, args, dist=None, rank=0, world=1, on_graph=None):
    """Step 3 on the GPU: each group's graph (``--correlation``, ``--min-corr`` over the samples of that label), the
    random walks (``-p``, ``-r``, ``--walk-q``, ``--seed``) and the path glue.  Returns the trainer's CSR windows and
    the per-gene vote: (rowptr, gene, label, code), device tensors as paths.build_windows gives them.

    dist: the torchrun process group (rank, world): each rank walks its share of the walkers and the rows are
    gathered back into the one-GPU order.  on_graph(group, rowptr, col): called with each group's CSR graph."""
    import torch
    from . import graph, paths, walks
    n_total = n_genes * args.numRepetition                     # walkers per group: w = repetition * n_genes + start gene
    L = args.lenPath
    dev = torch.device("cuda", torch.cuda.current_device())
    rows = torch.empty((2 * n_total, L), dtype=torch.int32, device=dev)
    lens = torch.empty(2 * n_total, dtype=torch.int32, device=dev)
    key = torch.empty(2 * n_total, dtype=torch.int64, device=dev)
    for i in (0, 1):
        rp, col, w = graph.group_csr_gpu(expr, label, i, src, dst, threshold=args.min_corr, method=args.correlation)
        if on_graph is not None:
            on_graph(i, rp, col)
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
    group = torch.cat([torch.zeros(n_total, dtype=torch.uint8, device=dev),
                       torch.ones(n_total, dtype=torch.uint8, device=dev)])
    return paths.build_windows(rows, lens, key, group, n_genes)


def train(windows, n_genes, args, log=None, return_info=False):
    """Step 4: the modified CBOW on the windows of walk_windows with every trainer option of args.  Returns W_ih as
    float32 [n_genes, D], and with return_info also the trainer's return_info dict without its device objects."""
    from . import cbow
    w_rowptr, w_gene, w_label = windows[:3]
    out = cbow.train_cbow(w_rowptr, w_gene, w_label, n_genes, args.sizeHiddenlayer, args.learningRate,
                          max_epoch=args.epoch, seed=args.seed, log=log, algo=args.algo, batch=args.batch,
                          optimizer=args.optimizer, reshuffle=args.reshuffle, deterministic=args.deterministic,
                          patience=args.patience, lr_patience=args.lr_patience, lr_factor=args.lr_factor,
                          min_lr=args.min_lr, weight_decay=args.weight_decay, monitor=args.monitor,
                          class_weight=args.class_weight, **({"return_info": True} if return_info else {}))
    if not return_info:
        return out
    mat, info = out
    return mat, {k: v for k, v in info.items() if k not in ("model", "windows")}


def find_lgroups(mat, args):
    """Step 5: (lgroup, kmeans result) -- the best of ``--kmeans-restarts`` restarts on the GPU at ``--seed``, or
    scikit-learn's KMeans(3, random_state=0) (cli.find_lgroups) and None."""
    if args.kmeans_restarts:
        from . import kmeans
        km = kmeans.kmeans_lgroups(mat, args.kmeans_restarts, seed=args.seed)
        return km.lgroups, km
    from .cli import find_lgroups as sklearn_lgroups
    return sklearn_lgroups(mat, None, None), None


def select_biomarkers(mat, lgroup, expr, label, genes, n):
    """Step 6: in each of the good and poor L-groups the n genes of largest score ½ (minmax |vector| + minmax |t|),
    |t| over expr's samples of label 0 against label 1.  Returns the sorted gene names (fewer than 2 n when an
    L-group holds fewer than n genes)."""
    from .cli import minmax, tscores
    biomarkers = []
    for i in (0, 1):
        sel = lgroup == i
        d = minmax(np.linalg.norm(mat[sel], axis=1))
        t = minmax(tscores(expr[:, sel], label))
        score = 0.5 * (d + t)
        ranked = sorted(zip(genes[sel], score), key=lambda gs: gs[1], reverse=True)
        biomarkers += sorted(g for g, _ in ranked[:n])
    return sorted(biomarkers)


def select(expr, label, src, dst, genes, args, log=None):
    """Steps 3-6 on the samples given: expr [samples, G] (host), label per sample, the step-2 edges as indices into
    genes.  Only these samples' expression and labels are read.  One GPU.  Returns a Selection."""
    from . import paths
    n_genes = len(genes)
    windows = walk_windows(expr, label, src, dst, n_genes, args)
    code = windows[3]
    gene_freq = paths.gene_freq_dict(code, genes)
    n_windows = int(windows[2].shape[0])
    mat, info = train(windows, n_genes, args, log=log, return_info=True)
    del windows
    lgroup, km = find_lgroups(mat, args)
    biomarkers = select_biomarkers(mat, lgroup, expr, label, genes, args.numBiomarker)
    return Selection(vectors=mat, lgroup=lgroup, biomarkers=biomarkers, gene_freq=gene_freq, n_windows=n_windows,
                     info=info, kmeans=km)
