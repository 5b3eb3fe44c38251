"""Cost of the nested cross-validation of the selection (DESIGN.md §4.34).

For each workload, at the command line's defaults (-p 80 -r 10 -s 128 -e 500 -n 50, --seed 0) with --nested-cv 5:

* full_selection_s   -- pipeline.select on every sample (what one run's steps 3-6 cost);
* one outer fit (repeat 1, fold 1) in parts, each a host clock around work that ends in a device synchronise:
  walks_s (edge weights, walks and path glue: pipeline.walk_windows), train_s (pipeline.train), step5_s
  (pipeline.find_lgroups: scikit-learn's KMeans, or the GPU restarts with --kmeans-restarts), step6_s
  (pipeline.select_biomarkers), top_t_s (signature.top_t of the training samples) and fits_s (nested.score_fit: the
  two-fold-row fits and AUC of the two lists);
* nested_cv_s        -- the whole nested.nested_cv call (the comparison rows and all 5 outer fits).

Workloads: the ex cohort (135 x 7 523, 216 540 edges, tests/golden) and a seeded 1 000 x 20 000 cohort in modules of
20 genes (x = 0.85 f + 0.5 e per module), each gene joined to 10 genes of its module plus 20 000 random edges, labels
half and half, one module whose level and co-expression shift with the label.  The card name, power limit and SM
clock are read in the same run.  Writes nothing into the tree; prints one JSON line per workload.

    python bench_nested.py [--workloads ex syn1000x20000] [--kmeans-restarts R]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_correlation import card  # noqa: E402


def workload(name):
    """-> (expr float32 [n, G], label [n], genes, src, dst)"""
    if name == "ex":
        e = np.load(os.path.join(ROOT, "tests", "golden", "ex_expr.npz"))
        lab = np.load(os.path.join(ROOT, "tests", "golden", "ex_graph.npz"))["label"]
        return e["expr"], lab.astype(np.int64), e["gene"], e["src"].astype(np.int32), e["dst"].astype(np.int32)
    n, G = (int(v) for v in name[3:].split("x"))
    rng = np.random.Generator(np.random.PCG64(2002))
    M = 20
    label = np.repeat([0, 1], [n // 2, n - n // 2])
    rng.shuffle(label)
    f = rng.standard_normal((n, G // M))
    x = (0.85 * np.repeat(f, M, axis=1) + 0.5 * rng.standard_normal((n, G))).astype(np.float32)
    poor = (label == 1)[:, None]
    x[:, :M] = np.where(poor, 1.0 + x[:, :M], rng.standard_normal((n, M)).astype(np.float32))
    base = np.arange(G) // M * M
    src = np.repeat(np.arange(G), 10)
    dst = base[src] + (src % M + rng.integers(1, M, src.size)) % M
    extra = rng.integers(0, G, (2, 20000))
    src = np.concatenate([src, extra[0]]).astype(np.int32)
    dst = np.concatenate([dst, extra[1]]).astype(np.int32)
    return x, label, np.array(["G%05d" % i for i in range(G)]), src, dst


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["ex", "syn1000x20000"])
    ap.add_argument("--kmeans-restarts", type=int, default=0)
    opts = ap.parse_args()
    import torch
    from g2vec_b200 import cli, nested, pipeline, signature
    if not torch.cuda.is_available():
        raise SystemExit("bench_nested.py needs a GPU")
    name, power, clock = card()
    for wl in opts.workloads:
        expr, label, genes, src, dst = workload(wl)
        args = cli.parse_arguments(["E", "C", "N", "R", "--nested-cv", "5", "--kmeans-restarts",
                                    str(opts.kmeans_restarts)])
        full, t_full = timed(lambda: pipeline.select(expr, label, src, dst, genes, args))
        x, lab, used = nested.check_inputs(expr, label, 5, 1)
        pos = {g: i for i, g in enumerate(genes)}
        bm = np.array(sorted(pos[g] for g in full.biomarkers), dtype=np.int32)
        head = np.stack([bm, signature.top_t(x, lab, len(bm))])
        fold = signature.cv_fits(x, lab, head, 0, 1, 5, args.seed)[1]
        train = fold[0] != 0
        rows = np.flatnonzero(used)[train]
        e_tr, l_tr = expr[rows], label[rows]
        windows, t_walk = timed(lambda: pipeline.walk_windows(e_tr, l_tr, src, dst, len(genes), args))
        n_windows = int(windows[2].shape[0])
        (mat, info), t_train = timed(lambda: pipeline.train(windows, len(genes), args, return_info=True))
        del windows
        (lgroup, _), t5 = timed(lambda: pipeline.find_lgroups(mat, args))
        sel, t6 = timed(lambda: pipeline.select_biomarkers(mat, lgroup, e_tr, l_tr, genes, args.numBiomarker))
        mine = np.array(sorted(pos[g] for g in sel), dtype=np.int32)
        tt, t_tt = timed(lambda: signature.top_t(x[train], lab[train], len(mine)))
        _, t_fit = timed(lambda: nested.score_fit(x, lab, fold, 0, 0, np.stack([mine, tt]), seed=args.seed))
        res, t_nested = timed(lambda: nested.nested_cv(expr, label, src, dst, genes, args, full.biomarkers))
        print(json.dumps(dict(
            workload=wl, n=int(expr.shape[0]), genes=int(expr.shape[1]), edges=int(src.size), folds=5,
            kmeans_restarts=opts.kmeans_restarts, full_selection_s=round(t_full, 3),
            outer_fit=dict(n_train=int(train.sum()), windows=n_windows, best_epoch=info["best_step"],
                           walks_s=round(t_walk, 3), train_s=round(t_train, 3), step5_s=round(t5, 3),
                           step6_s=round(t6, 3), top_t_s=round(t_tt, 3), fits_s=round(t_fit, 4)),
            nested_cv_s=round(t_nested, 2), auc_mean=[round(float(v), 4) for v in res.auc_mean],
            optimism=round(res.optimism, 4), gpu=name, power_limit=power, sm_clock=clock)), flush=True)


if __name__ == "__main__":
    main()
