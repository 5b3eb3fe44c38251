"""Cost of the nested survival cross-validation of the selection (DESIGN.md §4.36).

For each workload, at the command line's defaults (-p 80 -r 10 -s 128 -e 500 -n 50, --seed 0) with
--nested-survival-cv 5:

* full_selection_s   -- pipeline.select on every sample (what one run's steps 3-6 cost);
* one outer fit (repeat 1, fold 1) in parts, each a host clock around work that ends in a device synchronise:
  selection_s (nested.select_fit: steps 3-6 on every expression sample outside the test fold), top_t_s
  (signature.top_t of the training samples), top_z_s (survival.rank_genes of the training survival samples) and
  fits_s (nested_survival.score_fit: the two-fold-row Cox fits and concordance of the three lists);
* nested_survival_cv_s -- the whole nested_survival.nested_survival_cv call (the comparison rows and all 5 outer
  fits).

Workloads: the ex cohort (135 x 7 523, 216 540 edges, tests/golden) and the seeded 1 000 x 20 000 cohort of
bench_nested.py.  Survival records are seeded: exponential times whose hazard rises with the first module's mean
expression, about 30 % censored, 5 % of the samples without a record.  The card name, power limit and SM clock are
read in the same run.  Writes nothing into the tree; prints one JSON line per workload.

    python bench_nested_survival.py [--workloads ex syn1000x20000]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_correlation import card  # noqa: E402
from bench_nested import timed, workload  # noqa: E402


def records(expr):
    """(time, event) per sample: hazard exp(mean of the first 20 genes), about 30 % censored, 5 % NaN (no record)."""
    rng = np.random.Generator(np.random.PCG64(2036))
    n = expr.shape[0]
    x = np.asarray(expr[:, :20], dtype=np.float64).mean(axis=1)
    t = np.round(rng.exponential(1.0 / np.exp((x - x.mean()) / max(x.std(), 1e-12))) * 100.0, 2)
    e = (rng.uniform(size=n) < 0.7).astype(np.int64)
    t[rng.choice(n, n // 20, replace=False)] = np.nan
    return t, e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["ex", "syn1000x20000"])
    opts = ap.parse_args()
    import torch
    from g2vec_b200 import cli, nested, nested_survival, pipeline, signature, survival, survival_cv
    if not torch.cuda.is_available():
        raise SystemExit("bench_nested_survival.py needs a GPU")
    name, power, clock = card()
    for wl in opts.workloads:
        expr, label, genes, src, dst = workload(wl)
        t, e = records(expr)
        args = cli.parse_arguments(["E", "C", "N", "R", "--survival", "S", "--nested-survival-cv", "5"])
        full, t_full = timed(lambda: pipeline.select(expr, label, src, dst, genes, args))
        x, tu, eu, used = nested_survival.check_inputs(expr, t, e, label, 5, 1)
        bm = nested.run_list(genes, full.biomarkers)
        fold = survival_cv.cox_fits(x, tu, eu, bm[None, :], 0, 1, 5, args.seed)[1]
        test = fold[0] == 0
        in_test = np.zeros(expr.shape[0], dtype=bool)
        in_test[np.flatnonzero(used)[test]] = True
        rows = np.flatnonzero(~in_test)
        (sel, mine), t_sel = timed(lambda: nested.select_fit(expr, label, rows, src, dst, genes, args, 0, 0))
        q = mine.shape[0]
        tt, t_tt = timed(lambda: signature.top_t(expr[rows], label[rows], q))
        tz, t_tz = timed(lambda: np.sort(survival.rank_genes(x[~test], tu[~test], eu[~test])[:q]).astype(np.int32))
        _, t_fit = timed(lambda: nested_survival.score_fit(x, tu, eu, fold, 0, 0, np.stack([mine, tt, tz]),
                                                           seed=args.seed))
        res, t_nested = timed(lambda: nested_survival.nested_survival_cv(expr, label, t, e, src, dst, genes, args,
                                                                         full.biomarkers))
        print(json.dumps(dict(
            workload=wl, n=int(expr.shape[0]), n_survival=int(used.sum()), events=int(eu.sum()),
            genes=int(expr.shape[1]), edges=int(src.size), folds=5, full_selection_s=round(t_full, 3),
            outer_fit=dict(n_train=int(rows.size), n_test=int(test.sum()), windows=sel.n_windows,
                           best_epoch=sel.info["best_step"], selection_s=round(t_sel, 3), top_t_s=round(t_tt, 3),
                           top_z_s=round(t_tz, 4), fits_s=round(t_fit, 4)),
            nested_survival_cv_s=round(t_nested, 2), c_mean=[round(float(v), 4) for v in res.c_mean],
            optimism=round(res.optimism, 4), gpu=name, power_limit=power, sm_clock=clock)), flush=True)


if __name__ == "__main__":
    main()
