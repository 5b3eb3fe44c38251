"""Cost of the cross-validated lasso path (DESIGN.md §4.37):

* grad -- one g2v_lasso_grad round for every fit of the run (the DGEMM X R^T on the FP64 tensor cores), CUDA events,
  warmed, median of --iters, with the rate of its 2 G n_pad fits flops;
* lasso_cv -- g2vec_b200.lasso.lasso_cv end to end (synchronised wall time, after one warm-up call), with the path
  length, the rounds' Newton steps and the certified count.

Workloads: ex_* (135 samples x 7 523 genes) at F = 5 and 10, and a seeded TCGA-sized cohort (1 000 x 20 000, 20
planted genes) at F = 5 with K = 1 and 10.  The card name, power limit and SM clock are read in the same run.  The CPU
reference is the NumPy restatement of tests/lasso_oracle.py on fit 0 only, timed over --cpu-lambdas lambdas and scaled
linearly to the path length and the 1 + K F fits (its per-lambda cost grows along the path, so this is a lower bound).
Writes nothing into the tree; prints one JSON line per workload.

    python bench_lasso.py [--workloads ex5 ex10 tcga5 tcga5x10] [--iters 5] [--cpu-lambdas 5]
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

WORKLOADS = {"ex5": ("ex", 5, 1), "ex10": ("ex", 10, 1), "tcga5": ("tcga", 5, 1), "tcga5x10": ("tcga", 5, 10)}


def cohort(name):
    if name == "ex":
        e = np.load(os.path.join(ROOT, "tests", "golden", "ex_expr.npz"))
        lab = np.load(os.path.join(ROOT, "tests", "golden", "ex_graph.npz"))["label"]
        return e["expr"].astype(np.float64), lab
    rng = np.random.Generator(np.random.PCG64(2037))
    S, G = 1_000, 20_000
    lab = (rng.random(S) < 0.4).astype(np.int64)
    x = rng.standard_normal((S, G))
    x[:, :20] += 0.4 * lab[:, None]
    return x, lab


def grad_ms(x, lab, fits, iters):
    import torch
    from g2vec_b200 import _capi
    lib = _capi.load()
    n, G = x.shape
    n_pad = -(-n // 32) * 32
    Xt = np.zeros((G, n_pad)); Xt[:, :n] = x.T
    X = torch.from_numpy(Xt).cuda()
    y = torch.from_numpy(lab.astype(np.uint8)).cuda()
    fold = torch.zeros((1, n), dtype=torch.int8, device="cuda")
    ws = torch.empty(int(lib.g2v_lasso_workspace_bytes(G, n_pad, fits)), dtype=torch.uint8, device="cuda")
    ent = torch.empty((fits, G), dtype=torch.int16, device="cuda")
    ea = torch.empty((fits, G), dtype=torch.float64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    K, F = 1, max(2, fits - 1)
    _capi.check(lib.g2v_lasso_standardise(X.data_ptr(), G, n, n_pad, y.data_ptr(), fold.data_ptr(), K, F, 0, fits,
                                          ws.data_ptr(), ent.data_ptr(), ea.data_ptr(), st), "standardise")
    call = lambda: _capi.check(lib.g2v_lasso_grad(X.data_ptr(), G, n, n_pad, fits, ws.data_ptr(), 0.01, 1.0, st),
                               "grad")
    for _ in range(3):
        call()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); call(); b.record(); b.synchronize()
        times.append(a.elapsed_time(b))
    ms = float(np.median(times))
    return ms, 2.0 * G * n_pad * fits / (ms * 1e-3) / 1e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS))
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--cpu-lambdas", type=int, default=5)
    a = ap.parse_args()
    import torch
    from g2vec_b200 import lasso
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import lasso_oracle
    name, power, clock = card()
    for w in a.workloads:
        src, F, K = WORKLOADS[w]
        x, lab = cohort(src)
        fits = 1 + K * F
        g_ms, g_tf = grad_ms(x, lab, fits, a.iters)
        lasso.lasso_cv(x, lab, folds=F, repeats=K)                 # warm-up
        torch.cuda.synchronize()
        times = []
        for _ in range(2):
            t0 = time.perf_counter()
            res = lasso.lasso_cv(x, lab, folds=F, repeats=K)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        lasso_oracle.path(x, lab.astype(np.float64), 1.0, lams=res.lambdas[:a.cpu_lambdas])
        cpu = (time.perf_counter() - t0) / a.cpu_lambdas * res.n_lambda * fits
        print(json.dumps({"workload": w, "samples": x.shape[0], "genes": x.shape[1], "folds": F, "repeats": K,
                          "card": name, "power_limit": power, "sm_clock": clock, "grad_ms": round(g_ms, 4),
                          "grad_tflops": round(g_tf, 2), "lasso_cv_s": [round(t, 3) for t in times],
                          "n_lambda": res.n_lambda, "newton_steps": int(res.n_iter.sum()),
                          "certified": res.converged, "solutions": res.fits * res.n_lambda,
                          "cpu_oracle_s_extrapolated": round(cpu, 1), "auc_min": round(float(res.auc_mean[res.i_min]), 4)}),
              flush=True)


if __name__ == "__main__":
    main()
