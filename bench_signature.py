"""Cost of the signature test (DESIGN.md §4.29):

* folds, draw, fit, auc -- each kernel alone on the whole workload (one chunk of all S = R + 2 signatures), CUDA
  events, warmed, median of --iters;
* signature_cv          -- g2vec_b200.signature_cv end to end (synchronised wall time), its host preparation
  (top_t, the upload of X) included.

Workloads (n, G, p, R, K, F): the ex cohort (135 x 7 523, tests/golden) with p = 100, R = 1 000; a seeded 1 000 x
20 000 cohort with p = 100, R = 1 000 and with p = 128, R = 10 000; K = 10, F = 5 throughout.  From the shapes and the
fits' Newton iteration counts (one Gram pass per iteration) the JSON gives the Gram matrix's useful FP64 operations,
2 n_train (p+1)(p+2)/2 per pass, over the fit kernel's time and as a share of the data-sheet 67 TFLOP/s FP64 tensor-core
rate (a ratio, not a claim that the rate is reached), and the bytes of X the fit kernel must stream per fit (p n 8
bytes per pass: two for the standardisation, one per Gram pass, at least one Armijo trial per iteration, one for the
test logits) over its time.  scikit-learn's cross_val_score(make_pipeline(StandardScaler(), LogisticRegression(C=1)),
scoring="roc_auc") on the same splits is timed on --sklearn-sigs signatures on this host's cores and extrapolated to S;
the JSON says so.  The card name and power limit are read in the same run.  Writes nothing into the tree; prints one
JSON line per workload.

    python bench_signature.py [--workloads ex 1000x20000x100x1000 1000x20000x128x10000] [--iters 3]
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
from bench_perm import events_ms  # noqa: E402

K, F = 10, 5
PEAK_FP64_TC = 67e12


def workload(name):
    """-> (x [n, G], labels, p, R)"""
    if name == "ex":
        e = np.load(os.path.join(ROOT, "tests", "golden", "ex_expr.npz"))
        lab = np.load(os.path.join(ROOT, "tests", "golden", "ex_graph.npz"))["label"]
        return e["expr"], lab, 100, 1000
    n, G, p, R = (int(v) for v in name.split("x"))
    rng = np.random.Generator(np.random.PCG64(2002))
    x = rng.standard_normal((n, G), dtype=np.float32)
    lab = (rng.random(n) < 0.4).astype(np.int64)
    x[:, :200] += 0.3 * lab[:, None]
    return x, lab, p, R


def sklearn_seconds_per_signature(x, lab, genes, fold, n_sig):
    from sklearn.linear_model import LogisticRegression
    from sklearn.model_selection import cross_val_score
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler
    splits = [(np.flatnonzero(fold[k] != f), np.flatnonzero(fold[k] == f)) for k in range(K) for f in range(F)]
    pipe = make_pipeline(StandardScaler(), LogisticRegression(C=1.0))
    t0 = time.perf_counter()
    for s in range(n_sig):
        cross_val_score(pipe, x[:, genes[s]], lab, cv=splits, scoring="roc_auc")
    return (time.perf_counter() - t0) / n_sig


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["ex", "1000x20000x100x1000", "1000x20000x128x10000"])
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--sklearn-sigs", type=int, default=4)
    args = ap.parse_args()
    import torch
    from g2vec_b200 import _capi, signature
    lib = _capi.load()
    name, power, clock = card()
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    for wl in args.workloads:
        x, lab, p, R = workload(wl)
        used = (lab == 0) | (lab == 1)
        xs, ys = x[used].astype(np.float64), lab[used]
        n, G = xs.shape
        S = R + 2
        sig = np.arange(p) * (G // p)
        signature.signature_cv(x, lab, sig, R, folds=F, repeats=K, seed=1)    # warm-up of every shape
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = signature.signature_cv(x, lab, sig, R, folds=F, repeats=K, seed=1)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0

        n_pad = -(-n // 32) * 32
        Xt = np.zeros((G, n_pad)); Xt[:, :n] = xs.T
        X_d = torch.from_numpy(Xt).to(dev)
        y_d = torch.from_numpy(ys.astype(np.uint8)).to(dev)
        fold_d = torch.empty((K, n), dtype=torch.int8, device=dev)
        g_d = torch.from_numpy(res.genes).to(dev)
        gr_d = torch.empty((R, p), dtype=torch.int32, device=dev)
        sc = torch.empty((S, K, n), dtype=torch.float64, device=dev)
        it = torch.empty((S, K, F), dtype=torch.int32, device=dev)
        cv = torch.empty((S, K, F), dtype=torch.uint8, device=dev)
        auc, acc = (torch.empty((S, K, F), dtype=torch.float64, device=dev) for _ in range(2))
        cap = int(max((res.folds[k] == f).sum() for k in range(K) for f in range(F)))
        t_folds = events_ms(lambda: _capi.check(lib.g2v_sig_folds(y_d.data_ptr(), n, K, F, 1, fold_d.data_ptr(), st),
                                                "folds"), args.iters)
        t_draw = events_ms(lambda: _capi.check(lib.g2v_sig_draw(G, p, 1, 1, R, gr_d.data_ptr(), st), "draw"),
                           args.iters)
        t_fit = events_ms(lambda: _capi.check(lib.g2v_sig_fit(
            X_d.data_ptr(), G, n, n_pad, y_d.data_ptr(), fold_d.data_ptr(), K, F, g_d.data_ptr(), S, p, sc.data_ptr(),
            it.data_ptr(), cv.data_ptr(), None, 0, st), "fit"), args.iters)
        t_auc = events_ms(lambda: _capi.check(lib.g2v_sig_auc(
            sc.data_ptr(), y_d.data_ptr(), fold_d.data_ptr(), n, K, F, S, cap, auc.data_ptr(), acc.data_ptr(), st),
            "auc"), args.iters)
        assert (auc.cpu().numpy() == res.auc).all() and (it.cpu().numpy() == res.n_iter).all()
        n_train = np.array([[n - int((res.folds[k] == f).sum()) for f in range(F)] for k in range(K)])
        iters = res.n_iter.astype(np.float64)
        gram_flop = float((2.0 * n_train[None] * (p + 1) * (p + 2) / 2 * iters).sum())
        x_bytes = float((8.0 * p * n * (2 + 2 * iters + 1)).sum())
        fits = S * K * F
        sk = sklearn_seconds_per_signature(xs, ys, res.genes, res.folds, args.sklearn_sigs)
        print(json.dumps({
            "workload": wl, "n": n, "G": G, "p": p, "R": R, "K": K, "F": F, "fits": fits,
            "gpu": name, "power_limit": power, "sm_clock": clock,
            "signature_cv_s": round(wall, 3),
            "kernel_ms": {"folds": round(t_folds, 4), "draw": round(t_draw, 4), "fit": round(t_fit, 3),
                          "auc": round(t_auc, 4)},
            "mean_newton_iterations": round(float(iters.mean()), 3), "not_converged": fits - res.converged,
            "gram_tflops": round(gram_flop / (t_fit * 1e-3) / 1e12, 3),
            "gram_share_of_67_tflops": round(gram_flop / (t_fit * 1e-3) / PEAK_FP64_TC, 4),
            "x_stream_gb_per_s_at_least": round(x_bytes / (t_fit * 1e-3) / 1e9, 1),
            "us_per_fit": round(t_fit * 1e3 / fits, 3),
            "auc": {"biomarkers": round(float(res.auc_mean[0]), 4), "top_t": round(float(res.auc_mean[1]), 4),
                    "random_mean": round(float(res.auc_mean[2:].mean()), 4)},
            "sklearn_cross_val_score_s": {"timed_signatures": args.sklearn_sigs,
                                          "per_signature": round(sk, 3),
                                          "extrapolated_to_all": round(sk * S, 1),
                                          "host_cores": os.cpu_count()},
        }), flush=True)
        del X_d, sc


if __name__ == "__main__":
    main()
