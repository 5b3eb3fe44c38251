"""Cost of the survival CV (DESIGN.md §4.33), with the signature test (§4.29) at the same sizes beside it:

* folds, draw, fit, concordance -- each kernel alone on the whole workload (one chunk of all S = R + 3 signatures),
  CUDA events, warmed, median of --iters; sig_fit and sig_auc the same way on the same sizes (S = R + 2);
* survival_cv, signature_cv     -- end to end (synchronised wall time), host preparation included.

Workloads (n, G, p, R), K = 10, F = 5: the ex cohort (135 x 7 523, tests/golden) with p = 100, R = 1 000 and the
seeded survival table bench_survival.py makes; a seeded 1 000 x 20 000 cohort with p = 100 and R = 1 000 or 10 000.
From the shapes and the fits' Newton iteration counts the JSON gives the useful FP64 operations of the two Grams per
Gram pass, 2 n_train (p+1)(p+2)/2 for sum omega z z^T and 2 n_events (p+1)(p+2)/2 for sum d m m^T (an upper bound on
the groups with events), over the fit kernel's time, and the microseconds per fit and per Newton iteration of both
fits.  The card name and power limit are read in the same run.  Writes nothing into the tree; prints one JSON line per
workload.

    python bench_survival_cv.py [--workloads ex 1000x20000x100x1000 1000x20000x100x10000] [--iters 5]
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


def workload(name):
    """-> (x [n, G], time [n], event [n], label [n], p, R)"""
    rng = np.random.Generator(np.random.PCG64(1972))
    if name == "ex":
        x = np.load(os.path.join(ROOT, "tests", "golden", "ex_expr.npz"))["expr"]
        lab = np.load(os.path.join(ROOT, "tests", "golden", "ex_graph.npz"))["label"]
        p, R = 100, 1000
    else:
        n, G, p, R = (int(v) for v in name.split("x"))
        x = rng.standard_normal((n, G), dtype=np.float32)
        lab = (rng.random(n) < 0.4).astype(np.int64)
    S = x.shape[0]
    return x, np.round(rng.exponential(36.0, S), 1), (rng.random(S) < 0.5).astype(np.int64), lab, p, R


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["ex", "1000x20000x100x1000", "1000x20000x100x10000"])
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import torch
    from g2vec_b200 import _capi, signature, survival
    from g2vec_b200 import survival_cv as scv
    if not torch.cuda.is_available():
        raise SystemExit("bench_survival_cv.py needs a GPU")
    lib = _capi.load()
    name, power, clock = card()
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    for wl in args.workloads:
        x, t, e, lab, p, R = workload(wl)
        sig = np.arange(p) * (x.shape[1] // p)
        out = {"workload": wl, "n": x.shape[0], "G": x.shape[1], "p": p, "R": R, "K": K, "F": F,
               "gpu": name, "power_limit": power, "sm_clock": clock}
        for fn, label in ((lambda: scv.survival_cv(x, t, e, lab, sig, R, folds=F, repeats=K, seed=1), "survival_cv_s"),
                          (lambda: signature.signature_cv(x, lab, sig, R, folds=F, repeats=K, seed=1),
                           "signature_cv_s")):
            fn()                                                           # warm-up of every shape
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = fn()
            torch.cuda.synchronize()
            out[label] = round(time.perf_counter() - t0, 3)
            if label == "survival_cv_s":
                scv_res = res
            else:
                sig_res = res
        # ---- the kernels alone, on the survival CV's own layout
        xs, ts, es = x.astype(np.float64), t, e
        n, G = xs.shape
        order, _, flags, _, _ = survival.time_groups(ts, es)
        grp = np.cumsum(np.r_[0, (flags & 2)[:-1] > 0]).astype(np.int32)
        n_pad = -(-n // 32) * 32
        Xt = np.zeros((G, n_pad)); Xt[:, :n] = xs[order].T
        X_d = torch.from_numpy(Xt).to(dev)
        del Xt
        fl_d = torch.from_numpy(flags).to(dev)
        gr_d = torch.from_numpy(grp).to(dev)
        ev_d = torch.from_numpy((flags & 1).astype(np.uint8)).to(dev)
        fold_d = torch.empty((K, n), dtype=torch.int8, device=dev)
        S = R + 3
        g_d = torch.from_numpy(scv_res.genes).to(dev)
        gr_r = torch.empty((R, p), dtype=torch.int32, device=dev)
        sc = torch.empty((S, K, n), dtype=torch.float64, device=dev)
        ell = torch.empty((S * K * F, n), dtype=torch.float64, device=dev)
        it = torch.empty((S, K, F), dtype=torch.int32, device=dev)
        cv = torch.empty((S, K, F), dtype=torch.uint8, device=dev)
        cnt = torch.empty((S, K, F, 3), dtype=torch.int64, device=dev)
        n_ev = int(es.sum())
        cap = -(-n_ev // F) + -(-(n - n_ev) // F)
        t_folds = events_ms(lambda: _capi.check(lib.g2v_sig_folds(ev_d.data_ptr(), n, K, F, 1, fold_d.data_ptr(), st),
                                                "folds"), args.iters)
        t_draw = events_ms(lambda: _capi.check(lib.g2v_sig_draw(G, p, 1, 1, R, gr_r.data_ptr(), st), "draw"),
                           args.iters)
        t_fit = events_ms(lambda: _capi.check(lib.g2v_cox_fit(
            X_d.data_ptr(), G, n, n_pad, fl_d.data_ptr(), fold_d.data_ptr(), K, F, g_d.data_ptr(), S, p,
            ell.data_ptr(), sc.data_ptr(), it.data_ptr(), cv.data_ptr(), None, 0, st), "fit"), args.iters)
        t_conc = events_ms(lambda: _capi.check(lib.g2v_cox_concordance(
            sc.data_ptr(), fl_d.data_ptr(), gr_d.data_ptr(), fold_d.data_ptr(), n, K, F, S, cap, cnt.data_ptr(), st),
            "concordance"), args.iters)
        assert (cnt.cpu().numpy() == scv_res.counts).all() and (it.cpu().numpy() == scv_res.n_iter).all()
        del ell, sc
        # ---- the signature test's fit and AUC at the same sizes
        used = (lab == 0) | (lab == 1)
        xl, yl = x[used].astype(np.float64), lab[used]
        nl = xl.shape[0]
        nl_pad = -(-nl // 32) * 32
        Xl = np.zeros((G, nl_pad)); Xl[:, :nl] = xl.T
        Xl_d = torch.from_numpy(Xl).to(dev)
        del Xl
        y_d = torch.from_numpy(yl.astype(np.uint8)).to(dev)
        fl2 = torch.from_numpy(sig_res.folds).to(dev)
        Ss = R + 2
        gs_d = torch.from_numpy(sig_res.genes).to(dev)
        sc2 = torch.empty((Ss, K, nl), dtype=torch.float64, device=dev)
        it2 = torch.empty((Ss, K, F), dtype=torch.int32, device=dev)
        cv2 = torch.empty((Ss, K, F), dtype=torch.uint8, device=dev)
        t_sfit = events_ms(lambda: _capi.check(lib.g2v_sig_fit(
            Xl_d.data_ptr(), G, nl, nl_pad, y_d.data_ptr(), fl2.data_ptr(), K, F, gs_d.data_ptr(), Ss, p,
            sc2.data_ptr(), it2.data_ptr(), cv2.data_ptr(), None, 0, st), "sig_fit"), args.iters)
        del Xl_d, sc2
        n_train = np.array([[n - int((scv_res.folds[k] == f).sum()) for f in range(F)] for k in range(K)])
        iters = scv_res.n_iter.astype(np.float64)
        ev_train = np.array([[n_ev - int(((scv_res.folds[k] == f) & (es == 1)).sum()) for f in range(F)]
                             for k in range(K)])
        tri = (p + 1) * (p + 2) / 2
        gram_flop = float((2.0 * (n_train + ev_train)[None] * tri * iters).sum())
        fits, sfits = S * K * F, Ss * K * F
        out.update({
            "kernel_ms": {"folds": round(t_folds, 4), "draw": round(t_draw, 4), "cox_fit": round(t_fit, 3),
                          "concordance": round(t_conc, 4), "sig_fit": round(t_sfit, 3)},
            "fits": fits, "us_per_fit": round(t_fit * 1e3 / fits, 3),
            "mean_newton_iterations": round(float(iters.mean()), 3), "not_converged": fits - scv_res.converged,
            "us_per_iteration": round(t_fit * 1e3 / float(iters.sum()), 3),
            "gram_tflops": round(gram_flop / (t_fit * 1e-3) / 1e12, 3),
            "signature_fit": {"fits": sfits, "us_per_fit": round(t_sfit * 1e3 / sfits, 3),
                              "mean_newton_iterations": round(float(sig_res.n_iter.mean()), 3),
                              "us_per_iteration": round(t_sfit * 1e3 / float(sig_res.n_iter.sum()), 3)},
            "c": {"biomarkers": round(float(scv_res.c_mean[0]), 4), "top_t": round(float(scv_res.c_mean[1]), 4),
                  "top_z": round(float(scv_res.c_mean[2]), 4), "random_mean": round(float(scv_res.c_mean[3:].mean()), 4)},
        })
        print(json.dumps(out), flush=True)
        del X_d


if __name__ == "__main__":
    main()
