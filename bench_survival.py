"""Cost of the permutation Cox score test (DESIGN.md §4.31):

* rows (g2v_surv_rows), scores (g2v_surv_scores, the risk-set scan) and tally (g2v_dcx_tally over the genes) -- each
  kernel alone on one chunk of permutations, CUDA events, warmed, median of --iters;
* survival_test -- g2vec_b200.survival_test end to end (synchronised wall time), with the host preparation
  (validation, quantisation, time order) timed on its own; the device part is the rest.

Workloads: ex_* (135 samples x 7 523 genes) with seeded times at B = 10^3 and 10^4, and a seeded TCGA-sized cohort
(1 000 x 20 000) at B = 10^4.  The scan makes rows * n * G sample steps; its achieved rate is reported in steps/s and,
at the 128-byte line of q a warp loads per step, in bytes/s against 3.35 TB/s (the loads are served mostly from L1/L2,
so this is not an HBM share).  The card name, power limit and SM clock are read in the same run.  The CPU reference is
the NumPy restatement of tests/survival_oracle.py, timed on --cpu-perms permutations and scaled linearly to B.  Writes
nothing into the tree; prints one JSON line per workload.

    python bench_survival.py [--workloads ex1e3 ex1e4 tcga] [--iters 5] [--cpu-perms 2] [--chunk 2048]
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

HBM_TBPS = 3.35
WORKLOADS = {"ex1e3": ("ex", 1_000), "ex1e4": ("ex", 10_000), "tcga": ("tcga", 10_000)}


def workload(name):
    """-> (expr [S, G] float32, time [S], event [S]), the times in months with ties and about half the events."""
    rng = np.random.Generator(np.random.PCG64(1972))
    if name == "ex":
        x = np.load(os.path.join(ROOT, "tests", "golden", "ex_expr.npz"))["expr"]
    else:
        x = rng.standard_normal((1_000, 20_000), dtype=np.float32)
    S = x.shape[0]
    return x, np.round(rng.exponential(36.0, S), 1), (rng.random(S) < 0.5).astype(np.int64)


def kernels(x, t, e, rows, iters):
    """Per-kernel median ms on one chunk of `rows` permutations."""
    import torch
    from g2vec_b200 import _capi, survival
    lib = _capi.load()
    prep = survival.prepare(x, t, e)
    n, q = prep["n"], prep["q"]
    G = q.shape[1]
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    q_d, slot_d, flags_d, a_d, c_d = (up(q.astype(np.int32)), up(prep["slot"]), up(prep["flags"]), up(prep["a"]),
                                      up(prep["c"]))
    idx = torch.empty((rows, n), dtype=torch.uint16, device="cuda")
    T = torch.empty((rows, G), dtype=torch.float64, device="cuda")
    Tobs = up(np.full(G, 1.0))
    cnt = torch.zeros(G, dtype=torch.int64, device="cuda")
    cm = torch.zeros(G, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    ms = {
        "rows": events_ms(lambda: lib.g2v_surv_rows(slot_d.data_ptr(), n, 0, 0, rows, idx.data_ptr(), st), iters),
        "scores": events_ms(lambda: lib.g2v_surv_scores(q_d.data_ptr(), n, G, idx.data_ptr(), rows, flags_d.data_ptr(),
                                                        a_d.data_ptr(), c_d.data_ptr(), T.data_ptr(), None, st), iters),
        "tally": events_ms(lambda: lib.g2v_dcx_tally(T.data_ptr(), rows, G, Tobs.data_ptr(), cnt.data_ptr(),
                                                     cm.data_ptr(), st), iters),
    }
    steps = float(rows) * n * G
    s = ms["scores"] * 1e-3
    return {"chunk_rows": rows, "kernel_ms": {k: round(v, 3) for k, v in ms.items()},
            "scan_steps_per_s": float("%.3g" % (steps / s)),
            "scan_q_line_bytes_per_s": float("%.3g" % (steps * 4 / s)),
            "scan_q_line_bytes_over_hbm_peak": round(steps * 4 / s / 1e12 / HBM_TBPS, 3),
            "T_bytes_written_per_s": float("%.3g" % (8.0 * rows * G / s))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS))
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--cpu-perms", type=int, default=2)
    ap.add_argument("--chunk", type=int, default=2048)
    args = ap.parse_args()
    import torch
    from g2vec_b200 import _capi, survival
    from tests import survival_oracle
    _capi.load()
    if not torch.cuda.is_available():
        raise SystemExit("bench_survival.py needs a GPU")
    name, power, clock = card()
    cache = {}
    for w in args.workloads:
        kind, B = WORKLOADS[w]
        if kind not in cache:
            cache[kind] = workload(kind)
        x, t, e = cache[kind]
        out = {"workload": w, "samples": int(x.shape[0]), "genes": int(x.shape[1]), "events": int(e.sum()), "B": B,
               "card": name, "power_limit": power, "sm_clock": clock}
        out.update(kernels(x, t, e, min(B, args.chunk), args.iters))
        survival.survival_test(x, t, e, min(B, 100), seed=1)                # warm every shape
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        survival.prepare(x, t, e, B)
        host = time.perf_counter() - t0
        t0 = time.perf_counter()
        survival.survival_test(x, t, e, B, seed=1)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        out.update({"survival_test_s": round(wall, 3), "host_prepare_s": round(host, 3),
                    "device_and_rest_s": round(wall - host, 3)})
        t0 = time.perf_counter()
        survival_oracle.survival_test(x, t, e, args.cpu_perms, seed=1)
        cpu = time.perf_counter() - t0
        out.update({"numpy_oracle_s_for_%d_perms" % args.cpu_perms: round(cpu, 2),
                    "numpy_oracle_s_scaled_to_B": round(cpu * B / args.cpu_perms, 1)})
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
