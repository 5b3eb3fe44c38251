"""Cost of the label-permutation test (DESIGN.md §4.24):

* labels, sums, tally -- each kernel alone on one chunk of B permutations, CUDA events, warmed, median of --iters;
* perm_test           -- g2vec_b200.perm_test end to end (synchronised wall time), with the host preparation
                         (validation, quantisation, observed statistics, byte planes) timed on its own.

Workloads: ex_* (135 samples x 7 523 genes), a TCGA-sized seeded cohort (1 000 x 20 000) and a large-S one
(32 768 x 2 000), at B = 10^4, and the TCGA size at B = 10^5.  Rates from the shapes: the sums kernel does
2 * 3 * B * S_pad * G integer operations (three byte planes), reported against the data sheet's dense INT8 rate of the
H100 SXM (1 979 TOPS at 700 W); the tally reads 8 * B * G bytes of sums.  The card name, power limit and SM clock are
read in the same run.  The CPU reference is NumPy permuting the labels and recomputing |t| of every gene, timed on
--cpu-perms permutations and scaled to B.  Writes nothing into the tree; prints one JSON line per workload.

    python bench_perm.py [--workloads ex tcga tcga1e5 bigS] [--iters 5] [--cpu-perms 20]
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

INT8_DENSE_TOPS = 1979.0
WORKLOADS = {"ex": (None, None, 10_000), "tcga": (1_000, 20_000, 10_000), "tcga1e5": (1_000, 20_000, 100_000),
             "bigS": (32_768, 2_000, 10_000)}


def workload(name):
    """-> (expr [S, G] float32, label [S])"""
    S, G, _ = WORKLOADS[name]
    if S is None:
        e = np.load(os.path.join(ROOT, "tests", "golden", "ex_expr.npz"))
        return e["expr"], np.load(os.path.join(ROOT, "tests", "golden", "ex_graph.npz"))["label"]
    rng = np.random.Generator(np.random.PCG64(2003))
    x = rng.standard_normal((S, G), dtype=np.float32)
    lab = (rng.random(S) < 0.4).astype(np.int64)
    x[:, : G // 100] += 0.5 * lab[:, None]               # 1 % of the genes differ between the groups
    return x, lab


def events_ms(fn, iters):
    import torch
    fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record(); fn(); b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def cpu_reference(x, lab, n_perm, B):
    """NumPy: permute the labels, recompute the pooled |t| of every gene (vectorised over genes)."""
    xs = x[(lab == 0) | (lab == 1)].astype(np.float64)
    ls = lab[(lab == 0) | (lab == 1)]
    rng = np.random.default_rng(0)
    n = len(ls)
    t0 = time.perf_counter()
    for _ in range(n_perm):
        p = rng.permutation(ls)
        a, b = xs[p == 0], xs[p == 1]
        sp = np.sqrt(((len(a) - 1) * a.var(0, ddof=1) + (len(b) - 1) * b.var(0, ddof=1)) / (n - 2))
        np.abs((a.mean(0) - b.mean(0)) / sp / np.sqrt(1 / len(a) + 1 / len(b)))
    s = time.perf_counter() - t0
    return s / n_perm * B


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS))
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--cpu-perms", type=int, default=20)
    args = ap.parse_args()
    import torch
    from g2vec_b200 import _capi, perm
    lib = _capi.load()
    name, power, clock = card()
    for wl in args.workloads:
        x, lab = workload(wl)
        B = WORKLOADS[wl][2]
        t0 = time.perf_counter()
        prep = perm.prepare(x, lab, B)
        pl = perm.planes(prep["q"], prep["order"])
        host_ms = (time.perf_counter() - t0) * 1e3
        n, k, o = prep["n"], prep["k"], prep["order"]
        G, S_pad = pl.shape[1], pl.shape[2]
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        obs, pld = dev(prep["obs"]), dev(pl)
        Q, W, aN, rho = dev(prep["Q"][o]), dev(prep["W"][o]), dev(np.abs(prep["N_obs"][o])), dev(prep["rho_obs"][o])
        rows = perm.chunk_rows(S_pad, G, B, torch.cuda.mem_get_info()[0] // 2)
        M = torch.empty((rows, S_pad), dtype=torch.uint8, device="cuda")
        A = torch.empty((rows, G), dtype=torch.int64, device="cuda")
        c, cm = torch.zeros(G, dtype=torch.int64, device="cuda"), torch.zeros(G, dtype=torch.int64, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        lab_ms = events_ms(lambda: _capi.check(lib.g2v_perm_labels(obs.data_ptr(), n, S_pad, 0, 0, rows, M.data_ptr(), st),
                                               "labels"), args.iters)
        sum_ms = events_ms(lambda: _capi.check(lib.g2v_perm_sums(M.data_ptr(), pld.data_ptr(), rows, S_pad, G,
                                                                 A.data_ptr(), st), "sums"), args.iters)
        tal_ms = events_ms(lambda: _capi.check(lib.g2v_perm_tally(A.data_ptr(), rows, G, n, k, Q.data_ptr(), W.data_ptr(),
                                                                  aN.data_ptr(), rho.data_ptr(), c.data_ptr(),
                                                                  cm.data_ptr(), st), "tally"), args.iters)
        del M, A
        torch.cuda.empty_cache()
        perm.perm_test(x, lab, min(B, 100), seed=0)      # warm
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = perm.perm_test(x, lab, B, seed=0)
        torch.cuda.synchronize()
        wall_ms = (time.perf_counter() - t0) * 1e3
        ops = 2.0 * 3 * rows * S_pad * G
        cpu_s = cpu_reference(x, lab, args.cpu_perms, B)
        print(json.dumps({
            "workload": wl, "n": n, "G": G, "S_pad": S_pad, "B": B, "chunk_rows": rows,
            "labels_ms": round(lab_ms, 3), "sums_ms": round(sum_ms, 3), "tally_ms": round(tal_ms, 3),
            "sums_TOPS": round(ops / (sum_ms * 1e-3) / 1e12, 1),
            "sums_share_of_int8_datasheet": round(ops / (sum_ms * 1e-3) / 1e12 / INT8_DENSE_TOPS, 3),
            "tally_GBps": round(8.0 * rows * G / (tal_ms * 1e-3) / 1e9, 1),
            "perm_test_wall_ms": round(wall_ms, 1), "host_prepare_ms": round(host_ms, 1),
            "genes_P_maxT_le_0.05": int((res.P_maxT <= 0.05).sum()),
            "cpu_numpy_s_scaled": round(cpu_s, 1), "cpu_perms_timed": args.cpu_perms,
            "gpu": name, "power_limit": power, "sm_clock": clock}), flush=True)


if __name__ == "__main__":
    main()
