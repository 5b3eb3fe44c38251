"""Cost of the edge-weight coefficients (DESIGN.md §4.22): for pearson, spearman and bicor,

* transform -- the per-gene transform alone (g2v_pcc_zscore for pearson, g2v_corr_transform for the others), CUDA
               events, warmed, median of --iters launches;
* csr       -- graph.group_csr_gpu end to end (upload, transform, edge weights, cutoff, CSR), synchronised, median.

Workloads: ex_* (135 samples split 77/58, 7 523 genes, 216 540 edges; group 0), a TCGA-sized synthetic cohort
(V = 20 000, S = 600, E = 500 000, seeded) and a large-S case (V = 2 000, S = 32 768, E = 20 000).  Byte model from the
shapes: the transform reads S*V*4 and writes S*V*4 bytes; spearman and bicor also transpose (read + write S*V*4), so
their model is 16*S*V bytes against pearson's 8*S*V.  The card name, power limit and SM clock are read in the same run;
scipy.stats.spearmanr per edge on ex_* is timed on the CPU for scale.  Writes nothing into the tree; prints one JSON
line per (workload, method) and one for the CPU reference.

    python bench_correlation.py [--workloads ex tcga bigS] [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METHODS = ("pearson", "spearman", "bicor")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = (x.strip() for x in out.split(","))
        return name, power, clock
    except Exception as e:                                  # the numbers are still reported
        return "unknown (%s)" % type(e).__name__, "unknown", "unknown"


def workload(name):
    """-> (expr [S, V] float32 of one group, src, dst)"""
    if name == "ex":
        e = np.load(os.path.join(ROOT, "tests", "golden", "ex_expr.npz"))
        label = np.load(os.path.join(ROOT, "tests", "golden", "ex_graph.npz"))["label"]
        return e["expr"][label == 0], e["src"].astype(np.int32), e["dst"].astype(np.int32)
    V, S, E = {"tcga": (20_000, 600, 500_000), "bigS": (2_000, 32_768, 20_000)}[name]
    rng = np.random.Generator(np.random.PCG64(2012))
    # log-normal values rounded to 0.1: heavy-tailed and full of ties, as expression data is
    X = np.round(np.exp(rng.standard_normal((S, V), dtype=np.float32) * 1.5) * 10.0) / 10.0
    src = rng.integers(0, V, size=E, dtype=np.int64).astype(np.int32)
    dst = rng.integers(0, V, size=E, dtype=np.int64).astype(np.int32)
    return X.astype(np.float32), src, dst


def median_ms(fn, iters):
    import torch
    fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record(); fn(); b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def median_wall_ms(fn, iters):
    import torch
    fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(iters):
        t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def cpu_spearman_per_edge(n=2000):
    from scipy import stats
    X, src, dst = workload("ex")
    t0 = time.perf_counter()
    for a, b in zip(src[:n], dst[:n]):
        stats.spearmanr(X[:, a], X[:, b])
    us = (time.perf_counter() - t0) / n * 1e6
    return {"cpu_reference": "scipy.stats.spearmanr per edge, ex_* group 0", "us_per_edge": round(us, 2),
            "s_all_216540_edges": round(us * len(src) / 1e6, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["ex", "tcga", "bigS"])
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import torch
    from g2vec_b200 import _capi, graph
    lib = _capi.load()
    name, power, clock = card()
    for wl in args.workloads:
        X, src, dst = workload(wl)
        S, V = X.shape
        lab = np.zeros(S, np.int64)
        xd = torch.from_numpy(np.ascontiguousarray(X)).cuda()
        z = torch.empty((V, S), dtype=torch.float32, device="cuda")
        for m in METHODS:
            st = torch.cuda.current_stream().cuda_stream
            if m == "pearson":
                kern = lambda: _capi.check(lib.g2v_pcc_zscore(xd.data_ptr(), S, V, z.data_ptr(), st), "zscore")
            else:
                code = graph.CORR_METHODS[m]
                kern = lambda: _capi.check(lib.g2v_corr_transform(xd.data_ptr(), S, V, code, z.data_ptr(), st), "corr")
            ms = median_ms(kern, args.iters)
            model = (8 if m == "pearson" else 16) * S * V
            csr = median_wall_ms(lambda: graph.group_csr_gpu(X, lab, 0, src, dst, method=m), max(10, args.iters // 2))
            print(json.dumps({"workload": wl, "S": S, "V": V, "E": int(len(src)), "method": m,
                              "transform_ms": round(ms, 4), "model_bytes": model,
                              "model_GBps": round(model / (ms * 1e-3) / 1e9, 1), "group_csr_gpu_ms": round(csr, 3),
                              "gpu": name, "power_limit": power, "sm_clock": clock}), flush=True)
    print(json.dumps(cpu_spearman_per_edge()), flush=True)


if __name__ == "__main__":
    main()
