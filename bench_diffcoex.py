"""Cost of the differential co-expression test (DESIGN.md §4.30):

* perm_sums (A), sums_diag (B = sums of q^2), sums_D (the DMMA kernel with the fused D epilogue), tally -- each kernel
  alone on one chunk of permutations, CUDA events, warmed, median of --iters;
* diffcoex_test -- g2vec_b200.diffcoex_test end to end (synchronised wall time), with the host preparation
  (validation, quantisation) timed on its own; the device part is the rest.

Workloads: ex_* (135 samples x 7 523 genes, E = 140 902 pairs of the example network) at B = 10^3 and 10^4, and a
seeded TCGA-sized cohort (1 000 x 20 000, E = 5 * 10^5 random pairs) at B = 10^4.  Rates from the shapes: sums_D does
2 * rows * S_pad * E flop, reported against the data sheet's FP64 tensor-core rate of the H100 SXM (67 TFLOP/s at
700 W); D is written by sums_D and read by tally, 16 * rows * E bytes, reported against 3.35 TB/s.  The card name,
power limit and SM clock are read in the same run.  The CPU reference is the NumPy restatement of
tests/diffcoex_oracle.py, timed on --cpu-perms permutations and scaled linearly to B.  Writes nothing into the tree;
prints one JSON line per workload.

    python bench_diffcoex.py [--workloads ex1e3 ex1e4 tcga] [--iters 5] [--cpu-perms 2] [--chunk 2048]
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

FP64_TC_TFLOPS = 67.0
HBM_TBPS = 3.35
WORKLOADS = {"ex1e3": ("ex", 1_000), "ex1e4": ("ex", 10_000), "tcga": ("tcga", 10_000)}


def workload(name):
    """-> (expr [S, G] float32, label [S], pairs [E, 2] int32)"""
    from g2vec_b200 import diffcoex
    if name == "ex":
        e = np.load(os.path.join(ROOT, "tests", "golden", "ex_expr.npz"))
        lab = np.load(os.path.join(ROOT, "tests", "golden", "ex_graph.npz"))["label"]
        return e["expr"], lab, diffcoex.pairs_from_edges(e["src"], e["dst"])
    S, G, E = 1_000, 20_000, 500_000
    rng = np.random.Generator(np.random.PCG64(1921))
    x = rng.standard_normal((S, G), dtype=np.float32)
    lab = (rng.random(S) < 0.4).astype(np.int64)
    pairs = diffcoex.pairs_from_edges(rng.integers(0, G, 2 * E), rng.integers(0, G, 2 * E))
    pairs = pairs[np.sort(rng.permutation(len(pairs))[:E])]
    return x, lab, pairs


def kernels(x, lab, pairs, rows, iters):
    """Per-kernel median ms on one chunk of `rows` permutations."""
    import torch
    from g2vec_b200 import _capi, diffcoex, perm
    lib = _capi.load()
    prep = diffcoex.prepare(x, lab, pairs)
    n, k, q = prep["n"], prep["k"], prep["q"]
    G, E = q.shape[1], pairs.shape[0]
    S_pad = -(-n // 32) * 32
    qt = np.zeros((G, S_pad), np.int32); qt[:, :n] = q.T
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    q_d, pl_d, obs_d = up(qt), up(perm.planes(q, np.arange(G))), up(prep["obs"])
    diag = up(np.arange(G, dtype=np.int32))
    pi, pj = up(pairs[:, 0]), up(pairs[:, 1])
    At, Bt, Pt = up(q.sum(axis=0)), up((q * q).sum(axis=0)), up(np.zeros(E, np.int64))
    M = torch.empty((rows, S_pad), dtype=torch.uint8, device="cuda")
    A = torch.empty((rows, G), dtype=torch.int64, device="cuda")
    Bq = torch.empty((rows, G), dtype=torch.int64, device="cuda")
    D = torch.empty((rows, E), dtype=torch.float64, device="cuda")
    Dobs = up(np.full(E, 0.5))
    cnt = torch.zeros(E, dtype=torch.int64, device="cuda")
    cm = torch.zeros(E, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    _capi.check(lib.g2v_perm_labels(obs_d.data_ptr(), n, S_pad, 0, 0, rows, M.data_ptr(), st), "labels")
    ms = {
        "perm_sums": events_ms(lambda: lib.g2v_perm_sums(M.data_ptr(), pl_d.data_ptr(), rows, S_pad, G, A.data_ptr(),
                                                         st), iters),
        "sums_diag": events_ms(lambda: lib.g2v_dcx_sums(M.data_ptr(), rows, S_pad, q_d.data_ptr(), G, diag.data_ptr(),
                                                        diag.data_ptr(), G, 0, 0, None, None, None, None, None,
                                                        Bq.data_ptr(), None, st), iters),
        "sums_D": events_ms(lambda: lib.g2v_dcx_sums(M.data_ptr(), rows, S_pad, q_d.data_ptr(), G, pi.data_ptr(),
                                                     pj.data_ptr(), E, n, k, A.data_ptr(), Bq.data_ptr(),
                                                     At.data_ptr(), Bt.data_ptr(), Pt.data_ptr(), None, D.data_ptr(),
                                                     st), iters),
        "tally": events_ms(lambda: lib.g2v_dcx_tally(D.data_ptr(), rows, E, Dobs.data_ptr(), cnt.data_ptr(),
                                                     cm.data_ptr(), st), iters),
    }
    flop = 2.0 * rows * S_pad * E
    d_bytes = 16.0 * rows * E
    t = ms["sums_D"] * 1e-3
    return {"chunk_rows": rows, "kernel_ms": {k_: round(v, 3) for k_, v in ms.items()},
            "sums_D_tflops": round(flop / t / 1e12, 2), "sums_D_share_of_fp64_tc_peak": round(flop / t / 1e12 / FP64_TC_TFLOPS, 3),
            "D_round_trip_share_of_hbm": round(d_bytes / ((ms["sums_D"] + ms["tally"]) * 1e-3) / 1e12 / HBM_TBPS, 3),
            "sums_D_flop_per_D_byte": round(flop / d_bytes, 1),
            "sums_D_bound": "compute" if flop / (FP64_TC_TFLOPS * 1e12) >= d_bytes / 2 / (HBM_TBPS * 1e12) else "memory"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS))
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--cpu-perms", type=int, default=2)
    ap.add_argument("--chunk", type=int, default=2048)
    args = ap.parse_args()
    import torch
    from g2vec_b200 import _capi, diffcoex
    from tests import diffcoex_oracle
    _capi.load()
    if not torch.cuda.is_available():
        raise SystemExit("bench_diffcoex.py needs a GPU")
    name, power, clock = card()
    cache = {}
    for w in args.workloads:
        kind, B = WORKLOADS[w]
        if kind not in cache:
            cache[kind] = workload(kind)
        x, lab, pairs = cache[kind]
        out = {"workload": w, "samples": int(x.shape[0]), "genes": int(x.shape[1]), "pairs": int(pairs.shape[0]),
               "B": B, "card": name, "power_limit": power, "sm_clock": clock}
        out.update(kernels(x, lab, pairs, min(B, args.chunk), args.iters))
        diffcoex.diffcoex_test(x, lab, pairs, min(B, 100), seed=1)          # warm every shape
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        diffcoex.prepare(x, lab, pairs, B)
        host = time.perf_counter() - t0
        t0 = time.perf_counter()
        diffcoex.diffcoex_test(x, lab, pairs, B, seed=1)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        out.update({"diffcoex_test_s": round(wall, 3), "host_prepare_s": round(host, 3),
                    "device_and_rest_s": round(wall - host, 3)})
        t0 = time.perf_counter()
        diffcoex_oracle.diffcoex_test(x, lab, pairs, args.cpu_perms, seed=1)
        cpu = time.perf_counter() - t0
        out.update({"numpy_oracle_s_for_%d_perms" % args.cpu_perms: round(cpu, 2),
                    "numpy_oracle_s_scaled_to_B": round(cpu * B / args.cpu_perms, 1)})
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
