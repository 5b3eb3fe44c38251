"""Cost of the NetRank test (DESIGN.md §4.35):

* seed, step and tally -- each kernel alone on one chunk of permutations, CUDA events, warmed, median of --iters; the
  step as T iterations over the chunk in column tiles that fit the L2 (what netrank_test runs) and as T iterations
  over the whole chunk in one tile, each reported per iteration;
* netrank_test -- g2vec_b200.netrank_test end to end (synchronised wall time).

Workloads: ex_* (135 samples x 7 523 genes, 140 902 pairs of the example network) at B = 10^3 and 10^4 with d = 0.5
and 0.9, and a seeded TCGA-sized cohort (1 000 x 20 000, 5 * 10^5 random pairs) at B = 10^4, d = 0.5.  The step's byte
model counts, per iteration and column, the gathered neighbour values (8 bytes per CSR entry), S read and x written
(16 bytes per gene), and reports the rate over the step time; the CSR itself (12 bytes per entry, shared by the 32
columns of a warp) is left out.  The card name, power limit and SM clock are read in the same run.  The CPU reference
is the NumPy restatement of tests/netrank_oracle.py, timed on --cpu-perms permutations and scaled linearly to B.
Writes nothing into the tree; prints one JSON line per workload.

    python bench_netrank.py [--workloads ex1e3 ex1e4 ex1e3_d09 ex1e4_d09 tcga] [--iters 5] [--cpu-perms 2]
                            [--chunk 2048]
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
from bench_diffcoex import workload  # noqa: E402
from bench_perm import events_ms  # noqa: E402

WORKLOADS = {"ex1e3": ("ex", 1_000, 0.5), "ex1e4": ("ex", 10_000, 0.5), "ex1e3_d09": ("ex", 1_000, 0.9),
             "ex1e4_d09": ("ex", 10_000, 0.9), "tcga": ("tcga", 10_000, 0.5)}


def kernels(x, lab, pairs, rows, d, iters):
    """Per-kernel median ms on one chunk of `rows` permutations."""
    import torch
    from g2vec_b200 import _capi, netrank, perm
    lib = _capi.load()
    x, lab, pairs = netrank.check_inputs(x, lab, pairs, rows, d)
    prep = perm.prepare(x, lab)
    n, k, G = prep["n"], prep["k"], x.shape[1]
    S_pad = -(-n // 32) * 32
    ld = -(-rows // 32) * 32
    rowptr, col, deg, w = netrank.csr(pairs, G)
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    net = (up(rowptr), up(col), up(w), up(netrank.row_order(deg)))
    pl_d, Q_d, W_d, obs_d = up(perm.planes(prep["q"], np.arange(G))), up(prep["Q"]), up(prep["W"]), up(prep["obs"])
    M = torch.empty((rows, S_pad), dtype=torch.uint8, device="cuda")
    A = torch.empty((rows, G), dtype=torch.int64, device="cuda")
    S, xa, xb = (torch.empty((G, ld), dtype=torch.float64, device="cuda") for _ in range(3))
    obs_score = up(np.full(G, 0.5))
    cnt = torch.zeros(G, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    _capi.check(lib.g2v_perm_labels(obs_d.data_ptr(), n, S_pad, 0, 0, rows, M.data_ptr(), st), "labels")
    _capi.check(lib.g2v_perm_sums(M.data_ptr(), pl_d.data_ptr(), rows, S_pad, G, A.data_ptr(), st), "sums")
    T = netrank.n_iterations(d)
    tile = int(lib.g2v_nr_tile_cols(G))
    ms = {
        "seed": events_ms(lambda: lib.g2v_nr_seed(A.data_ptr(), rows, G, n, k, Q_d.data_ptr(), W_d.data_ptr(),
                                                  S.data_ptr(), ld, st), iters),
        "step_l2_tiles": events_ms(lambda: netrank.propagate(lib, net, S, xa, xb, G, ld, rows, T, d, tile, st),
                                   iters) / T,
        "step_one_tile": events_ms(lambda: netrank.propagate(lib, net, S, xa, xb, G, ld, rows, T, d, ld, st),
                                   iters) / T,
        "tally": events_ms(lambda: lib.g2v_nr_tally(xa.data_ptr(), G, rows, ld, obs_score.data_ptr(), cnt.data_ptr(),
                                                    st), iters),
    }
    nnz = int(rowptr[-1])
    step_bytes = (8.0 * nnz + 16.0 * G) * rows
    return {"chunk_rows": rows, "T": T, "tile_cols": tile, "nnz": nnz, "max_degree": int(deg.max()),
            "kernel_ms": {k_: round(v, 4) for k_, v in ms.items()},
            "step_model_bytes": step_bytes,
            "step_l2_tiles_GBps": round(step_bytes / (ms["step_l2_tiles"] * 1e-3) / 1e9, 1),
            "step_one_tile_GBps": round(step_bytes / (ms["step_one_tile"] * 1e-3) / 1e9, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS))
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--cpu-perms", type=int, default=2)
    ap.add_argument("--chunk", type=int, default=2048)
    args = ap.parse_args()
    import torch
    from g2vec_b200 import _capi, netrank
    from tests import netrank_oracle
    _capi.load()
    if not torch.cuda.is_available():
        raise SystemExit("bench_netrank.py needs a GPU")
    name, power, clock = card()
    cache = {}
    for wl in args.workloads:
        kind, B, d = WORKLOADS[wl]
        if kind not in cache:
            cache[kind] = workload(kind)
        x, lab, pairs = cache[kind]
        out = {"workload": wl, "samples": int(x.shape[0]), "genes": int(x.shape[1]), "pairs": int(pairs.shape[0]),
               "B": B, "damping": d, "card": name, "power_limit": power, "sm_clock": clock}
        out.update(kernels(x, lab, pairs, min(B, args.chunk), d, args.iters))
        netrank.netrank_test(x, lab, pairs, min(B, 100), damping=d, seed=1)          # warm every shape
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        netrank.netrank_test(x, lab, pairs, B, damping=d, seed=1)
        torch.cuda.synchronize()
        out["netrank_test_s"] = round(time.perf_counter() - t0, 3)
        t0 = time.perf_counter()
        netrank_oracle.netrank_test(x, lab, pairs, args.cpu_perms, damping=d, seed=1)
        cpu = time.perf_counter() - t0
        out.update({"numpy_oracle_s_for_%d_perms" % args.cpu_perms: round(cpu, 2),
                    "numpy_oracle_s_scaled_to_B": round(cpu * B / args.cpu_perms, 1)})
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
