"""Cost of the exact cosine nearest-genes search (DESIGN.md §4.25):

* norms, partial, merge -- each kernel alone, CUDA events, warmed, median of --iters;
* search               -- the three kernels back to back (what nearest_genes launches), CUDA events, median;
* nearest_genes        -- g2vec_b200.nearest_genes end to end with the upload and the copy back (synchronised wall
                          time), once after a warm call.

Sizes m x D: 2 835 x 128 (about the ex_* scale), 20 000 x 128, 20 000 x 512 and 200 000 x 512 (the gene-slab trainer's
table), at K = 10 on seeded Gaussian vectors.  The FP64 rate is 2 m^2 D / t of the search, against the H100 SXM data
sheet's 34 TFLOP/s FP64 (non-tensor) at 700 W; the card name, power limit and SM clock are read in the same run.  The CPU
reference, at the smallest size only, is NumPy float64 (W W^T in row blocks, then argpartition / argsort per block) on
the host.  Writes nothing into the tree; prints one JSON line per size.

    python bench_neighbors.py [--sizes 2835x128 20000x128 20000x512 200000x512] [--k 10] [--iters 5]
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

FP64_TFLOPS = 34.0
SIZES = ["2835x128", "20000x128", "20000x512", "200000x512"]


def events_ms(fn, iters):
    import torch
    fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record(); fn(); b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def cpu_reference_s(W, k, block=1024):
    """NumPy float64 on the host: cosines of a row block against all rows, top k by argpartition + argsort."""
    t0 = time.perf_counter()
    X = W.astype(np.float64)
    X /= np.maximum(np.linalg.norm(X, axis=1), 1e-300)[:, None]
    m = X.shape[0]
    for r0 in range(0, m, block):
        s = X[r0:r0 + block] @ X.T
        s[np.arange(s.shape[0]), np.arange(r0, r0 + s.shape[0])] = -np.inf
        part = np.argpartition(-s, k, axis=1)[:, :k]
        np.take_along_axis(s, part, axis=1).argsort(axis=1)
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", nargs="+", default=SIZES)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import torch
    from g2vec_b200 import _capi, neighbors
    lib = _capi.load()
    name, power, clock = card()
    K = args.k
    for size in args.sizes:
        m, D = (int(x) for x in size.split("x"))
        W = np.random.Generator(np.random.PCG64(2025)).standard_normal((m, D), dtype=np.float32)
        splits = int(lib.g2v_nbr_splits(m))
        Wd = torch.from_numpy(W).cuda()
        inv = torch.empty(m, dtype=torch.float64, device="cuda")
        idx = torch.empty((m, K), dtype=torch.int32, device="cuda")
        sim = torch.empty((m, K), dtype=torch.float64, device="cuda")
        if splits > 1:
            pidx = torch.empty((splits, m, K), dtype=torch.int32, device="cuda")
            psim = torch.empty((splits, m, K), dtype=torch.float64, device="cuda")
        else:
            pidx, psim = idx, sim
        st = torch.cuda.current_stream().cuda_stream
        norms = lambda: _capi.check(lib.g2v_nbr_norms(Wd.data_ptr(), m, D, inv.data_ptr(), st), "norms")
        partial = lambda: _capi.check(lib.g2v_nbr_partial(Wd.data_ptr(), inv.data_ptr(), m, D, K, pidx.data_ptr(),
                                                          psim.data_ptr(), st), "partial")
        merge = lambda: _capi.check(lib.g2v_nbr_merge(pidx.data_ptr(), psim.data_ptr(), splits, m, K, idx.data_ptr(),
                                                      sim.data_ptr(), st), "merge")

        def search():
            norms(); partial()
            if splits > 1:
                merge()
        iters = args.iters if m * m * D < 1e12 else max(2, args.iters // 2)
        norms_ms = events_ms(norms, iters)
        partial_ms = events_ms(partial, iters)
        merge_ms = events_ms(merge, iters) if splits > 1 else 0.0
        search_ms = events_ms(search, iters)
        neighbors.nearest_genes(W[:100], K)                                   # warm
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        neighbors.nearest_genes(W, K)
        torch.cuda.synchronize()
        wall_ms = (time.perf_counter() - t0) * 1e3
        flops = 2.0 * m * m * D
        rate = flops / (search_ms * 1e-3) / 1e12
        cpu_s = cpu_reference_s(W, K) if size == args.sizes[0] else None
        print(json.dumps({
            "m": m, "D": D, "K": K, "splits": splits,
            "norms_ms": round(norms_ms, 3), "partial_ms": round(partial_ms, 3), "merge_ms": round(merge_ms, 3),
            "search_ms": round(search_ms, 3), "nearest_genes_wall_ms": round(wall_ms, 1),
            "fp64_TFLOPs": round(rate, 2), "share_of_fp64_datasheet": round(rate / FP64_TFLOPS, 3),
            "datasheet_bound_ms": round(flops / (FP64_TFLOPS * 1e12) * 1e3, 3),
            "cpu_numpy_float64_s": None if cpu_s is None else round(cpu_s, 3),
            "gpu": name, "power_limit": power, "sm_clock": clock}), flush=True)
        del Wd, inv, idx, sim, pidx, psim
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
