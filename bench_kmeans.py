"""Cost of the best-of-R k-means restarts (DESIGN.md §4.26):

* assign, blocks, update, seed, contingency, agree -- each kernel alone over R restarts, CUDA events, warmed, median of
                                                     --iters (assign with all 3 centres: one Lloyd assignment pass);
* iteration    -- assign + blocks + update back to back (one Lloyd iteration of every restart), CUDA events, median;
* kmeans_lgroups -- g2vec_b200.kmeans_lgroups end to end with the upload, the per-iteration synchronisations and the
                    copies back (synchronised wall time), once after a warm call; with its mean n_iter;
* sklearn      -- scikit-learn's KMeans(3, n_init=1) and (n_init=10) on the same data on the host cores.

Sizes n x D: 20 000 x 128, 20 000 x 512 and 200 000 x 512, R in {1, 10, 100}, on seeded Gaussian vectors.  The assign
pass does 3 n D 3R FP64 operations (a sub, a mul and an add per row, centre and d); its rate is reported against the
H100 SXM data sheet's 34 TFLOP/s FP64 (non-tensor) at 700 W.  The card name, power limit and SM clock are read in the
same run.  Writes nothing into the tree; prints one JSON line per size and R.

    python bench_kmeans.py [--sizes 20000x128 20000x512 200000x512] [--restarts 1 10 100] [--iters 5] [--no-sklearn]
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
from bench_neighbors import events_ms, FP64_TFLOPS  # noqa: E402

SIZES = ["20000x128", "20000x512", "200000x512"]


def sklearn_s(W, n_init):
    from sklearn.cluster import KMeans
    t0 = time.perf_counter()
    KMeans(n_clusters=3, random_state=0, n_init=n_init).fit(W)
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", nargs="+", default=SIZES)
    ap.add_argument("--restarts", nargs="+", type=int, default=[1, 10, 100])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--no-sklearn", action="store_true")
    args = ap.parse_args()
    import torch
    from g2vec_b200 import _capi, kmeans
    lib = _capi.load()
    name, power, clock = card()
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    for size in args.sizes:
        n, D = (int(x) for x in size.split("x"))
        nb = -(-n // kmeans.BLOCK)
        W = np.random.Generator(np.random.PCG64(2026)).standard_normal((n, D), dtype=np.float32)
        Wd = torch.from_numpy(W).to(dev)
        sk = {} if args.no_sklearn else {"sklearn_n_init_1_s": round(sklearn_s(W, 1), 2),
                                         "sklearn_n_init_10_s": round(sklearn_s(W, 10), 2)}
        for R in args.restarts:
            p = lambda t: t.data_ptr()
            rs = np.random.RandomState(R)
            centres = torch.from_numpy(W[rs.randint(0, n, size=(R, 3))].astype(np.float64)).to(dev)
            active = torch.arange(R, dtype=torch.int32, device=dev)
            labels = torch.full((R, n), -1, dtype=torch.int8, device=dev)
            mind = torch.empty((R, n), dtype=torch.float64, device=dev)
            psum = torch.empty((R, nb, 3, D), dtype=torch.float64, device=dev)
            pcnt = torch.empty((R, nb, 3), dtype=torch.int32, device=dev)
            pin = torch.empty((R, nb), dtype=torch.float64, device=dev)
            flags = torch.zeros(R, dtype=torch.int32, device=dev)
            state = torch.zeros(R, dtype=torch.int32, device=dev)
            inertia = torch.empty(R, dtype=torch.float64, device=dev)
            n_iter = torch.empty(R, dtype=torch.int32, device=dev)
            seeds = torch.empty((R, 3), dtype=torch.int32, device=dev)
            table = torch.zeros((R, 9), dtype=torch.int64, device=dev)
            perm = torch.zeros((R, 3), dtype=torch.int8, device=dev)
            count = torch.zeros(n, dtype=torch.int32, device=dev)
            best = torch.zeros(n, dtype=torch.int8, device=dev)
            assign = lambda: _capi.check(lib.g2v_km_assign(p(Wd), n, D, p(centres), 3, p(active), R, p(labels),
                                                           p(mind), p(flags), st), "assign")
            blocks = lambda: _capi.check(lib.g2v_km_blocks(p(Wd), p(labels), p(mind), n, D, p(active), R, p(psum),
                                                           p(pcnt), p(pin), st), "blocks")
            update = lambda: _capi.check(lib.g2v_km_update(p(Wd), p(mind), p(psum), p(pcnt), p(pin), n, D, p(active),
                                                           R, 2, 300, p(flags), p(centres), p(state), p(inertia),
                                                           p(n_iter), st), "update")
            seed = lambda: _capi.check(lib.g2v_km_seed(p(Wd), n, D, p(mind), 0, 0, 2, R, p(centres), p(seeds), st),
                                       "seed")
            cont = lambda: _capi.check(lib.g2v_km_contingency(p(labels), p(best), n, R, p(table), st), "contingency")
            agree = lambda: _capi.check(lib.g2v_km_agree(p(labels), p(best), p(perm), n, R, p(count), st), "agree")

            def iteration():
                assign(); blocks(); update()
            assign()                                            # labels in [0, 3) before the other passes read them
            t = {k: events_ms(f, args.iters) for k, f in (("assign", assign), ("blocks", blocks), ("update", update),
                                                          ("iteration", iteration), ("seed", seed),
                                                          ("contingency", cont), ("agree", agree))}
            del labels, mind, psum, pcnt, pin
            torch.cuda.empty_cache()
            kmeans.kmeans_lgroups(W[:1000], min(R, 4), seed=0)       # warm
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = kmeans.kmeans_lgroups(W, R, seed=0)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            flops = 3.0 * n * D * 3 * R
            rate = flops / (t["assign"] * 1e-3) / 1e12
            print(json.dumps(dict(
                {"n": n, "D": D, "R": R},
                **{k + "_ms": round(v, 3) for k, v in t.items()},
                assign_fp64_TFLOPs=round(rate, 2), assign_share_of_fp64_datasheet=round(rate / FP64_TFLOPS, 3),
                assign_datasheet_bound_ms=round(flops / (FP64_TFLOPS * 1e12) * 1e3, 3),
                kmeans_lgroups_s=round(wall, 3), mean_n_iter=round(float(res.n_iter.mean()), 1),
                reach=res.reach, **sk, gpu=name, power_limit=power, sm_clock=clock)), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
