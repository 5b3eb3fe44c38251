"""Cost of the exact t-SNE map (DESIGN.md §4.27):

* dist, affinity, symmetrize  -- each kernel alone (affinity on a fresh d, symmetrize on fresh c), CUDA events, median
                                 of --iters;
* grad, iteration             -- g2v_tsne_grad alone, and one iteration (g2v_tsne_grad + g2v_tsne_update), CUDA events,
                                 warmed, median of --iters;
* kl                          -- g2v_tsne_kl (a gradient pass, the row chains, the KL terms and their sum);
* tsne_map                    -- g2vec_b200.tsne_map end to end with 1000 iterations (synchronised wall time, once
                                 after a warm call), and its host PCA initialisation alone;
* sklearn                     -- scikit-learn's default TSNE (Barnes-Hut, all host cores) on the same vectors, at the
                                 sizes of --sklearn-sizes.

Sizes m x D: 3 769 (the genes in paths of the ex_* data), 10 000, 20 000 and 32 768 genes, D in {128, 512}, on seeded
Gaussian vectors.  The gradient does 19 FP64 operations per ordered pair (i, j), j != i -- 2 subs for t, 2 muls and an
add for d, an add and a reciprocal for w, 2 muls for a and r, and 5 adds and 4 muls for the chains -- and reads P once
(8 m^2 bytes).  Its rate is reported against the H100 SXM data sheet's 34 TFLOP/s FP64 (non-tensor, an FMA counted as
two operations; the contract forbids FMA, so the ceiling of this instruction mix is at most half of it) and its P
traffic against 3.35 TB/s of HBM3.  The card name, power limit and SM clock are read in the same run.  Writes nothing
into the tree; prints one JSON line per size.

    python bench_tsne.py [--sizes 3769x128 3769x512 10000x128 ...] [--iters 5] [--sklearn-sizes 3769 10000]
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

HBM_TBS = 3.35
SIZES = ["3769x128", "3769x512", "10000x128", "10000x512", "20000x128", "20000x512", "32768x128", "32768x512"]
GRAD_OPS = 19


def after_ms(prepare, fn, iters):
    """Median of CUDA-event times of fn, each run after an untimed prepare() on the same stream."""
    import torch
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    prepare(); fn()
    for a, b in ev:
        prepare()
        a.record(); fn(); b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def sklearn_s(W):
    from sklearn.manifold import TSNE
    t0 = time.perf_counter()
    TSNE(n_components=2, perplexity=30.0, random_state=0).fit_transform(W)
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", nargs="+", default=SIZES)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--sklearn-sizes", nargs="*", type=int, default=[3769, 10000])
    args = ap.parse_args()
    import torch
    from g2vec_b200 import _capi, tsne
    lib = _capi.load()
    name, power, clock = card()
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    done_sklearn = set()
    for size in args.sizes:
        m, D = (int(x) for x in size.split("x"))
        W = np.random.Generator(np.random.PCG64(2026)).standard_normal((m, D), dtype=np.float32)
        Wd = torch.from_numpy(W).to(dev)
        P = torch.empty((m, m), dtype=torch.float64, device=dev)
        beta = torch.empty(m, dtype=torch.float64, device=dev)
        steps = torch.empty(m, dtype=torch.int32, device=dev)
        ws = torch.empty(int(lib.g2v_tsne_workspace_bytes(m)) // 8, dtype=torch.float64, device=dev)
        t0 = time.perf_counter()
        Y0 = tsne.pca_init(W)
        pca_s = time.perf_counter() - t0
        Y = torch.from_numpy(Y0).to(dev)
        u = torch.zeros((m, 2), dtype=torch.float64, device=dev)
        gains = torch.ones((m, 2), dtype=torch.float64, device=dev)
        kl = torch.empty(1, dtype=torch.float64, device=dev)
        eta = tsne.learning_rate(m)
        dist = lambda: _capi.check(lib.g2v_tsne_dist(Wd.data_ptr(), m, D, P.data_ptr(), st), "dist")
        aff = lambda: _capi.check(lib.g2v_tsne_affinity(P.data_ptr(), m, 30.0, beta.data_ptr(), steps.data_ptr(), st),
                                  "affinity")
        sym = lambda: _capi.check(lib.g2v_tsne_symmetrize(P.data_ptr(), m, st), "symmetrize")
        grad = lambda: _capi.check(lib.g2v_tsne_grad(P.data_ptr(), Y.data_ptr(), m, ws.data_ptr(), st), "grad")
        update = lambda: _capi.check(lib.g2v_tsne_update(ws.data_ptr(), m, 300, eta, Y.data_ptr(), u.data_ptr(),
                                                         gains.data_ptr(), st), "update")
        klf = lambda: _capi.check(lib.g2v_tsne_kl(P.data_ptr(), Y.data_ptr(), m, ws.data_ptr(), kl.data_ptr(), st), "kl")

        def both():
            dist(); aff()

        def iteration():
            grad(); update()
        t = {"dist": events_ms(dist, args.iters), "affinity": after_ms(dist, aff, args.iters),
             "symmetrize": after_ms(both, sym, args.iters)}
        max_steps = int(steps.max().item())
        mean_steps = float(steps.double().mean().item())
        t["grad"] = events_ms(grad, args.iters)
        t["iteration"] = events_ms(iteration, args.iters)
        t["kl"] = events_ms(klf, args.iters)
        del P, ws
        torch.cuda.empty_cache()
        tsne.tsne_map(W[:600], 30.0, n_iter=20)                           # warm
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = tsne.tsne_map(W, 30.0)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        ops = float(GRAD_OPS) * m * (m - 1)
        rate = ops / (t["grad"] * 1e-3) / 1e12
        bw = 8.0 * m * m / (t["grad"] * 1e-3) / 1e12
        sk = None
        if m in args.sklearn_sizes and m not in done_sklearn:
            sk = round(sklearn_s(W), 2)
            done_sklearn.add(m)
        print(json.dumps(dict(
            {"m": m, "D": D},
            **{k + "_ms": round(v, 3) for k, v in t.items()},
            affinity_mean_steps=round(mean_steps, 1), affinity_max_steps=max_steps,
            grad_fp64_TFLOPs=round(rate, 2), grad_share_of_fp64_datasheet=round(rate / FP64_TFLOPS, 3),
            grad_P_TBs=round(bw, 2), grad_share_of_hbm=round(bw / HBM_TBS, 3),
            tsne_map_s=round(wall, 3), pca_init_s=round(pca_s, 3), kl=round(res.kl, 5),
            sklearn_barnes_hut_s=sk, host_cores=os.cpu_count(), gpu=name, power_limit=power, sm_clock=clock)),
            flush=True)
        del Wd, Y, u, gains, res
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
