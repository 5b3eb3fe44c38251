#!/usr/bin/env python
"""bench_minibatch.py -- one mini-batch optimizer step of the CBOW rows trainer on H100, dense `adam` against
`lazy_adam` (DESIGN.md §4.11).

    python bench_minibatch.py --steps K --warmup W [--batches 1024 16384] [--no-hbm]

One step = fwd + bwd + update of one batch of B consecutive windows of the shuffled training list, launched as
train_cbow(batch=B) launches it:
  adam       g2v_cbow_fwdbwd (scatter backward into g_ih) + g2v_cbow_update (TF1 Adam over all V*D parameters);
  lazy_adam  g2v_cbow_fwd_do (dO per batch position) + g2v_cbow_lazy_adam (per-gene dO sums fused with Adam on the
             rows the batch gathered, then the W_ho step).
Two workloads: the syn10k windows of bench.py's headline (walks -> windows, 10k genes, hidden 128) and the table of
its roofline_hbm block (200k genes x 512, synthetic windows of 80 distinct genes, seed 777).  For every B it reports
the per-step time of both optimizers, the mean number of distinct genes per batch and the byte model of both steps
(minibatch_bytes, computed from shapes, not measured).

Timing: CUDA events on the launching stream, W warm-up steps, L2 flushed (256 MiB write) before every timed step,
cycling over the first (at most 32) batches of the training list.  Prints one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def expected_touched(V, B, L):
    """Expected number of distinct genes in a batch of B windows of L genes drawn uniformly from V: V*(1 - e^(-B*L/V))."""
    return V * (1.0 - np.exp(-B * L / V))


def minibatch_bytes(V, D, n_win, nnz, T):
    """Algorithmic bytes of one mini-batch optimizer step over n_win windows with nnz gene incidences, T of them distinct
    genes.  adam: the scatter forward+backward (l*(8D+4)+5 per window) + dense TF1 Adam (read W, m, v, g + write W, m,
    v, g: 32*V*D).  lazy_adam: the forward that stores dO per window (l*(4D+4)+9) + per incidence the position and the
    dO of the segmented sum (8 B) + per touched row read and write W, m, v (24*D*T).  The [D] output layer is left out."""
    dense = nnz * (8 * D + 4) + 5 * n_win + 32 * V * D
    lazy = nnz * (4 * D + 12) + 9 * n_win + 24 * D * T
    return {"adam": int(dense), "lazy_adam": int(lazy)}


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--batches", type=int, nargs="+", default=[1024, 16384])
    p.add_argument("--max-batches", type=int, default=32, help="timed steps cycle over this many batches at most")
    p.add_argument("--hbm-reps", type=int, default=2, help="numRepetition of the 200k x 512 windows (2*reps*V windows)")
    p.add_argument("--no-hbm", action="store_true", help="skip the 200k x 512 table")
    a = p.parse_args(argv)
    if a.steps < 1 or a.warmup < 0 or min(a.batches) < 1:
        p.error("--steps and every batch size must be >= 1, --warmup >= 0")
    return a


def headline_windows(dev, reps=10):
    """bench.py's headline CBOW input: syn10k walks of both groups (seed 12345) -> windows (csrc/g2v_paths.cu)."""
    import torch
    import g2vec_b200 as g2v
    from g2vec_b200 import paths
    from bench import workload
    gs, V, D, L, desc = workload("syn10k")
    n_walk = g2v.walks.num_walkers(V, reps, 0, None, 1)
    rows = torch.empty((2 * n_walk, L), dtype=torch.int32, device=dev)
    lens = torch.empty((2 * n_walk,), dtype=torch.int32, device=dev)
    keys = torch.empty((2 * n_walk,), dtype=torch.int64, device=dev)
    for g, (rp, col, w) in enumerate(gs):
        sl = slice(g * n_walk, (g + 1) * n_walk)
        g2v.generate_paths(g2v.WalkGraph(rp, col, weights=w), L, reps, seed=12345, group=g,
                           out=(rows[sl], lens[sl], keys[sl]), canonical=True)
    grp = torch.cat([torch.zeros(n_walk, dtype=torch.uint8, device=dev), torch.ones(n_walk, dtype=torch.uint8, device=dev)])
    rowptr, gene, label, _ = paths.build_windows(rows, lens, keys, grp, V)
    return rowptr, gene, label, V, D, "syn10k windows (%s), hidden %d, lenPath %d, numRepetition %d" % (desc, D, L, reps)


def run(args):
    import torch
    import g2vec_b200 as g2v
    from g2vec_b200 import cbow
    from bench import synthetic_windows
    assert torch.cuda.is_available(), "bench_minibatch.py needs a GPU (no CPU fallback)"
    dev = torch.device("cuda", torch.cuda.current_device())
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def timed(fn, n):
        pairs = []
        for i in range(n):
            flush.fill_(i & 0xFF)
            a, b = ev(), ev()
            a.record(); fn(); b.record()
            pairs.append((a, b))
        torch.cuda.synchronize()
        return [a.elapsed_time(b) for a, b in pairs]

    def block(rowptr, gene, label, tr, V, D, W0, Wo0, desc):
        lens = (rowptr[1:] - rowptr[:-1]).to(torch.int64)
        out = {"config": desc, "windows_train": int(tr.shape[0])}
        for B in args.batches:
            nb = min(int(tr.shape[0]) // B, args.max_batches)
            if nb < 1:
                continue
            sub = tr[:nb * B].clone()
            nnz = float(lens[sub.to(torch.int64)].sum()) / nb
            r = {"batches": nb, "mean_window_len": nnz / B}
            for opt in ("adam", "lazy_adam"):
                m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, optimizer=opt, lr=0.005)
                if opt == "lazy_adam":
                    m.prepare_batches(sub, B)
                    r["mean_touched_genes"] = float(np.mean([m.batch_touched(sub, k * B, B) for k in range(nb)]))
                it = [0]

                def step():
                    m.fwdbwd(sub, B, win_begin=(it[0] % nb) * B, n_win=B)
                    m.update()
                    it[0] += 1
                timed(step, max(args.warmup, 1))
                r[opt + "_ms"] = float(np.mean(timed(step, args.steps)))
                del m
                torch.cuda.empty_cache()
            r["lazy_speedup"] = r["adam_ms"] / r["lazy_adam_ms"]
            r["bytes_model"] = minibatch_bytes(V, D, B, nnz, r["mean_touched_genes"])
            r["touched_model"] = expected_touched(V, B, nnz / B)
            out["B%d" % B] = r
        return out

    res = {}
    rowptr, gene, label, V, D, desc = headline_windows(dev)
    tr, _ = cbow.split_indices(int(rowptr.shape[0]) - 1, 1000)
    W0, Wo0 = cbow.init_weights(V, D, 0)
    res["headline"] = block(rowptr, gene, label, torch.from_numpy(tr.astype(np.int32)).to(dev), V, D, W0, Wo0, desc)
    del rowptr, gene, label
    torch.cuda.empty_cache()

    if not args.no_hbm:
        V, D, L = 200_000, 512, 80
        N = 2 * args.hbm_reps * V
        rowptr, gene, label = synthetic_windows(N, V, L, dev)
        g = torch.Generator(device=dev); g.manual_seed(0)
        s = 1.0 / np.sqrt(D)
        W0 = (torch.randn(V, D, device=dev, generator=g) * s).clamp_(-2 * s, 2 * s)
        Wo0 = (torch.randn(D, device=dev, generator=g) * s).clamp_(-2 * s, 2 * s)
        tr = torch.randperm(N, device=dev, generator=g)[:int(N * 0.8)].to(torch.int32)
        res["roofline_hbm"] = block(rowptr, gene, label, tr, V, D, W0, Wo0,
                                    "%d x %d table (410 MB), %d synthetic windows of %d distinct genes (seed 777)"
                                    % (V, D, N, L))
    props = torch.cuda.get_device_properties(dev)
    print(json.dumps({"metric": "cbow_minibatch_step_ms", "unit": "ms", "lower_is_better": True, "device": props.name,
                      "steps": args.steps, "warmup": args.warmup, "minibatch": res,
                      "note": "per-batch step = fwd+bwd+update, eager launches, CUDA events, L2 flushed before every "
                              "step; bytes from minibatch_bytes (shapes, not measured)"}))


if __name__ == "__main__":
    run(parse())
