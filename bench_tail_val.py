#!/usr/bin/env python
"""bench_tail_val.py -- what running the certified validation pass inside the carried tail's launch
(g2v_cbow_loop_tail_val, DESIGN.md §4.32) saves on one step of the device loop, on one H100.

    python bench_tail_val.py --steps K --warmup W [--rounds R] [--workload syn10k|syn20k|syn50k]

Workload: bench.py's walks -> windows of the chosen synthetic workload (default syn10k, the headline), full batch,
split seed 1000.  Two arms in the same process:
  parent  the launches DeviceLoop.one ran before: g2v_cbow_eval_certified over the validation list, then
          g2v_cbow_loop_tail over the training list;
  fused   g2v_cbow_loop_tail_val (st's launch, the one window launch, the carry).
Timed: `step`, the one-step CUDA graph bench.py times, and `production`, the 5-step graph train_cbow replays, divided
by 5.  The arms alternate, R rounds of K timed replays after W warm-up replays each (CUDA events on the launching
stream, L2 flushed by a 256 MiB write before every timed replay).  Reported: each arm's median over the rounds of its
mean, every round's means, the ratio fused / parent, and the card's name and power limit read in the same run.  Prints
one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--workload", default="syn10k", choices=["syn10k", "syn20k", "syn50k"])
    a = p.parse_args(argv)
    if a.steps < 1 or a.warmup < 0 or a.rounds < 1:
        p.error("--steps and --rounds must be >= 1, --warmup >= 0")
    return a


def windows(dev, name, reps=10):
    """bench.py's CBOW input for workload `name`: walks of both groups (seed 12345) -> windows."""
    import torch
    import g2vec_b200 as g2v
    from g2vec_b200 import paths
    from bench import workload
    gs, V, D, L, desc = workload(name)
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
    return rowptr, gene, label, V, D, "%s windows (%s), hidden %d, lenPath %d, numRepetition %d" % (name, desc, D, L,
                                                                                                   reps)


def run(args):
    import torch
    import g2vec_b200 as g2v
    from g2vec_b200 import cbow
    from bench_deterministic import gpu_facts
    assert torch.cuda.is_available(), "bench_tail_val.py needs a GPU (no CPU fallback)"
    dev = torch.device("cuda", torch.cuda.current_device())
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    K, W, R = args.steps, args.warmup, args.rounds

    def timed(fn, n):
        pairs = []
        for i in range(n):
            flush.fill_(i & 0xFF)
            a, b = ev(), ev()
            a.record(); fn(); b.record()
            pairs.append((a, b))
        torch.cuda.synchronize()
        return [a.elapsed_time(b) for a, b in pairs]

    def alternate(fns, scale=1.0):
        for fn in fns.values():
            timed(fn, max(W, 1))
        means = {k: [] for k in fns}
        for _ in range(R):
            for k, fn in fns.items():
                means[k].append(float(np.mean(timed(fn, K))) / scale)
        out = {k + "_ms": float(np.median(v)) for k, v in means.items()}
        out["rounds_ms"] = means
        out["ratio"] = out["fused_ms"] / out["parent_ms"]
        out["fused_lower_every_round"] = all(f < p for f, p in zip(means["fused"], means["parent"]))
        return out

    rowptr, gene, label, V, D, desc = windows(dev, args.workload)
    tr, va = cbow.split_indices(int(rowptr.shape[0]) - 1, 1000)
    W0, Wo0 = cbow.init_weights(V, D, 0)
    tr_d = torch.from_numpy(tr.astype(np.int32)).to(dev)
    va_d = torch.from_numpy(va.astype(np.int32)).to(dev)
    res = {"config": desc + ", full batch, %d training / %d validation windows" % (len(tr), len(va))}
    n_steps = (W + 1 + 2 * R * K) * 5 + 16
    step, prod, keep, hist = {}, {}, [], {}
    shipped = cbow.TAIL_VAL_D
    for name in ("parent", "fused"):
        cbow.TAIL_VAL_D = () if name == "parent" else shipped
        try:
            m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005)
            m.prepare_csc(tr_d)
            m.prepare_slabs(tr_d)
            m.prepare_slabs(va_d)
            loop = cbow.DeviceLoop(m, None, tr_d, va_d, len(tr), n_steps, False, snapshot=False)
            loop.attach()
            try:
                for _ in range(max(W, 1)):
                    loop.one(True)
                loop.reset()
                step[name] = loop.capture([True]).replay
                loop.reset()
                prod[name] = loop.capture([False] * 4 + [True]).replay
            finally:
                loop.detach()
        finally:
            cbow.TAIL_VAL_D = shipped
        keep += [m, loop]
    res["step"] = alternate(step)
    res["production"] = alternate(prod, scale=5.0)
    print(json.dumps({"metric": "cbow_tail_val", "unit": "ms", "lower_is_better": True, "gpu": gpu_facts(),
                      "workload": args.workload, "steps": K, "warmup": W, "rounds": R, "results": res}))


if __name__ == "__main__":
    run(parse())
