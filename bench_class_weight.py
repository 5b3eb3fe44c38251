#!/usr/bin/env python
"""bench_class_weight.py -- what class weights of the training loss (DESIGN.md §4.20) cost on one H100.

    python bench_class_weight.py --steps K --warmup W [--rounds R]

Four measurements; inside each, the unweighted and the weighted arm live in the same process and are timed alternately,
R rounds of K calls after W warm-up calls each (CUDA events on the launching stream).  Reported: the median over the
rounds of each arm's mean, every round's means, and the ratio weighted / unweighted.  The weights are (0.37, 1.9).
  graph_rows   syn10k full batch (bench.py's headline windows, split seed 1000), the production 5-iteration CUDA graph
               of the device loop timed per step (graph time / 5, L2 flushed by a 256 MiB write before every replay),
               algo rows (the carried CSC path).  Early stopping is off on the device.
  graph_rank1  the same with algo rank1 (the rank-1 step).
  lazy_step    one lazy_adam mini-batch step (forward + dO, then g2v_cbow_lazy_adam) on the first batch of 4096 syn10k
               training windows.
  slab_step    one full-batch rows step on the gene-slab route of bench.py's 200k x 512 table (stress200k,
               numRepetition 2): g2v_cbow_fwdbwd_slabs[_cw] and the dense Adam pass.
The card's name and power limit are read (nvidia-smi query) in the same run.  Prints one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CHUNK = 5
CW = (0.37, 1.9)


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--rounds", type=int, default=3)
    a = p.parse_args(argv)
    if a.steps < 1 or a.warmup < 0 or a.rounds < 1:
        p.error("--steps and --rounds must be >= 1, --warmup >= 0")
    return a


def run(args):
    import torch
    import g2vec_b200 as g2v
    from g2vec_b200 import cbow
    from bench_deterministic import gpu_facts
    from bench_lr_plateau import windows
    assert torch.cuda.is_available(), "bench_class_weight.py needs a GPU (no CPU fallback)"
    dev = torch.device("cuda", torch.cuda.current_device())
    facts_before = gpu_facts()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    K, W, R = args.steps, args.warmup, args.rounds

    def timed(fn, n, do_flush):
        pairs = []
        for i in range(n):
            if do_flush:
                flush.fill_(i & 0xFF)
            a, b = ev(), ev()
            a.record(); fn(); b.record()
            pairs.append((a, b))
        torch.cuda.synchronize()
        return [a.elapsed_time(b) for a, b in pairs]

    def alternate(arms, per=1.0, do_flush=True):
        for fn in arms.values():
            timed(fn, max(W, 1), do_flush)
        means = {k: [] for k in arms}
        for _ in range(R):
            for k, fn in arms.items():
                means[k].append(float(np.mean(timed(fn, K, do_flush))) / per)
        out = {k + "_ms": float(np.median(v)) for k, v in means.items()}
        out["rounds_ms"] = means
        out["cw_over_plain"] = out["cw_ms"] / out["plain_ms"]
        return out

    res = {}
    rowptr, gene, label, V, D, desc = windows(dev, "syn10k")
    tr, va = cbow.split_indices(int(rowptr.shape[0]) - 1, 1000)
    W0, Wo0 = cbow.init_weights(V, D, 0)
    tr_d = torch.from_numpy(tr.astype(np.int32)).to(dev)
    va_d = torch.from_numpy(va.astype(np.int32)).to(dev)
    n_steps = 1 + (max(W, 1) + R * K) * CHUNK + 16
    for algo in ("rows", "rank1"):
        arms, keep = {}, []
        for name, cw in (("plain", None), ("cw", CW)):
            m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005, algo=algo, class_weight=cw)
            m.prepare_csc(tr_d)
            loop = cbow.DeviceLoop(m, None, tr_d, va_d, len(tr), n_steps, True, snapshot=True)
            loop.attach()
            try:
                loop.one(True)
                loop.reset()
                loop.ctl[5] = 0                              # early_stop off on the device: the timed loop never stops
                arms[name] = loop.capture([loop.carried or (1 + i) % 5 == 0 for i in range(CHUNK)]).replay
            finally:
                loop.detach()
            keep += [m, loop]
        r = alternate(arms, per=CHUNK)
        r["config"] = desc + ", full batch, %d training windows, algo %s" % (len(tr), algo)
        res["graph_" + algo] = r
        del keep, arms
    B = 4096
    arms, keep = {}, []
    for name, cw in (("plain", None), ("cw", CW)):
        m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, optimizer="lazy_adam", lr=0.005, class_weight=cw)
        m.prepare_batches(tr_d, B)

        def step(m=m):
            m.acc.zero_()
            m.fwdbwd(tr_d, B, win_begin=0, n_win=B)
            m.update()
        arms[name] = step
        keep.append(m)
    r = alternate(arms)
    r["config"] = "one lazy_adam step: the first batch of %d syn10k training windows (%d touched genes), hidden %d" % (
        B, keep[0].batch_touched(tr_d, 0, B), D)
    res["lazy_step"] = r
    del keep, arms, rowptr, gene, label, tr_d, va_d
    torch.cuda.empty_cache()
    # the gene-slab route, 200k x 512
    rowptr, gene, label, V, D, desc = windows(dev, "stress200k", 2)
    tr, _ = cbow.split_indices(int(rowptr.shape[0]) - 1, 1000)
    W0, Wo0 = cbow.init_weights(V, D, 0)
    tr_d = torch.from_numpy(tr.astype(np.int32)).to(dev)
    arms, keep = {}, []
    for name, cw in (("plain", None), ("cw", CW)):
        m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005, class_weight=cw)
        assert m.prepare_slabs(tr_d), "the 200k x 512 table fits the L2 on this card: no slab route"

        def step(m=m):
            m.acc.zero_()
            m.fwdbwd(tr_d, len(tr))
            m.update()
        arms[name] = step
        keep.append(m)
        del m
        torch.cuda.synchronize()
    r = alternate(arms, do_flush=False)
    r["config"] = desc + ", one full-batch rows step on the gene-slab route (%d slabs), %d training windows" % (
        keep[0]._n_slabs, len(tr))
    res["slab_step"] = r
    del keep, arms
    torch.cuda.empty_cache()
    print(json.dumps({"metric": "cbow_class_weight_cost", "unit": "ms per step", "lower_is_better": True,
                      "gpu": facts_before, "gpu_after": gpu_facts(), "steps": K, "warmup": W, "rounds": R,
                      "class_weight": CW, "results": res}))


if __name__ == "__main__":
    run(parse())
