#!/usr/bin/env python
"""bench_weight_decay.py -- what decoupled weight decay (DESIGN.md §4.18) costs on one H100.

    python bench_weight_decay.py --steps K --warmup W [--rounds R]

Three measurements; inside each, the arms live in the same process and are timed alternately, R rounds of K calls
after W warm-up calls each (CUDA events on the launching stream).  Reported: the median over the rounds of each arm's
mean, every round's means, and the ratios to λ = 0.
  graph   syn10k full batch (bench.py's headline windows, split seed 1000), the production 5-iteration CUDA graph of the
          device loop timed per step (graph time / 5, L2 flushed by a 256 MiB write before every replay), for
          algo rows (carried CSC path) and rank1, at λ = 0 and λ = 1e-2.  Early stopping is off on the device.
  update  the dense optimizer pass alone (g2v_cbow_update[_wd], TF1 Adam, device alpha) on a 200k x 512 table:
          λ = 0; fused λ = 1e-2; composed: a float32 torch decay W - (λ W) over [W_ih | W_ho], then the λ = 0 pass.
  lazy    one lazy_adam mini-batch step (forward + dO, then g2v_cbow_lazy_adam[_wd]) on the first batch of 4096
          syn10k training windows, at λ = 0 and λ = 1e-2.
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
LAM = 1e-2


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
    from g2vec_b200 import _capi, cbow
    from bench_deterministic import gpu_facts
    from bench_lr_plateau import windows
    assert torch.cuda.is_available(), "bench_weight_decay.py needs a GPU (no CPU fallback)"
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
        first = next(iter(arms))
        for k in arms:
            if k != first:
                out[k + "_over_" + first] = out[k + "_ms"] / out[first + "_ms"]
        return out

    res = {}
    # 1. the production graph, syn10k full batch
    rowptr, gene, label, V, D, desc = windows(dev, "syn10k")
    tr, va = cbow.split_indices(int(rowptr.shape[0]) - 1, 1000)
    W0, Wo0 = cbow.init_weights(V, D, 0)
    tr_d = torch.from_numpy(tr.astype(np.int32)).to(dev)
    va_d = torch.from_numpy(va.astype(np.int32)).to(dev)
    n_steps = 1 + (max(W, 1) + R * K) * CHUNK + 16
    for algo in ("rows", "rank1"):
        arms, keep = {}, []
        for name, lam in (("wd0", 0.0), ("wd", LAM)):
            m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005, algo=algo, weight_decay=lam)
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
    # 3. one lazy_adam mini-batch step
    B = 4096
    arms, keep = {}, []
    for name, lam in (("wd0", 0.0), ("wd", LAM)):
        m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, optimizer="lazy_adam", lr=0.005, weight_decay=lam)
        m.prepare_batches(tr_d, B)

        def step(m=m):
            m.acc.zero_()
            m.fwdbwd(tr_d, B, win_begin=0, n_win=B)
            m.update()
        arms[name] = step
        keep.append(m)
    r = alternate(arms, do_flush=True)
    r["config"] = "one lazy_adam step: the first batch of %d syn10k training windows (%d touched genes), hidden %d" % (
        B, keep[0].batch_touched(tr_d, 0, B), D)
    res["lazy_step"] = r
    del keep, arms, rowptr, gene, label, tr_d, va_d
    torch.cuda.empty_cache()
    # 2. the dense update pass alone, 200k x 512
    lib, st = _capi.load(), torch.cuda.current_stream().cuda_stream
    Vb, Db = 200_000, 512
    n = Vb * Db + Db
    w, mm, vv, gg = (torch.zeros(n, dtype=torch.float32, device=dev) for _ in range(4))
    w.normal_(); mm.normal_(std=1e-3); vv.uniform_(0, 1e-6)
    hyper = torch.tensor([0.9, 0.999, 1e-3, 0.0], dtype=torch.float32, device=dev)
    k = 4 * Vb * Db
    args_ = lambda: (w.data_ptr(), w.data_ptr() + k, mm.data_ptr(), vv.data_ptr(), mm.data_ptr() + k,
                     vv.data_ptr() + k, gg.data_ptr(), gg.data_ptr() + k, Vb, Db, 0, 0.005, 0.9, 0.999, 1e-8)
    lam32 = float(np.float32(LAM))

    def plain():
        _capi.check(lib.g2v_cbow_update(*args_(), 0, hyper.data_ptr(), st), "g2v_cbow_update")

    def fused():
        _capi.check(lib.g2v_cbow_update_wd(*args_(), lam32, 0, hyper.data_ptr(), st), "g2v_cbow_update_wd")

    def composed():
        w.sub_(lam32 * w)
        plain()
    r = alternate({"wd0": plain, "fused": fused, "composed": composed}, do_flush=False)
    r["config"] = "dense TF1 Adam pass over [W_ih | W_ho], V = %d, D = %d (%.0f MB per buffer), device alpha" % (
        Vb, Db, 4 * n / 1e6)
    # composed: torch's λ * W (read 4, write 4) and W -= that (read 8, write 4) before the 32 B pass
    r["bytes_per_element"] = {"wd0": 32, "fused": 32, "composed": 32 + 20}
    res["update_200k_x_512"] = r
    del w, mm, vv, gg
    torch.cuda.empty_cache()
    print(json.dumps({"metric": "cbow_weight_decay_cost", "unit": "ms per step", "lower_is_better": True,
                      "gpu": facts_before, "gpu_after": gpu_facts(), "steps": K, "warmup": W, "rounds": R,
                      "weight_decay": LAM, "results": res}))


if __name__ == "__main__":
    run(parse())
