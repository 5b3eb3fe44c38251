#!/usr/bin/env python
"""bench_val_loss.py -- what monitoring the validation loss (DESIGN.md §4.19) costs in the full-batch device loop on one
H100.

    python bench_val_loss.py --steps K --warmup W [--rounds R] [--workloads syn10k,ex,stress200k]

Two arms per workload, the production 5-iteration CUDA graph that train_cbow replays, timed per step (graph time / 5):
  val_acc   the default: the validation count, g2v_cbow_loop_decide.
  val_loss  the same step plus g2v_cbow_val_loss after the validation count (and g2v_cbow_st_prepare before it on the
            gene-slab route), deciding with g2v_cbow_loop_decide_score.
The loops never stop while they are timed (early_stop is off on the device, as in bench_lr_plateau.py).  Both arms of a
workload live in the same process and are timed alternately, R rounds of K graph replays after W warm-up replays each
(CUDA events on the launching stream, L2 flushed by a 256 MiB write before every replay).  Reported: the median over
the rounds of each arm's mean, every round's means, and the ratio.  Workloads, rows trainer as train_cbow runs it:
  syn10k      the windows of bench.py's headline (10k genes, hidden 128, split seed 1000): carried CSC path;
  ex          the windows of the ex_* graphs (7523 genes, hidden 128, split seed 0): carried CSC path;
  stress200k  bench.py's table larger than the L2 (numRepetition 2): the gene-slab route.
Prints one JSON line; writes nothing.
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
REPS = {"syn10k": 10, "ex": 10, "stress200k": 2}
SPLIT = {"syn10k": 1000, "ex": 0, "stress200k": 1000}


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--workloads", default="syn10k,ex,stress200k")
    a = p.parse_args(argv)
    if a.steps < 1 or a.warmup < 0 or a.rounds < 1:
        p.error("--steps and --rounds must be >= 1, --warmup >= 0")
    a.workloads = a.workloads.split(",")
    if not set(a.workloads) <= set(REPS):
        p.error("--workloads: a comma-separated subset of %s" % ",".join(REPS))
    return a


def run(args):
    import torch
    import g2vec_b200 as g2v
    from g2vec_b200 import cbow
    from bench_deterministic import gpu_facts
    from bench_lr_plateau import windows
    assert torch.cuda.is_available(), "bench_val_loss.py needs a GPU (no CPU fallback)"
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

    def measure(rowptr, gene, label, V, D, tr_d, va_d, W0, Wo0, n_tr):
        n_steps = 1 + (max(W, 1) + R * K) * CHUNK + 16
        arms, loops, keep, route = {}, {}, [], None
        for name in ("val_acc", "val_loss"):
            m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005)
            if m.prepare_slabs(tr_d):                    # as train_cbow: gene slabs on tables larger than the L2
                m.prepare_slabs(va_d)
            else:
                m.prepare_csc(tr_d)
            route = "slabs" if m.route(va_d) == "slabs" else "certified"   # the validation pass's route
            loop = cbow.DeviceLoop(m, None, tr_d, va_d, n_tr, n_steps, True, snapshot=True, monitor=name)
            loop.attach()
            try:
                loop.one(True)                           # eager warm-up of every kernel before the capture
                loop.reset()
                loop.ctl[5] = 0                          # early_stop off on the device: the timed loop never stops
                arms[name] = loop.capture([loop.carried or (1 + i) % 5 == 0 for i in range(CHUNK)]).replay
            finally:
                loop.detach()
            loops[name] = loop
            keep += [m, loop]
        for fn in arms.values():
            timed(fn, max(W, 1))
        means = {k: [] for k in arms}
        for _ in range(R):
            for k, fn in arms.items():
                means[k].append(float(np.mean(timed(fn, K))) / CHUNK)
        out = {k + "_ms": float(np.median(v)) for k, v in means.items()}
        out["rounds_ms"] = means
        out["val_loss_over_val_acc"] = out["val_loss_ms"] / out["val_acc_ms"]
        done = (max(W, 1) + R * K) * CHUNK
        for name, loop in loops.items():
            loop.fetch()
            torch.cuda.synchronize()
            assert int(loop.ctl_pin[0]) == 0 and int(loop.ctl_pin[1]) == done, "the timed loop stopped"
        sc = loops["val_loss"].score_pin[:done]
        assert int(sc.min()) > 0, "a step left no score"
        out["last_val_loss"] = cbow.val_loss_mean(cbow.SCORE_TOP - int(sc[-1]), int(va_d.shape[0]))
        out["steps_per_arm"] = done
        out["carried"] = bool(loops["val_acc"].carried)
        out["validation_route"] = route
        del keep, arms, loops
        return out

    res = {}
    for name in args.workloads:
        rowptr, gene, label, V, D, desc = windows(dev, name, REPS[name])
        tr, va = cbow.split_indices(int(rowptr.shape[0]) - 1, SPLIT[name])
        W0, Wo0 = cbow.init_weights(V, D, 0)
        tr_d = torch.from_numpy(tr.astype(np.int32)).to(dev)
        va_d = torch.from_numpy(va.astype(np.int32)).to(dev)
        r = measure(rowptr, gene, label, V, D, tr_d, va_d, W0, Wo0, len(tr))
        r["config"] = desc + ", full batch, %d training / %d validation windows, split seed %d" % (
            len(tr), len(va), SPLIT[name])
        res[name] = r
        del rowptr, gene, label, tr_d, va_d
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "cbow_val_loss_cost", "unit": "ms per step", "lower_is_better": True,
                      "gpu": gpu_facts(), "steps": K, "warmup": W, "rounds": R, "results": res}))


if __name__ == "__main__":
    run(parse())
