#!/usr/bin/env python
"""bench_lr_plateau.py -- what the reduce-on-plateau learning rate (DESIGN.md §4.17) costs in the full-batch device
loop on one H100.

    python bench_lr_plateau.py --steps K --warmup W [--rounds R]

Three arms per workload, the production 5-iteration CUDA graph that train_cbow replays, timed per step (graph time / 5):
  off     no schedule: g2v_cbow_adam_tick with the rate as a kernel argument, g2v_cbow_loop_decide.
  never   lr_patience larger than the run: g2v_cbow_adam_tick_lr reads the rate from the device, and
          g2v_cbow_lr_plateau runs after g2v_cbow_loop_decide on every step, but never cuts the rate.
  firing  lr_patience 2, factor 0.9, with the state's best count set above any count after the reset, so that no step
          improves and the rate is cut on every second step (the number of cuts is reported).
The loops never stop while they are timed (early_stop is off on the device, as in bench_patience.py).  All arms of a
workload live in the same process and are timed alternately, R rounds of K graph replays after W warm-up replays each
(CUDA events on the launching stream, L2 flushed by a 256 MiB write before every replay).  Reported: the median over
the rounds of each arm's mean, every round's means, and the ratios to `off`.  Two workloads, both rows trainer on the
carried CSC path as train_cbow runs it:
  syn10k  the windows of bench.py's headline (10k genes, hidden 128, split seed 1000);
  ex      the windows of the ex_* graphs (tests/golden/ex_graph.npz: 7523 genes, hidden 128, lenPath 80,
          numRepetition 10, walk seed 12345, split seed 0).
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


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--rounds", type=int, default=3)
    a = p.parse_args(argv)
    if a.steps < 1 or a.warmup < 0 or a.rounds < 1:
        p.error("--steps and --rounds must be >= 1, --warmup >= 0")
    return a


def windows(dev, name, reps=10):
    """Walks of both groups of bench.py's workload ``name`` (seed 12345) -> windows, on the device."""
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
    return rowptr, gene, label, V, D, "%s windows (%s), hidden %d, lenPath %d, numRepetition %d" % (name, desc, D, L, reps)


def run(args):
    import torch
    import g2vec_b200 as g2v
    from g2vec_b200 import cbow
    from bench_deterministic import gpu_facts
    assert torch.cuda.is_available(), "bench_lr_plateau.py needs a GPU (no CPU fallback)"
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
        arms, loops, keep = {}, {}, []
        for name, lr_patience in (("off", 0), ("never", n_steps + 1), ("firing", 2)):
            m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005)
            if lr_patience:
                m.set_lr_plateau(lr_patience, 0.9, 0.0, n_steps)
            m.prepare_csc(tr_d)
            loop = cbow.DeviceLoop(m, None, tr_d, va_d, n_tr, n_steps, True, snapshot=True)
            loop.attach()
            try:
                loop.one(True)                           # eager warm-up of every kernel before the capture
                loop.reset()
                loop.ctl[5] = 0                          # early_stop off on the device: the timed loop never stops
                if name == "firing":
                    m.plateau[1] = 1 << 62               # no count improves on this best: a cut every 2nd step
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
        out["never_over_off"] = out["never_ms"] / out["off_ms"]
        out["firing_over_off"] = out["firing_ms"] / out["off_ms"]
        done = (max(W, 1) + R * K) * CHUNK
        for name, loop in loops.items():
            loop.fetch()
            torch.cuda.synchronize()
            assert int(loop.ctl_pin[0]) == 0 and int(loop.ctl_pin[1]) == done, "the timed loop stopped"
        st = loops["never"].plateau_pin
        assert int(st[4]) == done and int(st[3]) == 0, "the `never` arm cut its rate"
        st = loops["firing"].plateau_pin
        out["firing_cuts"] = int(st[3])
        out["firing_last_lr"] = float(st.numpy()[8:].view(np.float32)[0])
        out["steps_per_arm"] = done
        out["carried"] = bool(loops["off"].carried)
        del keep, arms, loops
        return out

    res = {}
    for name, split_seed in (("syn10k", 1000), ("ex", 0)):
        rowptr, gene, label, V, D, desc = windows(dev, name)
        tr, va = cbow.split_indices(int(rowptr.shape[0]) - 1, split_seed)
        W0, Wo0 = cbow.init_weights(V, D, 0)
        tr_d = torch.from_numpy(tr.astype(np.int32)).to(dev)
        va_d = torch.from_numpy(va.astype(np.int32)).to(dev)
        r = measure(rowptr, gene, label, V, D, tr_d, va_d, W0, Wo0, len(tr))
        r["config"] = desc + ", full batch, %d training windows, split seed %d" % (len(tr), split_seed)
        res[name] = r
        del rowptr, gene, label, tr_d, va_d
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "cbow_lr_plateau_cost", "unit": "ms per step", "lower_is_better": True,
                      "gpu": gpu_facts(), "steps": K, "warmup": W, "rounds": R, "results": res}))


if __name__ == "__main__":
    run(parse())
