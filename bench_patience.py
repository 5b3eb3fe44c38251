#!/usr/bin/env python
"""bench_patience.py -- what early stopping with patience (DESIGN.md §4.15) costs against the default rule in the
full-batch device loop on one H100.

    python bench_patience.py --steps K --warmup W [--rounds R] [--no-hbm]

Two arms per workload, the production 5-iteration CUDA graph that train_cbow replays, timed per step (graph time / 5):
  patience1  the default rule: g2v_cbow_loop_begin copies W_ih into the snapshot on every step, g2v_cbow_loop_decide.
  patience5  g2v_cbow_loop_begin without the snapshot, g2v_cbow_loop_decide_best, and g2v_cbow_loop_keep_best, which
             copies W_ih only on the steps whose validation count is >= the best so far.
The loops never stop while they are timed: patience1 runs with early_stop off (the same launches and copies as with it
on), and patience5's early_stop word is cleared after its reset.  So patience5 copies on the steps that improve, as it
would in a run; the share of such steps among the timed ones is reported beside its time.  Each workload is measured
twice: `trained`, with its validation list, where the share is whatever training gives; and `every_step_improves`, the
worst case for patience5, with an empty validation list in both arms (every count is 0, which ties the best), so
patience5 copies on every step and the two arms differ only in where the copy is made.
Two workloads:
  syn10k    the windows of bench.py's headline (10k genes, hidden 128, split seed 1000), rows trainer on the carried CSC
            path, as train_cbow runs it.
  200k_512  the table of bench.py's roofline_hbm block (200k genes x 512, synthetic windows of 80 distinct genes, seed
            777, a random 80/20 split), gene-slab passes as train_cbow picks them for tables larger than the L2.
Both arms of a workload live in the same process and are timed alternately, R rounds of K graph replays after W warm-up
replays each (CUDA events on the launching stream, L2 flushed by a 256 MiB write before every replay).  Reported: the
median over the rounds of each arm's mean, every round's means, and the ratio patience5 / patience1.  Prints one JSON
line; writes nothing.
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
    p.add_argument("--hbm-reps", type=int, default=2, help="numRepetition of the 200k x 512 windows (2*reps*V windows)")
    p.add_argument("--no-hbm", action="store_true", help="skip the 200k x 512 table")
    a = p.parse_args(argv)
    if a.steps < 1 or a.warmup < 0 or a.rounds < 1:
        p.error("--steps and --rounds must be >= 1, --warmup >= 0")
    return a


def improving_share(hist, lo, hi):
    """Share of steps lo..hi-1 whose validation count (hist[step][2]) is >= every count before it."""
    val = hist.reshape(-1, 4)[:hi, 2]
    best = np.maximum.accumulate(val)
    return float(np.mean(val[lo:hi] >= np.concatenate([[-1], best[:-1]])[lo:hi]))


def run(args):
    import torch
    import g2vec_b200 as g2v
    from g2vec_b200 import cbow
    from bench import synthetic_windows
    from bench_deterministic import gpu_facts
    from bench_minibatch import headline_windows
    assert torch.cuda.is_available(), "bench_patience.py needs a GPU (no CPU fallback)"
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
        # steps the loop runs: one eager warm-up step, then every replay advances it by CHUNK
        n_steps = 1 + (W + R * K) * CHUNK + 16
        arms, loops, keep = {}, {}, []
        for name, patience in (("patience1", 1), ("patience5", 5)):
            m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005)
            slabs = m.prepare_slabs(tr_d)
            m.prepare_slabs(va_d)
            if not slabs:
                m.prepare_csc(tr_d)
            loop = cbow.DeviceLoop(m, None, tr_d, va_d, n_tr, n_steps, patience > 1, snapshot=True, patience=patience)
            assert (loop.best is not None) == (patience > 1)
            loop.attach()
            try:
                loop.one(True)                           # eager warm-up of every kernel before the capture
                loop.reset()
                loop.ctl[5] = 0                          # early_stop off on the device: the timed loop never stops
                # train_cbow's chunk of steps 1..5: the training-accuracy pass on the 5th (every step when carried)
                arms[name] = loop.capture([loop.carried or (1 + i) % 5 == 0 for i in range(CHUNK)]).replay
            finally:
                loop.detach()                            # the graph keeps the loop's `stopped` word baked in
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
        out["ratio"] = out["patience5_ms"] / out["patience1_ms"]
        lp = loops["patience5"]
        lp.fetch()
        torch.cuda.synchronize()
        done = int(lp.ctl_pin[1])
        assert int(lp.ctl_pin[0]) == 0 and done == (max(W, 1) + R * K) * CHUNK, "the timed loop stopped"
        out["patience5_improving_share"] = improving_share(lp.hist_pin.numpy(), max(W, 1) * CHUNK, done)
        out["steps_per_arm"] = done
        out["carried"] = bool(lp.carried)
        out["gene_slabs"] = int(getattr(keep[0], "_n_slabs", 1)) if keep[0].prepared(tr_d).slabs else 0
        del keep, arms, loops
        return out

    def both(rowptr, gene, label, V, D, tr_d, va_d, W0, Wo0, n_tr):
        none = torch.empty(0, dtype=torch.int32, device=dev)
        return {"trained": measure(rowptr, gene, label, V, D, tr_d, va_d, W0, Wo0, n_tr),
                "every_step_improves": measure(rowptr, gene, label, V, D, tr_d, none, W0, Wo0, n_tr)}

    res = {}
    rowptr, gene, label, V, D, desc = headline_windows(dev)
    tr, va = cbow.split_indices(int(rowptr.shape[0]) - 1, 1000)
    W0, Wo0 = cbow.init_weights(V, D, 0)
    tr_d = torch.from_numpy(tr.astype(np.int32)).to(dev)
    va_d = torch.from_numpy(va.astype(np.int32)).to(dev)
    r = both(rowptr, gene, label, V, D, tr_d, va_d, W0, Wo0, len(tr))
    r["config"] = desc + ", full batch, %d training windows" % len(tr)
    res["syn10k"] = r
    del rowptr, gene, label, tr_d, va_d
    torch.cuda.empty_cache()

    if not args.no_hbm:
        V, D, L = 200_000, 512, 80
        N = 2 * args.hbm_reps * V
        rowptr, gene, label = synthetic_windows(N, V, L, dev)
        g = torch.Generator(device=dev); g.manual_seed(0)
        s = 1.0 / np.sqrt(D)
        W0 = (torch.randn(V, D, device=dev, generator=g) * s).clamp_(-2 * s, 2 * s)
        Wo0 = (torch.randn(D, device=dev, generator=g) * s).clamp_(-2 * s, 2 * s)
        n_tr = int(N * 0.8)
        perm = torch.randperm(N, device=dev, generator=g).to(torch.int32)
        r = both(rowptr, gene, label, V, D, perm[:n_tr].contiguous(), perm[n_tr:].contiguous(), W0, Wo0, n_tr)
        r["config"] = ("%d x %d table (410 MB), %d synthetic windows of %d distinct genes (seed 777), %d training"
                       % (V, D, N, L, n_tr))
        res["200k_512"] = r
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "cbow_patience_cost", "unit": "ms per step", "lower_is_better": True,
                      "gpu": gpu_facts(), "steps": K, "warmup": W, "rounds": R, "results": res}))


if __name__ == "__main__":
    run(parse())
