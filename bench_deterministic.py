#!/usr/bin/env python
"""bench_deterministic.py -- what train_cbow(deterministic=True) (DESIGN.md §4.13) costs against the default rows
trainer, full batch, on one H100.

    python bench_deterministic.py --steps K --warmup W [--rounds R] [--no-hbm]

Two workloads:
  headline  the syn10k windows of bench.py's headline (walks -> windows, 10k genes, hidden 128, split seed 1000): one
            iteration of the device loop as train_cbow replays it, as CUDA graphs -- `step_ms` from a one-iteration
            graph with both accuracy passes, `production_ms` from the 5-iteration graph train_cbow replays, divided by 5.
            default = g2v_cbow_fwdbwd_csc + g2v_cbow_loop_tail; deterministic = their _det forms.
  stress    the table of bench.py's roofline_hbm block (200k genes x 512, synthetic windows of 80 distinct genes, seed
            777): one full-batch fwd+bwd over the training list.  default = the gene-slab passes train_cbow runs for
            tables larger than the L2; deterministic = the single-pass g2v_cbow_fwdbwd_csc_det.
Both arms of a workload live in the same process and are timed alternately, R rounds of K timed steps after W warm-up
steps each (CUDA events on the launching stream, L2 flushed by a 256 MiB write before every timed step).  Reported: the
median over the rounds of each arm's mean, every round's means, and the ratio deterministic / default.  Prints one JSON
line; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


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


def gpu_facts():
    """Name, power limit and maximum SM clock of GPU 0, read with a query (nothing is changed)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


def run(args):
    import torch
    import g2vec_b200 as g2v
    from g2vec_b200 import cbow
    from bench import synthetic_windows
    from bench_minibatch import headline_windows
    assert torch.cuda.is_available(), "bench_deterministic.py needs a GPU (no CPU fallback)"
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

    def alternate(arms, scale=1.0):
        """arms: name -> callable.  R rounds, each timing every arm in turn; per-arm median of the round means."""
        for fn in arms.values():
            timed(fn, max(W, 1))
        means = {k: [] for k in arms}
        for _ in range(R):
            for k, fn in arms.items():
                means[k].append(float(np.mean(timed(fn, K))) / scale)
        out = {k + "_ms": float(np.median(v)) for k, v in means.items()}
        out["rounds_ms"] = means
        out["ratio"] = out["deterministic_ms"] / out["default_ms"]
        return out

    res = {}
    # ---- headline: the full-batch device loop as CUDA graphs
    rowptr, gene, label, V, D, desc = headline_windows(dev)
    tr, va = cbow.split_indices(int(rowptr.shape[0]) - 1, 1000)
    W0, Wo0 = cbow.init_weights(V, D, 0)
    tr_d = torch.from_numpy(tr.astype(np.int32)).to(dev)
    va_d = torch.from_numpy(va.astype(np.int32)).to(dev)
    n_steps = (W + 1 + 2 * R * K) * 5 + 16               # the loop's step cap must not end the timed steps
    step, prod, keep = {}, {}, []                        # keep: the models and loops the graphs run on
    for name, det in (("default", False), ("deterministic", True)):
        m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005, deterministic=det)
        m.prepare_csc(tr_d)
        m.prepare_slabs(tr_d)
        m.prepare_slabs(va_d)
        loop = cbow.DeviceLoop(m, None, tr_d, va_d, len(tr), n_steps, False, snapshot=False)
        loop.attach()
        try:
            for _ in range(max(W, 1)):                   # eager warm-up of every kernel before the captures
                loop.one(True)
            loop.reset()
            step[name] = loop.capture([True]).replay
            loop.reset()
            prod[name] = loop.capture([False] * 4 + [True]).replay
        finally:
            loop.detach()                                # the graphs keep the loop's `stopped` word baked in
        keep += [m, loop]
    res["headline"] = {"config": desc + ", full batch, %d training windows" % len(tr),
                       "step": alternate(step), "production": alternate(prod, scale=5.0),
                       "default": "g2v_cbow_fwdbwd_csc + g2v_cbow_loop_tail (carried loop)",
                       "deterministic": "g2v_cbow_fwdbwd_csc_det + g2v_cbow_loop_tail_det (carried loop)"}
    del keep, step, prod, m, loop, rowptr, gene, label
    torch.cuda.empty_cache()

    # ---- 200k x 512: slab passes against the deterministic single pass
    if not args.no_hbm:
        V, D, L = 200_000, 512, 80
        N = 2 * args.hbm_reps * V
        rowptr, gene, label = synthetic_windows(N, V, L, dev)
        g = torch.Generator(device=dev); g.manual_seed(0)
        s = 1.0 / np.sqrt(D)
        W0 = (torch.randn(V, D, device=dev, generator=g) * s).clamp_(-2 * s, 2 * s)
        Wo0 = (torch.randn(D, device=dev, generator=g) * s).clamp_(-2 * s, 2 * s)
        n_tr = int(N * 0.8)
        tr = torch.randperm(N, device=dev, generator=g)[:n_tr].to(torch.int32)
        slab = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005)
        slabs = slab.prepare_slabs(tr)
        det = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005, deterministic=True)
        det.prepare_csc(tr)
        r = alternate({"default": lambda: slab.fwdbwd(tr, n_tr), "deterministic": lambda: det.fwdbwd(tr, n_tr)})
        r.update(config="%d x %d table (410 MB), %d synthetic windows of %d distinct genes (seed 777), %d training"
                        % (V, D, N, L, n_tr),
                 default="gene-slab passes (%d slabs)" % getattr(slab, "_n_slabs", 1) if slabs else "single pass",
                 deterministic="g2v_cbow_fwdbwd_csc_det, single pass")
        res["stress200k_512"] = r
        del slab, det
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "cbow_deterministic_cost", "unit": "ms", "lower_is_better": True, "gpu": gpu_facts(),
                      "steps": K, "warmup": W, "rounds": R, "results": res}))


if __name__ == "__main__":
    run(parse())
