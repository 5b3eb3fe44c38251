"""Cost of node2vec's in-out bias in the walk sampler: the production walk pass (packed graph, canonical rows + keys,
every repetition of one group) per graph, in four arms:

* q1      -- q = 1, the shipped first-order route (the two-walker kernel where it applies, e.g. syn10k);
* forced  -- the biased kernel at (a_near, a_far) = (256, 256) (G2V_WALK_BIAS=kernel): the bias machinery alone,
             same walks as q1;
* q0.5    -- q = 0.5 (DFS-like: multipliers (128, 256));
* q2      -- q = 2 (BFS-like: multipliers (256, 128)).

Walk lengths change with q, so every arm reports ms and visited nodes per second.  The card name and power limit are
read in the same run.  Writes nothing into the tree; prints one JSON line per graph.

    python bench_walk_bias.py [--graphs syn10k syn20k stress200k ex0 ex1] [--iters 10] [--reps R]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = (x.strip() for x in out.split(","))
        return name, power
    except Exception as e:                                  # the numbers are still reported
        return "unknown (%s)" % type(e).__name__, "unknown"


def load_graph(name):
    import numpy as np
    from g2vec_b200 import graph
    if name in ("ex0", "ex1"):
        z = np.load(os.path.join(ROOT, "tests", "golden", "ex_graph.npz"))
        g = int(name[-1])
        return z["rowptr%d" % g], z["col%d" % g], graph.quantise_weights(z["w%d" % g]), 80, 10
    V, E, _D, L = graph.BENCH_CONFIGS[name]
    rp, col, w = graph.synthetic_graph(V, E, 0)
    return rp, col, graph.quantise_weights(w), L, 10


def time_arm(g2v, g, L, reps, q, force, iters):
    import torch
    old = os.environ.pop("G2V_WALK_BIAS", None)
    if force:
        os.environ["G2V_WALK_BIAS"] = "kernel"
    try:
        n = g.V * reps
        out = (torch.empty((n, L), dtype=torch.int32, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda"),
               torch.empty(n, dtype=torch.int64, device="cuda"))
        run = lambda: g2v.generate_paths(g, L, reps, seed=0, group=0, canonical=True, out=out, q=q)
        run()
        torch.cuda.synchronize()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
        for a, b in ev:
            a.record()
            run()
            b.record()
        torch.cuda.synchronize()
        ms = sorted(a.elapsed_time(b) for a, b in ev)
        visits = int(out[1].sum())
    finally:
        os.environ.pop("G2V_WALK_BIAS", None)
        if old is not None:
            os.environ["G2V_WALK_BIAS"] = old
    med = ms[len(ms) // 2]
    return {"ms_median": round(med, 4), "ms_min": round(ms[0], 4), "visits": visits,
            "visits_per_s": round(visits / (med * 1e-3), 1)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--graphs", nargs="*", default=["syn10k", "syn20k", "stress200k", "ex0", "ex1"])
    p.add_argument("--iters", type=int, default=10)
    p.add_argument("--reps", type=int, default=0, help="repetitions (walkers = reps * V); 0 = the graph's default")
    args = p.parse_args()
    import torch
    import g2vec_b200 as g2v
    torch.cuda.set_device(0)
    name, power = card()
    for gname in args.graphs:
        rp, col, qw, L, reps = load_graph(gname)
        reps = args.reps or reps
        g = g2v.WalkGraph(rp, col, qw=qw)
        row = {"graph": gname, "V": g.V, "E": g.E, "L": L, "reps": reps, "layout": g.layout, "card": name,
               "power_limit": power}
        for arm, q, force in (("q1", 1.0, False), ("forced", 1.0001, True), ("q0.5", 0.5, False), ("q2", 2.0, False)):
            row[arm] = time_arm(g2v, g, L, reps, q, force, args.iters)
        row["forced_over_q1"] = round(row["forced"]["ms_median"] / row["q1"]["ms_median"], 3)
        print(json.dumps(row), flush=True)
        del g
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
