#!/usr/bin/env python
"""bench_minibatch.py -- one mini-batch optimizer step of the CBOW rows trainer on H100, dense `adam` against
`lazy_adam` (DESIGN.md §4.11).

    python bench_minibatch.py --steps K --warmup W [--batches 1024 16384] [--no-hbm]

One step = fwd + bwd + update of one batch of B consecutive windows of the shuffled training list, launched as
train_cbow(batch=B) launches it:
  adam       g2v_cbow_fwdbwd (scatter backward into g_ih) + g2v_cbow_update (TF1 Adam over all V*D parameters);
  lazy_adam  g2v_cbow_fwd_do (dO per batch position) + g2v_cbow_lazy_adam (per-gene dO sums fused with Adam on the
             rows the batch gathered, then the W_ho step);
  adam_det   train_cbow(batch=B, deterministic=True) (DESIGN.md §4.13): g2v_cbow_fwd_do_det (tiled forward + fixed-order
             tile sum) + g2v_cbow_batch_expand (per-gene dO sums over the batch plan into g_ih) + g2v_cbow_update.
Two workloads: the syn10k windows of bench.py's headline (walks -> windows, 10k genes, hidden 128) and the table of
its roofline_hbm block (200k genes x 512, synthetic windows of 80 distinct genes, seed 777).  For every B it reports
the per-step time of both optimizers, the mean number of distinct genes per batch and the byte model of both steps
(minibatch_bytes, computed from shapes, not measured).

Reshuffled epochs (DESIGN.md §4.12), per B, over the whole training list: order_ms (g2v_cbow_epoch_order), plan_ms
(g2v_cbow_batch_plan plus the read-back of the per-batch row offsets, as prepare_batches runs it), sort_plan_ms (a
stand-in for the earlier prepare_batches: its torch.sort construction, tests/reshuffle_oracle.batch_plan_torch, on the
same list, without its per-batch dict loop), and epoch_ms / epoch_reshuffle_ms: one whole lazy_adam epoch over the training list without and with the new
order and the plan rebuild (CUDA events, after one warm-up epoch, no L2 flush).  plan_bytes is the builder's byte model
(batch_plan_bytes, from shapes).

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


def batch_plan_bytes(V, n_win, nnz, n_b, T_sum):
    """Algorithmic bytes of g2v_cbow_batch_plan over n_win windows with nnz incidences in n_b batches touching T_sum
    (batch, gene) rows: two passes over the windows (win + rowptr 12 B per window, gene + counter atomic 8 B per
    incidence, plus the 4 B scatter of the position), the segment sort (read 4 + write 4 per incidence), the counters
    (zero, tile sums, emit read, cursor write: 16 B per (batch, gene)) and rows + segptr (8 B per touched row)."""
    return int(2 * 12 * n_win + nnz * (8 + 12) + 16 * n_b * V + 8 * T_sum)


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

    def reshuffle_fields(rowptr, gene, label, tr, V, D, W0, Wo0, B, r):
        """order_ms, plan_ms, sort_plan_ms, epoch_ms, epoch_reshuffle_ms over the whole training list tr."""
        from tests.reshuffle_oracle import batch_plan_torch
        n = int(tr.shape[0])
        m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, optimizer="lazy_adam", lr=0.005)
        ep = torch.empty_like(tr)
        m.prepare_batches(tr, B)
        n_b = -(-n // B)

        def host(fn, k):
            ts = []
            for _ in range(k):
                torch.cuda.synchronize()
                a, b = ev(), ev()
                a.record(); fn(); b.record()
                torch.cuda.synchronize()
                ts.append(a.elapsed_time(b))
            return ts
        order = lambda: cbow.epoch_order(tr, 0, 1, out=ep)
        host(order, 2)
        r["order_ms"] = float(np.median(host(order, args.steps)))
        plan = lambda: m.prepare_batches(ep, B)
        host(plan, 2)
        r["plan_ms"] = float(np.median(host(plan, args.steps)))
        srt = lambda: batch_plan_torch(m.rowptr, m.gene, V, ep, B)
        host(srt, 2)
        r["sort_plan_ms"] = float(np.median(host(srt, args.steps)))
        r["plan_bytes"] = batch_plan_bytes(V, n, int(m.prepared(ep).plan.nnz), n_b,
                                           sum(m.batch_touched(ep, k * B, min(B, n - k * B)) for k in range(n_b)))

        def epoch(reshuffle, e=[1]):
            win = tr
            if reshuffle:
                e[0] += 1
                cbow.epoch_order(tr, 0, e[0], out=ep)
                m.prepare_batches(ep, B)
                win = ep
            for lo in range(0, n, B):
                nb = min(B, n - lo)
                m.fwdbwd(win, nb, win_begin=lo, n_win=nb)
                m.update()
        for flag, name in ((False, "epoch_ms"), (True, "epoch_reshuffle_ms")):
            host(lambda: epoch(flag), 1)
            r[name] = float(np.median(host(lambda: epoch(flag), 3)))
        r["reshuffle_overhead"] = r["epoch_reshuffle_ms"] / r["epoch_ms"] - 1.0
        del m, ep
        torch.cuda.empty_cache()

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
            for opt in ("adam", "lazy_adam", "adam_det"):
                det = opt == "adam_det"
                m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, optimizer="adam" if det else opt, lr=0.005,
                                  deterministic=det)
                if opt != "adam":
                    m.prepare_batches(sub, B)
                if opt == "lazy_adam":
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
            r["det_cost_vs_adam"] = r["adam_det_ms"] / r["adam_ms"]
            r["bytes_model"] = minibatch_bytes(V, D, B, nnz, r["mean_touched_genes"])
            r["touched_model"] = expected_touched(V, B, nnz / B)
            reshuffle_fields(rowptr, gene, label, tr, V, D, W0, Wo0, B, r)
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
