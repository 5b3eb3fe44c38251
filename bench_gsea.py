"""Cost of the gene-set enrichment test (DESIGN.md §4.28) on a seeded 1 000 x 20 000 cohort:

* keys, rank, es -- each kernel alone on one chunk of --rows permutations, CUDA events, warmed, median of --iters;
* norm           -- g2v_gsea_norm on the whole [B, S] matrix;
* gsea           -- g2vec_b200.gsea end to end (synchronised wall time), its host preparation included.

Workloads: S = 50 and 5 000 random sets of 15-500 genes, at B = 1 000 and 10 000.  The ES kernel's achieved gather
bandwidth counts the bytes it must touch: per (row, set) the members' pos (4 B) and u (8 B), the members' gene indices
(4 B) and the score (8 B).  The NumPy oracle (tests/gsea_oracle.py) is timed on a slice of the same work (--oracle-es
(row, set) scores and one row's keys and ranks) and extrapolated to B rows and S sets; the JSON says so.  The card name
and power limit are read in the same run.  Writes nothing into the tree; prints one JSON line per workload.

    python bench_gsea.py [--workloads 50x1000 5000x1000 50x10000 5000x10000] [--iters 5] [--rows 256]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_correlation import card  # noqa: E402
from bench_perm import events_ms  # noqa: E402

N_SAMPLES, N_GENES = 1_000, 20_000


def cohort():
    rng = np.random.Generator(np.random.PCG64(2005))
    x = rng.standard_normal((N_SAMPLES, N_GENES), dtype=np.float32)
    lab = (rng.random(N_SAMPLES) < 0.4).astype(np.int64)
    x[:, :200] += 0.3 * lab[:, None]                     # one percent of the genes differ between the groups
    return x, lab


def random_sets(S, seed=7):
    rng = np.random.Generator(np.random.PCG64(seed))
    return [("set%d" % i, rng.choice(N_GENES, int(rng.integers(15, 501)), replace=False)) for i in range(S)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["50x1000", "5000x1000", "50x10000", "5000x10000"])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rows", type=int, default=256)
    ap.add_argument("--oracle-es", type=int, default=200)
    args = ap.parse_args()
    import torch
    from g2vec_b200 import _capi, perm
    from g2vec_b200.gsea import gsea, restrict_sets, sign_of
    from tests import gsea_oracle as go, perm_oracle
    lib = _capi.load()
    name, power, clock = card()
    x, lab = cohort()
    prep = perm.prepare(x, lab)
    n, k, s, G = prep["n"], prep["k"], sign_of(prep), N_GENES
    pl = perm.planes(prep["q"], np.arange(G))
    S_pad = pl.shape[2]
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    obs, pld, Q, W = dev(prep["obs"]), dev(pl), dev(prep["Q"]), dev(prep["W"])
    R = args.rows
    st = torch.cuda.current_stream().cuda_stream
    M = torch.empty((R, S_pad), dtype=torch.uint8, device="cuda")
    A = torch.empty((R, G), dtype=torch.int64, device="cuda")
    key = torch.empty((R, G), dtype=torch.int64, device="cuda")
    u = torch.empty((R, G), dtype=torch.int64, device="cuda")
    pos = torch.empty((R, G), dtype=torch.int32, device="cuda")
    wsb = int(lib.g2v_gsea_rank_workspace_bytes(R, G))
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    _capi.check(lib.g2v_perm_labels(obs.data_ptr(), n, S_pad, 0, 0, R, M.data_ptr(), st), "labels")
    _capi.check(lib.g2v_perm_sums(M.data_ptr(), pld.data_ptr(), R, S_pad, G, A.data_ptr(), st), "sums")
    keys_ms = events_ms(lambda: _capi.check(lib.g2v_gsea_keys(A.data_ptr(), R, G, n, k, s, Q.data_ptr(), W.data_ptr(),
                                                              key.data_ptr(), u.data_ptr(), st), "keys"), args.iters)
    rank_ms = events_ms(lambda: _capi.check(lib.g2v_gsea_rank(key.data_ptr(), R, G, pos.data_ptr(), ws.data_ptr(), wsb,
                                                              st), "rank"), args.iters)
    # the oracle's keys and ranks of one row, scaled to B rows below
    Mh = perm_oracle.labels(prep["obs"], S_pad, 0, 0, 1)
    t0 = time.perf_counter()
    _, u1, k1 = go.keys(perm_oracle.sums(Mh, prep["q"]), n, k, s, prep["Q"], prep["W"])
    p1 = go.rank(k1)
    oracle_row_s = time.perf_counter() - t0
    for wl in args.workloads:
        S, B = (int(v) for v in wl.split("x"))
        sets = random_sets(S)
        ptr, gene, _ = restrict_sets(sets, range(G), 15, 500)
        ptr_d, gene_d = dev(ptr), dev(gene)
        es = torch.empty((R, S), dtype=torch.float64, device="cuda")
        max_k = int(np.diff(ptr).max())
        es_ms = events_ms(lambda: _capi.check(lib.g2v_gsea_es(pos.data_ptr(), u.data_ptr(), R, G, ptr_d.data_ptr(),
                                                              gene_d.data_ptr(), S, max_k, es.data_ptr(), st), "es"),
                          args.iters)
        es_bytes = R * (12.0 * len(gene) + 4.0 * len(gene) + 8.0 * S)
        esB = torch.empty((B, S), dtype=torch.float64, device="cuda").uniform_(-1, 1)
        eo = torch.empty(S, dtype=torch.float64, device="cuda").uniform_(-1, 1)
        nes = torch.empty_like(esB)
        v = [torch.empty(S, dtype=torch.float64, device="cuda") for _ in range(3)]
        cnt = torch.empty((3, S), dtype=torch.int64, device="cuda")
        norm_ms = events_ms(lambda: _capi.check(lib.g2v_gsea_norm(esB.data_ptr(), B, S, eo.data_ptr(), nes.data_ptr(),
                                                                  v[0].data_ptr(), v[1].data_ptr(), v[2].data_ptr(),
                                                                  cnt.data_ptr(), st), "norm"), args.iters)
        del esB, nes
        torch.cuda.empty_cache()
        gsea(x, lab, sets, min(B, 50), seed=0)           # warm
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = gsea(x, lab, sets, B, seed=0)
        torch.cuda.synchronize()
        wall_s = time.perf_counter() - t0
        m = min(args.oracle_es, S)
        t0 = time.perf_counter()
        for i in range(m):
            go.es_one(p1[0], u1[0], gene[ptr[i]:ptr[i + 1]], G)
        oracle_es_s = (time.perf_counter() - t0) / m
        oracle_s = B * oracle_row_s + (B + 1) * S * oracle_es_s
        print(json.dumps({
            "workload": wl, "n": n, "G": G, "S": S, "B": B, "chunk_rows_timed": R, "mean_set_size": len(gene) / S,
            "keys_ms": round(keys_ms, 3), "rank_ms": round(rank_ms, 3), "es_ms": round(es_ms, 3),
            "norm_ms_full_B": round(norm_ms, 3),
            "es_per_row_us": round(es_ms * 1e3 / R, 2), "es_gather_GBps": round(es_bytes / (es_ms * 1e-3) / 1e9, 1),
            "gsea_wall_s": round(wall_s, 3), "sets_fdr_le_0.25": int((np.nan_to_num(res.FDR, nan=2) <= 0.25).sum()),
            "numpy_oracle_s_extrapolated": round(oracle_s, 1),
            "numpy_oracle_timed_on": "1 row of keys+rank and %d (row, set) scores, scaled to B rows and B+1 x S scores"
                                     % m,
            "gpu": name, "power_limit": power, "sm_clock": clock}), flush=True)


if __name__ == "__main__":
    main()
