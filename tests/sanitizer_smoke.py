"""Small end-to-end run of every kernel family, meant to be executed under compute-sanitizer on a GPU box:

    compute-sanitizer --tool memcheck  python tests/sanitizer_smoke.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke.py
    compute-sanitizer --tool synccheck python tests/sanitizer_smoke.py

(not a pytest test: the sanitizers slow kernels down 10-100x, so sizes are tiny).  Results are still checked
against the oracle."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import g2vec_b200 as g2v
    from g2vec_b200 import graph, paths
    import oracle
    from tests import helpers

    # walks: bitmap + hash, every edge layout, visit order and fused canonical epilogue
    rp, col, w = helpers.random_graph(300, 40, seed=3, dead_frac=0.2)
    q = graph.quantise_weights(w)
    want, wl = oracle.walks(rp, col, q, 20, 5, 1, 0, 600)
    for vis in ("bitmap", "hash"):
        for layout in ("csr", "e8", "e4"):
            os.environ.update(G2V_WALK_VISITED=vis, G2V_WALK_LAYOUT="e8" if layout == "e8" else "e4")
            g = g2v.WalkGraph(rp, col, qw=q)
            nodes, lens = g2v.generate_paths(g, 20, 2, seed=5, group=1, plain_csr=(layout == "csr"))
            torch.cuda.synchronize()
            assert (nodes.cpu().numpy() == want).all() and (lens.cpu().numpy() == wl).all(), (vis, layout)
            if layout != "csr":
                rows, _, key = g2v.generate_paths(g, 20, 2, seed=5, group=1, canonical=True)
                torch.cuda.synchronize()
    for k in ("G2V_WALK_VISITED", "G2V_WALK_LAYOUT"):
        os.environ.pop(k)
    a, al = g2v.generate_paths_host(rp, col, q, 20, 2, seed=5, group=1)
    assert (a == want).all()

    # glue: exact sort-based path, then the sort-free set pipeline on the sampler's canonical output
    rows = [paths.canonical_rows(*g2v.generate_paths(g2v.WalkGraph(rp, col, qw=q), 20, 2, seed=5, group=grp))
            for grp in (0, 1)]
    prow, plab = paths.integrate(rows[0], rows[1])
    rowptr, gene, label = paths.windows_csr(prow, plab)
    n = 600
    r_all = torch.empty((2 * n, 20), dtype=torch.int32, device="cuda")
    l_all = torch.empty(2 * n, dtype=torch.int32, device="cuda"); k_all = torch.empty(2 * n, dtype=torch.int64, device="cuda")
    for grp in (0, 1):
        sl = slice(grp * n, (grp + 1) * n)
        g2v.generate_paths(g2v.WalkGraph(rp, col, qw=q), 20, 2, seed=5, group=grp, canonical=True, out=(r_all[sl], l_all[sl], k_all[sl]))
    grp_t = torch.cat([torch.zeros(n, dtype=torch.uint8, device="cuda"), torch.ones(n, dtype=torch.uint8, device="cuda")])
    rowptr2, gene2, label2, code2 = paths.build_windows(r_all, l_all, k_all, grp_t, 300)
    assert rowptr2.shape == rowptr.shape and int(rowptr2[-1]) == int(rowptr[-1])

    # CBOW: every kernel variant, a few steps
    V = 300
    for D in (128, 256, 512, 96):
        W0, Wo0 = helpers.init_weights(V, D, 1)
        for algo in ("rows", "rank1"):
            out = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=4, seed=0, W_ih0=W0, W_ho0=Wo0,
                                 early_stop=False, log=None, algo=algo)
            assert np.isfinite(out).all()
    # gene-slab passes (forced on the small table), with 2 and 1 slabs per forward group; the device-side loop with
    # early stop
    for D in (128, 512):
        W0, Wo0 = helpers.init_weights(V, D, 1)
        for env in ({"G2V_CBOW_SLABS": "3"}, {"G2V_CBOW_SLABS": "3", "G2V_CBOW_SLAB_FWD_GROUP": "1"}):
            os.environ.update(env)
            out = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=12, seed=0, W_ih0=W0, W_ho0=Wo0, log=None)
            for k in env:
                os.environ.pop(k)
            assert np.isfinite(out).all()
    rp_h, ge_h, la_h = rowptr.cpu().numpy(), gene.cpu().numpy(), label.cpu().numpy()
    W0, Wo0 = helpers.init_weights(V, 128, 1)
    W, Wo = W0.copy(), Wo0.copy()
    g2v.cbow_step_host(rp_h, ge_h, la_h, W, Wo)

    # edge weights
    rs = np.random.RandomState(0)
    expr = rs.randn(30, 50).astype(np.float32)
    lab = (rs.rand(30) < 0.5).astype(np.int64)
    src, dst = rs.randint(0, 50, 400).astype(np.int32), rs.randint(0, 50, 400).astype(np.int32)
    graph.group_csr_gpu(expr, lab, 0, src, dst, threshold=0.1)
    torch.cuda.synchronize()
    print("sanitizer smoke OK")


if __name__ == "__main__":
    main()
