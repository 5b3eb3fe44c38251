"""GPU parity of HOT PATH 2 (modified CBOW) against the oracle, through the C ABI.

Tolerance (north_star): learned vectors / accuracy within 1e-4 relative.  Concretely
  vectors : max|W_gpu - W_oracle| <= 1e-4 * max|W_oracle|   (float32 reassociation; the oracle sums
            windows sequentially, the GPU with atomics in arbitrary order)
  accuracy: |acc_gpu - acc_oracle| <= 2 windows / N   (a logit within 1e-6 of 0 may change sign)
Gradients of ONE step are compared tighter: 2e-5 relative to the largest entry.
"""
import numpy as np
import pytest

import oracle
from tests import helpers

pytestmark = pytest.mark.gpu
RTOL_VEC = 1e-4


@pytest.fixture(scope="module")
def g2v():
    import torch
    assert torch.cuda.is_available()
    import g2vec_b200
    return g2vec_b200


def rel_max(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def one_step(g2v, rowptr, gene, label, V, D, reduce="sum", optimizer="adam", seed=1, win=None):
    import torch
    W0, Wo0 = helpers.init_weights(V, D, seed)
    N = len(rowptr) - 1
    win = np.arange(N, dtype=np.int64) if win is None else win
    m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, optimizer=optimizer, reduce=reduce, lr=0.005)
    wd = torch.from_numpy(win.astype(np.int32)).cuda()
    m.fwdbwd(wd, len(win))
    torch.cuda.synchronize()
    acc = m.acc.cpu()
    g_ih, g_ho = m.g_ih.cpu().numpy().copy(), m.g_ho.cpu().numpy().copy()
    m.update()
    torch.cuda.synchronize()
    return m, W0, Wo0, g_ih, g_ho, m.loss_sum(acc), int(acc[1])


@pytest.mark.parametrize("D", [128, 256, 512, 100, 64, 4])
def test_one_step_gradients_and_adam(g2v, D):
    V, N = 500, 3000
    rowptr, gene, label = helpers.random_windows(N, V, 1, 80, seed=D)
    # keep empty windows in the mix (an all-zero row of the reference's dense pathList): window 4 gives its
    # genes to window 5, the last window is emptied by dropping its genes
    rowptr[5] = rowptr[4]
    gene = gene[:rowptr[N - 1]].copy(); rowptr[N] = rowptr[N - 1]
    assert rowptr[5] == rowptr[4] and rowptr[N] == rowptr[N - 1] and (np.diff(rowptr) >= 0).all()
    m, W0, Wo0, g_ih, g_ho, loss, nc = one_step(g2v, rowptr, gene, label, V, D)
    win = np.arange(N, dtype=np.int64)
    o_gih, o_gho, o_loss, o_nc = oracle.cbow_grad(rowptr, gene, label, win, N, W0, Wo0)
    assert rel_max(g_ih, o_gih) < 2e-5 and rel_max(g_ho, o_gho) < 2e-5
    assert abs(loss / N - o_loss) < 1e-5 * max(1.0, abs(o_loss))
    assert abs(nc - o_nc) <= 2
    W, Wo = W0.copy(), Wo0.copy()
    mm, vv, mo, vo = np.zeros_like(W), np.zeros_like(W), np.zeros_like(Wo), np.zeros_like(Wo)
    oracle.adam_(W, mm, vv, o_gih, 0.005, 1); oracle.adam_(Wo, mo, vo, o_gho, 0.005, 1)
    assert rel_max(m.W_ih.cpu().numpy(), W) < RTOL_VEC
    assert rel_max(m.W_ho.cpu().numpy(), Wo) < RTOL_VEC
    assert float(m.g_ih.abs().max()) == 0.0 and float(m.g_ho.abs().max()) == 0.0   # zeroed for next step


def test_mean_reduce_and_sgd_variant(g2v):
    """north_star's variant (segmented MEAN, SGD) is the same kernel with two switches."""
    V, N, D = 300, 1000, 128
    rowptr, gene, label = helpers.random_windows(N, V, 1, 40, seed=9)
    m, W0, Wo0, g_ih, g_ho, loss, nc = one_step(g2v, rowptr, gene, label, V, D, reduce="mean", optimizer="sgd")
    # oracle of the mean variant: scale rows by 1/len == sum-variant on W/len per window -> restate directly
    lens = np.diff(rowptr).astype(np.float32)
    H = np.zeros((N, D), np.float32)
    for n in range(N):
        H[n] = W0[gene[rowptr[n]:rowptr[n + 1]]].sum(0) / lens[n]
    o = H @ Wo0
    dO = (1 / (1 + np.exp(-o.astype(np.float64))) - label) / N
    want_gho = (H * dO[:, None]).sum(0)
    want_gih = np.zeros((V, D), np.float64)
    for n in range(N):
        want_gih[gene[rowptr[n]:rowptr[n + 1]]] += dO[n] / lens[n] * Wo0
    assert rel_max(g_ho, want_gho) < 1e-4 and rel_max(g_ih, want_gih) < 1e-4
    assert rel_max(m.W_ih.cpu().numpy(), W0 - 0.005 * want_gih) < RTOL_VEC


def test_window_subset_and_offsets(g2v):
    import torch
    V, N, D = 200, 800, 128
    rowptr, gene, label = helpers.random_windows(N, V, 1, 30, seed=2)
    rs = np.random.RandomState(0)
    win = rs.permutation(N)[:500].astype(np.int64)
    m, W0, Wo0, g_ih, g_ho, loss, nc = one_step(g2v, rowptr, gene, label, V, D, win=win)
    o_gih, o_gho, _, o_nc = oracle.cbow_grad(rowptr, gene, label, win, len(win), W0, Wo0)
    assert rel_max(g_ih, o_gih) < 2e-5 and abs(nc - o_nc) <= 1
    # eval on a sub-range of the list
    m2 = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0)
    wd = torch.from_numpy(win.astype(np.int32)).cuda()
    m2.evaluate(wd, 2, win_begin=100, n_win=300)
    m2.evaluate(None, 3, win_begin=10, n_win=N - 10)
    torch.cuda.synchronize()
    acc = m2.acc.cpu()
    assert abs(int(acc[2]) - oracle.cbow_eval(rowptr, gene, label, win[100:400], W0, Wo0)) <= 1
    assert abs(int(acc[3]) - oracle.cbow_eval(rowptr, gene, label, np.arange(10, N), W0, Wo0)) <= 1


def test_ex_windows_five_steps_match_oracle(g2v):
    """BASELINE configs[0] shape: ex_* windows (oracle walks), hidden 128, lr 0.005, 5 Adam steps."""
    (rowptr, gene, label), _ = helpers.ex_windows(reps=2)
    V, D = 7523, 128
    N = len(rowptr) - 1
    tr, va = oracle.split_indices(N, 0)
    from g2vec_b200 import cbow
    tr2, va2 = cbow.split_indices(N, 0)
    assert (tr == tr2).all() and (va == va2).all()
    W0, Wo0 = helpers.init_weights(V, D, 0)
    want, hist, stop, _ = oracle.cbow_train(rowptr, gene, label, tr, va, W0, Wo0, 0.005, max_steps=5, early_stop=False)
    got, info = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=5, seed=0, W_ih0=W0, W_ho0=Wo0,
                               early_stop=False, log=None, return_info=True)
    assert rel_max(got, want) < RTOL_VEC
    for (s, av, at), (s2, av2, at2) in zip(hist, info["history"]):
        assert abs(av - av2) <= 2.0 / len(va) + 1e-7 and abs(at - at2) <= 2.0 / len(tr) + 1e-7
    # rows never touched by a training window keep their initial value (SURVEY 3.2-2)
    touched = np.zeros(V, bool); 
    for n in tr:
        touched[gene[rowptr[n]:rowptr[n + 1]]] = True
    assert (got[~touched] == W0[~touched]).all() and (~touched).sum() > 1000


def test_config1_parity_run_ten_repetitions(g2v):
    """SURVEY 8d config 1: ex_* graphs, -p 80 -s 128 -e 5, numRepetition 10, lr 0.005: windows from the
    GPU sampler equal the oracle's (bit-exact walks -> identical path sets), vectors within 1e-4."""
    import g2vec_b200
    from g2vec_b200 import paths
    (rowptr, gene, label), o_rows = helpers.ex_windows(reps=10)
    rows = []
    for grp in (0, 1):
        rp, col, w = helpers.ex_graph(grp)
        wg = g2vec_b200.WalkGraph(rp, col, weights=w)
        nodes, lens = g2vec_b200.generate_paths(wg, 80, 10, seed=0, group=grp)
        rows.append(paths.canonical_rows(nodes, lens))
    prow, plab = paths.integrate(rows[0], rows[1])
    g_rowptr, g_gene, g_label = paths.windows_csr(prow, plab)
    N = len(rowptr) - 1
    assert g_rowptr.shape[0] - 1 == N and 40000 < N < 50000          # README.md:31 reports 45402 (unseeded)
    got_set = {(int(l), tuple(int(x) for x in r[r != paths.PAD])) for r, l in zip(prow.cpu().numpy(), plab.cpu().numpy())}
    assert got_set == set(o_rows)
    V, D = 7523, 128
    tr, va = oracle.split_indices(N, 0)
    W0, Wo0 = helpers.init_weights(V, D, 0)
    want, hist, _, _ = oracle.cbow_train(rowptr, gene, label, tr, va, W0, Wo0, 0.005, max_steps=5, early_stop=False)
    for algo in ("rows", "rank1"):
        got = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=5, seed=0, W_ih0=W0, W_ho0=Wo0,
                             early_stop=False, log=None, algo=algo)
        assert rel_max(got, want) < RTOL_VEC, algo


def test_ex_windows_early_stop_run(g2v):
    """Full reference loop with early stopping from four different initialisations.  The stop step depends on exact
    accuracy comparisons (G2Vec.py:276) and the GPU sums in a different float32 order, so a tie may break one step
    apart; the test records how many of the runs stop on the oracle's step (all of them in every run so far) and
    compares the vectors of those."""
    (rowptr, gene, label), _ = helpers.ex_windows(reps=2)
    V, D = 7523, 128
    N = len(rowptr) - 1
    tr, va = oracle.split_indices(N, 0)
    same = []
    for init_seed in range(4):
        W0, Wo0 = helpers.init_weights(V, D, init_seed)
        want, hist, stop, _ = oracle.cbow_train(rowptr, gene, label, tr, va, W0, Wo0, 0.005, max_steps=60)
        lines = []
        got, info = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=60, seed=0, W_ih0=W0, W_ho0=Wo0,
                                   log=lines.append, return_info=True)
        assert lines[0] == "     Start training the modified CBOW with early stopping"
        assert lines[1].startswith("    - Epoch: 000\tACC[val]=") and lines[-1] == "    Optimization Finish"
        s_gpu = info["stop_step"]
        assert (stop is None) == (s_gpu is None) or abs((stop or 60) - (s_gpu or 60)) <= 1, (init_seed, stop, s_gpu)
        same.append(stop == s_gpu)
        if stop == s_gpu:
            assert rel_max(got, want) < 5 * RTOL_VEC      # up to ~40 Adam steps of accumulated reassociation noise
        k = min(len(hist), len(info["history"])) - 1
        assert abs(hist[k][1] - info["history"][k][1]) < 5e-3
    print("early-stop runs on the oracle's step: %d of %d" % (sum(same), len(same)))
    assert sum(same) >= len(same) - 1


@pytest.mark.parametrize("name", ["cbow_small.npz", "cbow_ex.npz"])
@pytest.mark.parametrize("algo", ["rows", "rank1"])
def test_gpu_equals_the_reference_run(g2v, name, algo):
    """Against the reference ITSELF: tests/golden/cbow_*.npz hold what the unmodified compute_genetovec
    (G2Vec.py:217-286, on oracle/tf1_shim.py) returned for these windows, this seed and these initial tensors.
    The GPU run goes through the product's own split and init (same seed) and must give the reference's stop
    step, accuracies (within 2 windows) and vectors (1e-4 relative, north_star)."""
    g = helpers.cbow_golden(name)
    from g2vec_b200 import cbow
    W0, Wo0 = cbow.init_weights(g["V"], g["D"], g["seed"])
    assert (W0 == g["W0"]).all() and (Wo0 == g["Wo0"]).all()      # product init == the tensors the reference drew
    lines = []
    got, info = g2v.train_cbow(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"], max_epoch=500,
                               seed=g["seed"], log=lines.append, return_info=True, algo=algo)
    assert info["stop_step"] == g["stop_step"], (info["stop_step"], g["stop_step"])
    n_va, n_tr = len(g["va"]), len(g["tr"])
    for (s, av, at), rv, rt in zip(info["history"], g["acc_val"], g["acc_tr"]):
        assert abs(av - rv) <= 2.0 / n_va + 1e-7
        assert at is None or abs(at - rt) <= 2.0 / n_tr + 1e-7
    assert rel_max(got, g["W_ref"]) < RTOL_VEC
    # same log lines as the reference printed (G2Vec.py:259,271,278,284): same epochs, same stop line; the
    # four-decimal accuracies may differ by the window-flip tolerance above
    import re
    ref_lines = g["log"].splitlines()
    assert len(lines) == len(ref_lines)
    num = re.compile(r"ACC\[val\]=([0-9.]+)\tACC\[tr\]=([0-9.]+)")
    for a, b in zip(lines, ref_lines):
        assert a.split("ACC[val]")[0] == b.split("ACC[val]")[0]
        ma, mb = num.search(a), num.search(b)
        assert (ma is None) == (mb is None)
        if ma:
            assert abs(float(ma.group(1)) - float(mb.group(1))) <= 2.0 / n_va + 1.01e-4
            assert abs(float(ma.group(2)) - float(mb.group(2))) <= 2.0 / n_tr + 1.01e-4


def test_step_host_entry_point(g2v):
    V, N, D = 300, 1000, 128
    rowptr, gene, label = helpers.random_windows(N, V, 1, 40, seed=4)
    W0, Wo0 = helpers.init_weights(V, D, 3)
    W, Wo = W0.copy(), Wo0.copy()
    state, loss, nc = g2v.cbow_step_host(rowptr, gene, label, W, Wo, lr=0.005, t=1)
    win = np.arange(N, dtype=np.int64)
    o_gih, o_gho, o_loss, o_nc = oracle.cbow_grad(rowptr, gene, label, win, N, W0, Wo0)
    Wr, Wor = W0.copy(), Wo0.copy()
    mm, vv, mo, vo = np.zeros_like(Wr), np.zeros_like(Wr), np.zeros_like(Wor), np.zeros_like(Wor)
    oracle.adam_(Wr, mm, vv, o_gih, 0.005, 1); oracle.adam_(Wor, mo, vo, o_gho, 0.005, 1)
    assert rel_max(W, Wr) < RTOL_VEC and rel_max(Wo, Wor) < RTOL_VEC
    assert rel_max(state[0], mm) < 1e-4 and abs(nc - o_nc) <= 1 and abs(loss / N - o_loss) < 1e-5


# ------------------------------------------------------------------ collapsed (rank-1) trainer, SURVEY 8f-3
@pytest.mark.parametrize("D,optimizer,reduce", [(128, "adam", "sum"), (256, "adam", "sum"), (512, "adam", "sum"),
                                                (100, "adam", "sum"), (128, "sgd", "sum"), (64, "sgd", "mean"),
                                                (128, "adam", "mean")])
def test_rank1_one_step_equals_oracle(g2v, D, optimizer, reduce):
    import torch
    V, N = 500, 3000
    rowptr, gene, label = helpers.random_windows(N, V, 1, 80, seed=D + 1)
    W0, Wo0 = helpers.init_weights(V, D, 5)
    win = np.arange(N, dtype=np.int64)
    m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, optimizer=optimizer, reduce=reduce, lr=0.005, algo="rank1")
    m.fwdbwd(None, N, win_begin=0, n_win=N)
    torch.cuda.synchronize()
    acc = m.acc.cpu()
    c = m.c.cpu().numpy().copy()
    m.update()
    torch.cuda.synchronize()
    if reduce == "sum":
        o_gih, o_gho, o_loss, o_nc = oracle.cbow_grad(rowptr, gene, label, win, N, W0, Wo0)
        assert abs(m.loss_sum(acc) / N - o_loss) < 1e-5 * max(1.0, abs(o_loss)) and abs(int(acc[1]) - o_nc) <= 2
    else:   # mean variant: restate densely in float64
        lens = np.diff(rowptr).astype(np.float64)
        H = np.stack([W0[gene[rowptr[n]:rowptr[n + 1]]].astype(np.float64).sum(0) / lens[n] for n in range(N)])
        dO = (1 / (1 + np.exp(-(H @ Wo0.astype(np.float64)))) - label) / N
        o_gho = (H * dO[:, None]).sum(0)
        o_gih = np.zeros((V, D))
        for n in range(N):
            o_gih[gene[rowptr[n]:rowptr[n + 1]]] += dO[n] / lens[n] * Wo0
        o_gih = o_gih.astype(np.float32); o_gho = o_gho.astype(np.float32)
    # rank-1 structure: the dense gradient is c (x) W_ho
    assert rel_max(np.outer(c, Wo0), o_gih) < 5e-5
    W, Wo = W0.copy(), Wo0.copy()
    if optimizer == "adam":
        mm, vv, mo, vo = np.zeros_like(W), np.zeros_like(W), np.zeros_like(Wo), np.zeros_like(Wo)
        oracle.adam_(W, mm, vv, o_gih, 0.005, 1); oracle.adam_(Wo, mo, vo, o_gho, 0.005, 1)
    else:
        oracle.sgd_(W, o_gih, 0.005); oracle.sgd_(Wo, o_gho, 0.005)
    assert rel_max(m.W_ih.cpu().numpy(), W) < RTOL_VEC and rel_max(m.W_ho.cpu().numpy(), Wo) < RTOL_VEC
    assert float(m.c.abs().max()) == 0.0
    s_want = W @ Wo
    assert np.abs(m.s.cpu().numpy() - s_want).max() < 1e-5 * max(1.0, np.abs(s_want).max())


def test_rank1_ex_windows_five_steps_match_oracle(g2v):
    (rowptr, gene, label), _ = helpers.ex_windows(reps=2)
    V, D = 7523, 128
    N = len(rowptr) - 1
    tr, va = oracle.split_indices(N, 0)
    W0, Wo0 = helpers.init_weights(V, D, 0)
    want, hist, stop, _ = oracle.cbow_train(rowptr, gene, label, tr, va, W0, Wo0, 0.005, max_steps=5, early_stop=False)
    got, info = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=5, seed=0, W_ih0=W0, W_ho0=Wo0,
                               early_stop=False, log=None, return_info=True, algo="rank1")
    assert rel_max(got, want) < RTOL_VEC
    for (s, av, at), (s2, av2, at2) in zip(hist, info["history"]):
        assert abs(av - av2) <= 2.0 / len(va) + 1e-7 and abs(at - at2) <= 2.0 / len(tr) + 1e-7
    rows, _ = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=5, seed=0, W_ih0=W0, W_ho0=Wo0,
                             early_stop=False, log=None, return_info=True, algo="rows")
    assert rel_max(got, rows) < RTOL_VEC


def test_minibatch_variant_and_dense_adapter(g2v):
    """north_star's mini-batch variant (one optimizer step per batch) against an oracle loop; batch >= N is
    the reference's full batch; and the reference-shaped adapter compute_genetovec(dense pathList, ...)."""
    V, N, D = 300, 1200, 128
    rowptr, gene, label = helpers.random_windows(N, V, 1, 30, seed=12)
    W0, Wo0 = helpers.init_weights(V, D, 2)
    tr, va = oracle.split_indices(N, 0)
    B = 256
    W, Wo = W0.copy(), Wo0.copy()
    st = [np.zeros_like(W), np.zeros_like(W), np.zeros_like(Wo), np.zeros_like(Wo)]
    t = 0
    for epoch in range(2):
        for lo in range(0, len(tr), B):
            sub = tr[lo:lo + B]
            g_ih, g_ho, _, _ = oracle.cbow_grad(rowptr, gene, label, sub, len(sub), W, Wo)
            t += 1
            oracle.adam_(W, st[0], st[1], g_ih, 0.005, t); oracle.adam_(Wo, st[2], st[3], g_ho, 0.005, t)
    for algo in ("rows", "rank1"):
        got = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=2, seed=0, W_ih0=W0, W_ho0=Wo0,
                             early_stop=False, log=None, batch=B, algo=algo)
        assert rel_max(got, W) < RTOL_VEC, algo
    full = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=3, seed=0, W_ih0=W0, W_ho0=Wo0,
                          early_stop=False, log=None)
    big = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=3, seed=0, W_ih0=W0, W_ho0=Wo0,
                         early_stop=False, log=None, batch=10 * N)
    assert rel_max(big, full) < 1e-5
    # dense adapter: pathList [N, V+1] as integrate_pathSet builds it (G2Vec.py:316-320)
    P = np.zeros((N, V + 1), dtype=np.int32)
    for n in range(N):
        P[n, gene[rowptr[n]:rowptr[n + 1]]] = 1
    P[:, -1] = label
    lines = []
    a = g2v.compute_genetovec(P, V, D, 0.005, max_epoch=3, seed=0, log=lines.append)
    b = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=3, seed=0, log=None)
    assert a.shape == (V, D) and a.dtype == np.float32 and rel_max(a, b) < 1e-5
    assert lines[0].strip() == "Start training the modified CBOW with early stopping"


def test_rank1_csc_backward_is_bit_reproducible(g2v):
    """With the transposed incidence (CSC) the collapsed trainer has no floating-point atomics: two runs
    give bit-identical vectors (the row formulation, with red.global.add, does not promise that)."""
    (rowptr, gene, label), _ = helpers.ex_windows(reps=2)
    V, D = 7523, 128
    W0, Wo0 = helpers.init_weights(V, D, 0)
    runs = [g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=6, seed=0, W_ih0=W0, W_ho0=Wo0,
                           early_stop=False, log=None, algo="rank1") for _ in range(2)]
    assert (runs[0] == runs[1]).all()
    # and it equals the atomics form of the same algorithm to reassociation
    import torch
    N = len(rowptr) - 1
    m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, algo="rank1")
    win = torch.arange(N, dtype=torch.int32, device="cuda")
    m.fwdbwd(win, N); torch.cuda.synchronize()
    c_atomic = m.c.cpu().numpy().copy(); m.c.zero_()
    m.prepare_csc(win); m.fwdbwd(win, N); torch.cuda.synchronize()
    c_csc = m.c.cpu().numpy()
    assert np.abs(c_csc - c_atomic).max() <= 1e-5 * np.abs(c_atomic).max()


@pytest.mark.parametrize("algo", ["rows", "rank1"])
def test_graph_replayed_steps_equal_eager_steps(g2v, algo):
    """On one GPU train_cbow replays a CUDA graph per step (device-side Adam tick); results must equal the
    eager launches: bit-identical for rank1 (no atomics), to reassociation for rows."""
    (rowptr, gene, label), _ = helpers.ex_windows(reps=2)
    V, D = 7523, 128
    W0, Wo0 = helpers.init_weights(V, D, 0)
    kw = dict(max_epoch=12, seed=0, W_ih0=W0, W_ho0=Wo0, early_stop=False, log=None, algo=algo, return_info=True)
    a, ia = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, use_graph=True, **kw)
    b, ib = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, use_graph=False, **kw)
    if algo == "rank1":
        assert (a == b).all() and ia["history"] == ib["history"]
    else:
        assert rel_max(a, b) < 1e-5
    # the device-side tick reproduces the host formula: alpha_t of step 12
    m = ia["model"]
    b1p, b2p = np.float32(1), np.float32(1)
    for _ in range(12):
        b1p = np.float32(b1p * np.float32(0.9)); b2p = np.float32(b2p * np.float32(0.999))
    alpha = np.float32(0.005) * np.sqrt(np.float32(1) - b2p) / (np.float32(1) - b1p)
    h = m.hyper.cpu().numpy()
    assert h[0] == b1p and h[1] == b2p and abs(h[2] - alpha) <= 1e-9


@pytest.mark.parametrize("algo", ["rows", "rank1"])
def test_device_loop_early_stop_equals_host_driven_steps(g2v, algo):
    """The early stop decided on the device inside a 5-step CUDA graph (iterations after the drop are no-ops,
    the snapshot is the weights before the dropping step) against the same launches run eagerly."""
    g = helpers.cbow_golden("cbow_small.npz")
    kw = dict(max_epoch=500, seed=g["seed"], log=None, algo=algo, return_info=True)
    a, ia = g2v.train_cbow(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"], use_graph=True, **kw)
    b, ib = g2v.train_cbow(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"], use_graph=False, **kw)
    assert ia["graph"] and not ib["graph"]
    assert ia["stop_step"] == ib["stop_step"] == g["stop_step"] and g["stop_step"] % 5 not in (0,)   # mid-chunk stop
    assert len(ia["history"]) == len(ib["history"]) == g["stop_step"] + 1
    assert rel_max(a, b) < 1e-5 and rel_max(a, g["W_ref"]) < RTOL_VEC
    # --epoch below the stop step: the cap ends the loop, the result is the final weights
    c, ic = g2v.train_cbow(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"], use_graph=True,
                           **dict(kw, max_epoch=7))
    assert ic["stop_step"] is None and len(ic["history"]) == 7 and all(h[2] is not None for h in ic["history"])
    want, _, _, _ = oracle.cbow_train(g["rowptr"], g["gene"], g["label"], g["tr"], g["va"], g["W0"], g["Wo0"], g["lr"],
                                      max_steps=7, early_stop=False)
    assert rel_max(c, want) < RTOL_VEC


def test_window_feeder_double_buffered_uploads(g2v):
    """Feeding the windows from pinned host memory (int16 gene ids on the wire, two device buffer sets)
    gives the same step results as resident windows."""
    import torch
    V, N, D = 400, 3000, 128
    rowptr, gene, label = helpers.random_windows(N, V, 1, 50, seed=21)
    W0, Wo0 = helpers.init_weights(V, D, 1)
    win = torch.arange(N, dtype=torch.int32, device="cuda")
    a = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, algo="rank1"); a.prepare_csc(win)
    b = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, algo="rank1"); b.prepare_csc(win)
    feeder = g2v.WindowFeeder(b, rowptr, gene, label)
    assert feeder.narrow and feeder.h2d_bytes == 4 * (N + 1) + 2 * len(gene) + N
    feeder.upload(0)
    for i in range(4):
        k = i & 1
        if i < 3:
            feeder.upload(k ^ 1)
        feeder.use(k)
        for m in (a, b):
            m.acc.zero_(); m.fwdbwd(win, N); m.update(); m.evaluate(win, 2)
        feeder.release(k)
        torch.cuda.synchronize()
        assert (a.acc.cpu() == b.acc.cpu()).all()
    assert (a.W_ih == b.W_ih).all()


def test_cbow_full_size_properties(g2v):
    """BASELINE configs[1] size (10k genes, 200k windows of 80 genes, 128-dim): size-independent properties.
    (1) linearity: the gradient of all training windows = sum of the gradients of two halves (same 1/N);
    (2) the row formulation and the collapsed one train to the same vectors; (3) oracle equality on a
    2000-window sample of the same data; (4) accuracy counters of fwd+bwd equal those of the eval kernel."""
    import torch
    V, N, D, Lw = 10_000, 200_000, 128, 80
    rs = np.random.RandomState(777)
    gene = np.stack([rs.choice(V, Lw, replace=False) for _ in range(2000)])      # 2000 base windows ...
    gene = np.tile(gene, (N // 2000, 1))                                         # ... relabelled 100 times
    perm = rs.permutation(V)
    gene = np.sort((perm[gene] + (np.arange(N) // 2000)[:, None] * 37) % V, axis=1).astype(np.int32)   # distinct rows
    rowptr = (np.arange(N + 1) * Lw).astype(np.int32)
    label = (rs.rand(N) < 0.5).astype(np.uint8)
    W0, Wo0 = helpers.init_weights(V, D, 5)
    m = g2v.CbowModel(rowptr, gene.ravel(), label, V, D, W0, Wo0)
    m.fwdbwd(None, N, win_begin=0, n_win=N); torch.cuda.synchronize()
    full = m.g_ih.clone(); full_ho = m.g_ho.clone(); acc_full = m.acc.cpu().clone()
    m.g_ih.zero_(); m.g_ho.zero_(); m.acc.zero_()
    m.fwdbwd(None, N, win_begin=0, n_win=N // 2); m.fwdbwd(None, N, win_begin=N // 2, n_win=N - N // 2)
    m.evaluate(None, 2, win_begin=0, n_win=N); torch.cuda.synchronize()
    assert float((m.g_ih - full).abs().max()) <= 2e-5 * float(full.abs().max())
    assert float((m.g_ho - full_ho).abs().max()) <= 2e-5 * float(full_ho.abs().max())
    acc = m.acc.cpu()
    assert int(acc[1]) == int(acc_full[1]) == int(acc[2])                    # (4)
    sample = np.sort(rs.choice(N, 2000, replace=False)).astype(np.int64)
    o_gih, o_gho, _, o_nc = oracle.cbow_grad(rowptr, gene.ravel(), label, sample, N, W0, Wo0)
    m.g_ih.zero_(); m.g_ho.zero_(); m.acc.zero_()
    m.fwdbwd(torch.from_numpy(sample.astype(np.int32)).cuda(), N); torch.cuda.synchronize()
    assert rel_max(m.g_ih.cpu().numpy(), o_gih) < 2e-5 and abs(int(m.acc.cpu()[1]) - o_nc) <= 1
    tr = np.arange(N, dtype=np.int64)[: int(N * 0.8)]; va = np.arange(N, dtype=np.int64)[int(N * 0.8):]
    kw = dict(max_epoch=3, seed=0, W_ih0=W0, W_ho0=Wo0, split=(tr, va), early_stop=False, log=None)
    a = g2v.train_cbow(rowptr, gene.ravel(), label, V, D, 0.005, algo="rows", **kw)
    b = g2v.train_cbow(rowptr, gene.ravel(), label, V, D, 0.005, algo="rank1", **kw)
    assert rel_max(a, b) < RTOL_VEC


# ------------------------------------------------------------- gene-slab passes (tables larger than the L2)
@pytest.mark.parametrize("D,reduce,slabs,group", [(128, "sum", 2, 1), (128, "sum", 5, 2), (256, "sum", 3, 2),
                                                  (512, "sum", 7, 3), (512, "mean", 4, 2), (128, "mean", 3, 1)])
def test_slab_passes_equal_oracle_and_fused_kernel(g2v, monkeypatch, D, reduce, slabs, group):
    """csrc/g2v_cbow_slab.cu: the step processed gene slab by gene slab (forced here on a small table with
    G2V_CBOW_SLABS) gives the oracle's gradients, loss and accuracy counts, and the same update as the fused
    single-pass kernel; windows that have no gene in a slab, empty windows and a window list with an offset."""
    import torch
    V, N = 700, 2500
    rowptr, gene, label = helpers.random_windows(N, V, 0, 60, seed=D + slabs)     # lengths 0..60: empty windows too
    assert (np.diff(rowptr) == 0).sum() > 5
    W0, Wo0 = helpers.init_weights(V, D, 5)
    rs = np.random.RandomState(1)
    win = rs.permutation(N)[:2000].astype(np.int64)
    monkeypatch.setenv("G2V_CBOW_SLABS", str(slabs))
    monkeypatch.setenv("G2V_CBOW_SLAB_FWD_GROUP", str(group))
    m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, reduce=reduce, lr=0.005)
    wd = torch.from_numpy(win.astype(np.int32)).cuda()
    assert m.prepare_slabs(wd) and m._n_slabs == slabs
    m.fwdbwd(wd, len(win))
    m.evaluate(wd, 2)
    torch.cuda.synchronize()
    acc = m.acc.cpu()
    g_ih, g_ho = m.g_ih.cpu().numpy().copy(), m.g_ho.cpu().numpy().copy()
    monkeypatch.delenv("G2V_CBOW_SLABS")
    f = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, reduce=reduce, lr=0.005)      # fused single-pass kernel
    f.fwdbwd(wd, len(win))
    f.evaluate(wd, 2)
    torch.cuda.synchronize()
    facc = f.acc.cpu()
    assert rel_max(g_ih, f.g_ih.cpu().numpy()) < 2e-5 and rel_max(g_ho, f.g_ho.cpu().numpy()) < 2e-5
    assert abs(int(acc[1]) - int(facc[1])) <= 1 and abs(int(acc[2]) - int(facc[2])) <= 1
    assert abs(m.loss_sum(acc) - f.loss_sum(facc)) < 1e-5 * max(1.0, abs(f.loss_sum(facc)))
    if reduce == "sum":
        o_gih, o_gho, o_loss, o_nc = oracle.cbow_grad(rowptr, gene, label, win, len(win), W0, Wo0)
        assert rel_max(g_ih, o_gih) < 2e-5 and rel_max(g_ho, o_gho) < 2e-5
        assert abs(m.loss_sum(acc) / len(win) - o_loss) < 1e-5 * max(1.0, abs(o_loss))
        assert abs(int(acc[1]) - o_nc) <= 2 and abs(int(acc[2]) - o_nc) <= 2
    m.update(); f.update()
    torch.cuda.synchronize()
    assert rel_max(m.W_ih.cpu().numpy(), f.W_ih.cpu().numpy()) < RTOL_VEC


def test_slab_training_run_routes_both_lists_to_slabs_and_equals_the_golden(g2v, monkeypatch):
    """The whole loop (train_cbow: CUDA-graph replays, early stop) on slab passes against the reference run."""
    monkeypatch.setenv("G2V_CBOW_SLABS", "3")
    g = helpers.cbow_golden("cbow_ex.npz")
    got, info = g2v.train_cbow(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"], max_epoch=500,
                               seed=g["seed"], log=None, return_info=True)
    m = info["model"]
    assert m._n_slabs == 3 and all(m.prepared(w).slabs and m.route(w) == "slabs" for w in info["windows"])
    assert info["stop_step"] == g["stop_step"]
    assert rel_max(got, g["W_ref"]) < RTOL_VEC


def test_slab_setup_rejects_unsorted_windows(g2v, monkeypatch):
    import torch
    monkeypatch.setenv("G2V_CBOW_SLABS", "2")
    rowptr = np.array([0, 3, 5], dtype=np.int32); gene = np.array([4, 2, 9, 1, 3], dtype=np.int32)
    W0, Wo0 = helpers.init_weights(10, 128, 0)
    m = g2v.CbowModel(rowptr, gene, np.array([0, 1], dtype=np.uint8), 10, 128, W0, Wo0)
    with pytest.raises(RuntimeError, match="not strictly ascending"):
        m.prepare_slabs(None)


def test_slab_plan_at_the_stress_table_size_equals_the_single_pass_kernel(g2v, monkeypatch):
    """BASELINE configs[4]'s table (200k genes x 512 = 410 MB, 8x H100's L2): g2v_cbow_slab_plan must choose gene slabs on
    its own, and one step over 40k synthetic windows of 80 distinct genes must give the single-pass kernel's gradient,
    loss and accuracy counts (same sums, different float32 order), and the same accuracy pass."""
    import torch
    V, D, L, N = 200_000, 512, 80, 40_000
    gen = torch.Generator(device="cuda"); gen.manual_seed(777)
    x = torch.randint(0, V - L + 1, (N, L), generator=gen, device="cuda", dtype=torch.int32)
    x, _ = torch.sort(x, dim=1)
    x += torch.arange(L, device="cuda", dtype=torch.int32)[None, :]
    label = (torch.rand(N, generator=gen, device="cuda") < 0.5).to(torch.uint8)
    rowptr = torch.arange(0, (N + 1) * L, L, device="cuda", dtype=torch.int32)
    gene = x.reshape(-1).contiguous()
    s = 1.0 / np.sqrt(D)
    W0 = (torch.randn(V, D, device="cuda", generator=gen) * s).clamp_(-2 * s, 2 * s)
    Wo0 = (torch.randn(D, device="cuda", generator=gen) * s).clamp_(-2 * s, 2 * s)
    win = torch.randperm(N, device="cuda", generator=gen)[:32_000].to(torch.int32)
    m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0)
    assert m.prepare_slabs(win) and m._n_slabs >= 4                # the plan decided for slabs by itself
    m.fwdbwd(win, len(win)); m.evaluate(win, 2)
    monkeypatch.setenv("G2V_CBOW_SLABS", "1")
    f = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0)
    assert not f.prepare_slabs(win)
    f.fwdbwd(win, len(win)); f.evaluate(win, 2)
    torch.cuda.synchronize()
    scale = float(f.g_ih.abs().max())
    assert float((m.g_ih - f.g_ih).abs().max()) < 2e-5 * scale
    assert float((m.g_ho - f.g_ho).abs().max()) < 2e-5 * float(f.g_ho.abs().max())
    a, b = m.acc.cpu(), f.acc.cpu()
    assert abs(int(a[1]) - int(b[1])) <= 2 and abs(int(a[2]) - int(b[2])) <= 2 and int(b[1]) == int(b[2])
    assert abs(m.loss_sum(a) - f.loss_sum(b)) < 1e-5 * abs(f.loss_sum(b))
    # size-independent property: rows no window touches have a zero gradient; the touched ones are multiples of W_ho
    touched = torch.zeros(V, dtype=torch.bool, device="cuda")
    touched[gene.view(N, L)[win.long()].reshape(-1).long()] = True
    assert float(m.g_ih[~touched].abs().max()) == 0.0
    g = m.g_ih[touched][:2000]
    c = (g @ Wo0) / (Wo0 @ Wo0)                                      # g_ih[row] = c * W_ho  (rank-1 structure, SURVEY 3.2-3)
    assert float((g - c[:, None] * Wo0[None, :]).abs().max()) < 1e-5 * scale
