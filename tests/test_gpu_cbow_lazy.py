"""GPU checks of optimizer="lazy_adam" (TF1 LazyAdam on the embedding-lookup form of the rows trainer): the forward
stores dO per batch position (g2v_cbow_fwd_do), then one warp per gene the batch gathered sums its dO and takes the
Adam step on its W/m/v row with g = c * W_ho, followed by the dense W_ho step (g2v_cbow_lazy_adam)."""
import re

import numpy as np
import pytest

import oracle
from tests import helpers, lazy_adam_oracle

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


def _windows(N, V, unused, seed):
    """Random windows over genes [0, V - unused), window 4 empty and window 5 listing a gene twice."""
    rowptr, gene, label = helpers.random_windows(N, V - unused, 1, 80, seed=seed)
    rowptr[5] = rowptr[4]
    gene = gene[:rowptr[N - 1]].copy(); rowptr[N] = rowptr[N - 1]
    gene[rowptr[5] + 1] = gene[rowptr[5]]
    return rowptr, gene, label


@pytest.mark.parametrize("reduce", ["sum", "mean"])
@pytest.mark.parametrize("D", [128, 256, 512, 100])
def test_one_lazy_step_equals_oracle(g2v, D, reduce):
    import torch
    V, N, B, unused = 600, 1500, 1000, 40
    rowptr, gene, label = _windows(N, V, unused, seed=D + 11)
    assert len(set(gene[rowptr[5]:rowptr[6]])) < rowptr[6] - rowptr[5]         # a gene listed twice in a window
    W0, Wo0 = helpers.init_weights(V, D, 3)
    win = np.random.RandomState(D).permutation(N).astype(np.int64)
    for k, n in ((B + 1, 4), (B + 2, 5)):                                        # both in the second batch
        j = int(np.nonzero(win == n)[0][0])
        win[j], win[k] = win[k], win[j]
    wd = torch.from_numpy(win.astype(np.int32)).cuda()
    rs = np.random.RandomState(D + 1)
    st = [(rs.randn(V, D) * 1e-3).astype(np.float32), (rs.rand(V, D) * 1e-6 + 1e-7).astype(np.float32),
          (rs.randn(D) * 1e-3).astype(np.float32), (rs.rand(D) * 1e-6 + 1e-7).astype(np.float32)]

    m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, optimizer="lazy_adam", reduce=reduce)
    assert m.g_ih is None
    for dst, src in zip((m.m_ih, m.v_ih, m.m_ho, m.v_ho), st):
        dst.copy_(torch.from_numpy(src))
    m.prepare_batches(wd, B)
    lo, nb = B, N - B                                                            # the shorter, second batch
    sub = win[lo:lo + nb]
    assert m.batch_touched(wd, lo, nb) == len(lazy_adam_oracle.touched(rowptr, gene, sub))
    m.fwdbwd(wd, nb, win_begin=lo, n_win=nb)
    m.update()
    torch.cuda.synchronize()

    W, Wo = W0.copy(), Wo0.copy()
    ost = [a.copy() for a in st]
    lazy_adam_oracle.lazy_step(rowptr, gene, label, sub, W, Wo, ost, 0.005, 1, reduce=reduce)
    got = [m.W_ih, m.m_ih, m.v_ih, m.W_ho, m.m_ho, m.v_ho]
    got = [x.cpu().numpy() for x in got]
    for g, want in zip(got, [W, ost[0], ost[1], Wo, ost[2], ost[3]]):
        assert rel_max(g, want) < 2e-5
    out = np.setdiff1d(np.arange(V), lazy_adam_oracle.touched(rowptr, gene, sub))
    assert len(out) >= unused
    for g, x0 in zip(got[:3], (W0, st[0], st[1])):
        assert (g[out] == x0[out]).all()                                         # bit for bit
    assert (m.g_ho.cpu().numpy() == 0).all()


@pytest.mark.parametrize("D", [128, 100])
def test_full_batch_step_equals_csc_backward_and_dense_update(g2v, D):
    """From zero moments, one full-batch lazy step is the dense step: W_ih, m_ih, v_ih agree with
    g2v_cbow_fwdbwd_csc + g2v_cbow_update (both apply the same Adam arithmetic to the same per-gene sums)."""
    import torch
    V, N, unused = 500, 2000, 30
    rowptr, gene, label = _windows(N, V, unused, seed=D)
    W0, Wo0 = helpers.init_weights(V, D, 4)
    wd = torch.from_numpy(np.random.RandomState(1).permutation(N).astype(np.int32)).cuda()
    lazy = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, optimizer="lazy_adam")
    lazy.prepare_batches(wd, N)
    dense = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0)
    dense.prepare_csc(wd)
    for mdl in (lazy, dense):
        for _ in range(2):
            mdl.fwdbwd(wd, N)
            mdl.update()
    torch.cuda.synchronize()
    for a, b in ((lazy.W_ih, dense.W_ih), (lazy.m_ih, dense.m_ih), (lazy.v_ih, dense.v_ih), (lazy.W_ho, dense.W_ho)):
        a, b = a.cpu().numpy(), b.cpu().numpy()
        assert rel_max(a, b) < 1e-6
    assert (lazy.W_ih.cpu().numpy()[V - unused:] == W0[V - unused:]).all()


@pytest.mark.parametrize("name", ["cbow_small.npz", "cbow_ex.npz"])
def test_train_cbow_lazy_adam_reproduces_the_reference(g2v, name):
    g = helpers.cbow_golden(name)
    for use_graph in (True, False):
        got, info = g2v.train_cbow(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"], max_epoch=500,
                                   seed=g["seed"], log=None, return_info=True, use_graph=use_graph,
                                   optimizer="lazy_adam")
        assert info["stop_step"] == g["stop_step"], use_graph
        assert rel_max(got, g["W_ref"]) < RTOL_VEC, use_graph


def test_minibatch_lazy_adam_equals_oracle_and_differs_from_adam(g2v):
    """B = 256 of 960 training windows over 3000 genes: about a quarter of the genes sit out each batch, so lazy and
    dense Adam part ways.  (The init seed keeps every W_ho entry away from zero over the run: an entry crossing zero
    makes the sign of c * W_ho in its column, and with it Adam's first steps, depend on the last bits of W_ho.)"""
    V, N, D, B = 3000, 1200, 128, 256
    rowptr, gene, label = helpers.random_windows(N, V, 1, 30, seed=12)
    W0, Wo0 = helpers.init_weights(V, D, 4)
    tr, va = oracle.split_indices(N, 0)
    want, _ = lazy_adam_oracle.lazy_minibatch_train(rowptr, gene, label, tr, W0, Wo0, 0.005, B, 2)
    got = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=2, seed=0, W_ih0=W0, W_ho0=Wo0,
                         early_stop=False, log=None, batch=B, optimizer="lazy_adam")
    assert rel_max(got, want) < RTOL_VEC
    dense = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, max_epoch=2, seed=0, W_ih0=W0, W_ho0=Wo0,
                           early_stop=False, log=None, batch=B)
    assert rel_max(dense, want) > 10 * RTOL_VEC


def test_lazy_steps_call_neither_the_scatter_nor_the_dense_update(g2v, monkeypatch):
    from g2vec_b200 import _capi
    lib = _capi.load()
    calls = {k: 0 for k in ("g2v_cbow_fwdbwd", "g2v_cbow_fwdbwd_csc", "g2v_cbow_update", "g2v_cbow_fwd_do",
                            "g2v_cbow_lazy_adam")}

    def count(name, fn):
        def wrapped(*a):
            calls[name] += 1
            return fn(*a)
        return wrapped
    for k in calls:
        monkeypatch.setattr(lib, k, count(k, getattr(lib, k)))
    g = helpers.cbow_golden("cbow_small.npz")
    for batch, use_graph in ((0, False), (0, True), (64, False)):
        g2v.train_cbow(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"], max_epoch=6, seed=g["seed"],
                       early_stop=False, log=None, batch=batch, use_graph=use_graph, optimizer="lazy_adam")
    assert calls["g2v_cbow_fwdbwd"] == calls["g2v_cbow_fwdbwd_csc"] == calls["g2v_cbow_update"] == 0
    assert calls["g2v_cbow_fwd_do"] >= 6 and calls["g2v_cbow_lazy_adam"] >= 6


def test_lazy_adam_rejects_rank1_and_several_ranks(g2v, monkeypatch):
    from g2vec_b200 import cbow
    g = helpers.cbow_golden("cbow_small.npz")
    args = (g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"])
    with pytest.raises(ValueError):
        g2v.train_cbow(*args, max_epoch=2, log=None, algo="rank1", optimizer="lazy_adam")
    with pytest.raises(ValueError):
        g2v.CbowModel(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["W0"], g["Wo0"], optimizer="lazy_adam",
                      algo="rank1")

    class TwoRanks:                       # a process group of two; any collective would fail on this object
        def get_world_size(self):
            return 2

        def get_rank(self):
            return 0
    monkeypatch.setattr(cbow, "_dist", lambda: TwoRanks())
    with pytest.raises(ValueError):
        g2v.train_cbow(*args, max_epoch=2, log=None, optimizer="lazy_adam")


def test_command_line_with_lazy_minibatches(g2v, tmp_path, capsys):
    from g2vec_b200 import cli
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    prefix = str(tmp_path / "lazy")
    cli.main([ef, cf, nf, prefix, "-r", "2", "-e", "3", "-n", "20", "--seed", "3", "--batch", "4096",
              "--optimizer", "lazy_adam"])
    log = capsys.readouterr().out
    assert ">>> 4. Compute distributed representations using modified CBOW" in log
    assert "    - Epoch: 000\tACC[val]=" in log and "    Optimization Finish" in log
    vec = open(prefix + "_vectors.txt").read().splitlines()
    assert vec[0] == "GeneSymbol\t" + "\t".join("V%d" % i for i in range(128)) and len(vec) == 7524
    assert vec[1].split("\t")[0] == genes[0] and len(vec[1].split("\t")) == 129
    assert all(re.match(r"^-?\d+\.\d{6}$", x) for x in vec[1].split("\t")[1:])     # "%.6f"
    lg = open(prefix + "_lgroups.txt").read().splitlines()
    assert lg[0] == "GeneSymbol\tLgroup(0:good,1:poor,2:other)" and len(lg) == 7524
    assert {l.split("\t")[1] for l in lg[1:]} <= {"0", "1", "2"}
    bm = open(prefix + "_biomarkers.txt").read().splitlines()
    assert bm[0] == "GeneSymbol" and 1 <= len(bm) - 1 <= 40 and bm[1:] == sorted(bm[1:])
