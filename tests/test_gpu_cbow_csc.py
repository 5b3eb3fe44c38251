"""GPU parity of the rows trainer's CSC backward (g2v_cbow_fwdbwd_csc): the fused forward stores dO per list
position, and one warp per gene adds (sum of its windows' dO) * W_ho into the gene's gradient row -- against the
oracle, against the scatter kernel, and with the accumulation semantics of g2v_cbow_fwdbwd."""
import numpy as np
import pytest

import oracle
from tests import helpers

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def g2v():
    import torch
    assert torch.cuda.is_available()
    import g2vec_b200
    return g2vec_b200


def rel_max(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def mean_grad(rowptr, gene, label, win, n_total, W0, Wo0):
    """The segmented-MEAN variant's gradient of the listed windows, restated densely in float64."""
    V, D = W0.shape
    g_ih, g_ho, loss, nc = np.zeros((V, D)), np.zeros(D), 0.0, 0
    for n in win:
        gs = gene[rowptr[n]:rowptr[n + 1]]
        scale = 1.0 / len(gs) if len(gs) else 1.0
        h = W0[gs].astype(np.float64).sum(0) * scale
        o = float(h @ Wo0)
        dO = (1 / (1 + np.exp(-o)) - label[n]) / n_total
        g_ho += h * dO
        np.add.at(g_ih, gs, dO * scale * Wo0)           # a window may list a gene twice (window 5 below)
        loss += max(o, 0) - o * label[n] + np.log1p(np.exp(-abs(o)))
        nc += int((o > 0) == (label[n] != 0))
    return g_ih, g_ho, loss / n_total, nc


@pytest.mark.parametrize("reduce", ["sum", "mean"])
@pytest.mark.parametrize("D", [128, 256, 512, 100])
def test_csc_backward_equals_oracle_and_scatter_kernel(g2v, D, reduce):
    import torch
    from g2vec_b200 import _capi
    V, N, unused = 500, 3000, 40
    rowptr, gene, label = helpers.random_windows(N, V - unused, 1, 80, seed=D + 3)   # genes >= V - unused: in no window
    rowptr[5] = rowptr[4]                                                           # empty windows in the list
    gene = gene[:rowptr[N - 1]].copy(); rowptr[N] = rowptr[N - 1]
    W0, Wo0 = helpers.init_weights(V, D, 2)
    win = np.random.RandomState(D).permutation(N)[:2600].astype(np.int64)          # list position != window index
    win[:2] = [4, N - 1]
    wd = torch.from_numpy(win.astype(np.int32)).cuda()

    m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, reduce=reduce)
    m.prepare_csc(wd)
    l0 = _capi.launch_count()
    m.fwdbwd(wd, N)
    torch.cuda.synchronize()
    assert _capi.launch_count() - l0 == 2                  # fused forward with dO out + per-gene expansion
    acc = m.acc.cpu()
    g_ih, g_ho = m.g_ih.cpu().numpy().copy(), m.g_ho.cpu().numpy().copy()

    if reduce == "sum":
        o_gih, o_gho, o_loss, o_nc = oracle.cbow_grad(rowptr, gene, label, win, N, W0, Wo0)
    else:
        o_gih, o_gho, o_loss, o_nc = mean_grad(rowptr, gene, label, win, N, W0, Wo0)
    assert rel_max(g_ih, o_gih) < 2e-5 and rel_max(g_ho, o_gho) < 2e-5
    assert abs(m.loss_sum(acc) / N - o_loss) < 1e-5 * max(1.0, abs(o_loss))
    assert abs(int(acc[1]) - o_nc) <= 2
    assert (g_ih[V - unused:] == 0).all()                   # rows of genes in no listed window: exactly 0

    f = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, reduce=reduce)     # unprepared: the scatter kernel
    l0 = _capi.launch_count()
    f.fwdbwd(wd, N)
    torch.cuda.synchronize()
    assert _capi.launch_count() - l0 == 1
    assert rel_max(g_ih, f.g_ih.cpu().numpy()) < 2e-5 and rel_max(g_ho, f.g_ho.cpu().numpy()) < 2e-5

    # accumulation: the step adds into what g_ih / g_ho already hold; untouched rows keep their value bit for bit
    rs = np.random.RandomState(7)
    G0 = rs.randn(V, D).astype(np.float32) * np.float32(np.abs(o_gih).max())
    H0 = rs.randn(D).astype(np.float32) * np.float32(np.abs(o_gho).max())
    m.g_ih.copy_(torch.from_numpy(G0)); m.g_ho.copy_(torch.from_numpy(H0)); m.acc.zero_()
    m.fwdbwd(wd, N)
    torch.cuda.synchronize()
    got = m.g_ih.cpu().numpy()
    assert (got[V - unused:] == G0[V - unused:]).all()
    assert np.abs((got - G0) - o_gih).max() < 2e-5 * np.abs(o_gih).max() + 1e-6 * np.abs(G0).max()
    assert np.abs((m.g_ho.cpu().numpy() - H0) - o_gho).max() < 2e-5 * np.abs(o_gho).max() + 1e-6 * np.abs(H0).max()
    # no floating-point atomics on g_ih: the same step twice gives the same bits
    m.g_ih.zero_(); m.fwdbwd(wd, N); torch.cuda.synchronize()
    assert (m.g_ih.cpu().numpy() == g_ih).all()


def test_train_cbow_rows_runs_the_csc_backward(g2v, monkeypatch):
    """Full-batch train_cbow(algo="rows") prepares the transposed incidence of its training list and every step's
    backward goes through g2v_cbow_fwdbwd_csc; with gene slabs it is not prepared (the slab passes run instead)."""
    from g2vec_b200 import _capi
    lib = _capi.load()
    calls = {"csc": 0, "scatter": 0}
    csc, scatter = lib.g2v_cbow_fwdbwd_csc, lib.g2v_cbow_fwdbwd

    def count(name, fn):
        def wrapped(*a):
            calls[name] += 1
            return fn(*a)
        return wrapped
    monkeypatch.setattr(lib, "g2v_cbow_fwdbwd_csc", count("csc", csc))
    monkeypatch.setattr(lib, "g2v_cbow_fwdbwd", count("scatter", scatter))
    g = helpers.cbow_golden("cbow_small.npz")
    for use_graph in (True, False):
        got, info = g2v.train_cbow(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"], max_epoch=500,
                                   seed=g["seed"], log=None, return_info=True, use_graph=use_graph)
        assert info["model"]._csc is not None and info["stop_step"] == g["stop_step"]
        assert rel_max(got, g["W_ref"]) < 1e-4
    assert calls["csc"] >= g["stop_step"] and calls["scatter"] == 0
    monkeypatch.setenv("G2V_CBOW_SLABS", "3")
    ex = helpers.cbow_golden("cbow_ex.npz")
    _, info = g2v.train_cbow(ex["rowptr"], ex["gene"], ex["label"], ex["V"], ex["D"], ex["lr"], max_epoch=3,
                             seed=ex["seed"], early_stop=False, log=None, return_info=True)
    assert info["model"]._n_slabs == 3 and getattr(info["model"], "_csc", None) is None
