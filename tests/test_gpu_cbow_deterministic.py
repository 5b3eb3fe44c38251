"""GPU checks of the deterministic rows trainer (DESIGN.md §4.13): the tiled forward gives the same bits for any launch
grid and agrees with the atomic path and the oracle; whole training runs repeat bit for bit (full batch with and
without the carry and CUDA graphs, mini-batches for every optimizer with and without reshuffling, tables forced onto
gene slabs, the command line); and each configuration launches the fixed-order kernels only."""

import numpy as np
import pytest

import oracle
from tests import helpers, lazy_adam_oracle, reshuffle_oracle as ro

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
def test_det_forward_on_a_prepared_record_is_grid_independent_and_matches_the_atomic_path(g2v, D, reduce):
    import torch
    from g2vec_b200 import _capi
    lib = _capi.load()
    V, N, n_list, unused = 700, 6000, 5600, 40            # 88 tiles, the last one partial
    rowptr, gene, label = _windows(N, V, unused, seed=D + 5)
    W0, Wo0 = helpers.init_weights(V, D, 2)
    win = np.random.RandomState(D).permutation(N)[:n_list].astype(np.int64)
    win[:2] = [4, 5]
    wd = torch.from_numpy(win.astype(np.int32)).cuda()
    m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, reduce=reduce, deterministic=True)
    m.prepare_csc(wd)
    rec = m.prepared(wd)
    ws = m.det_workspace(n_list)
    st = torch.cuda.current_stream().cuda_stream
    red = {"sum": 0, "mean": 1}[reduce]
    runs = []
    for max_ctas in (1, 3, 17, 0):
        dO = torch.full((n_list,), float("nan"), device="cuda")
        g_ih, g_ho = torch.zeros(V, D, device="cuda"), torch.zeros(D, device="cuda")
        acc = torch.zeros(2, dtype=torch.int64, device="cuda")
        l0 = _capi.launch_count()
        _capi.check(lib.g2v_cbow_fwdbwd_csc_det(m.rowptr.data_ptr(), m.gene.data_ptr(), m.label.data_ptr(),
                                                wd.data_ptr(), n_list, 1.0 / N, m.W_ih.data_ptr(), m.W_ho.data_ptr(),
                                                rec.cscptr.data_ptr(), rec.pos.data_ptr(), dO.data_ptr(), g_ih.data_ptr(),
                                                g_ho.data_ptr(), acc.data_ptr(), acc.data_ptr() + 8, V, D, red,
                                                ws.data_ptr(), max_ctas, st), "g2v_cbow_fwdbwd_csc_det")
        torch.cuda.synchronize()
        assert _capi.launch_count() - l0 == 3                # tiled forward, tile sum, per-gene expansion
        runs.append([x.cpu().numpy().copy() for x in (dO, g_ih, g_ho, acc)])
    for r in runs[1:]:
        for a, b in zip(r, runs[0]):
            assert a.tobytes() == b.tobytes()
    dO, g_ih, g_ho, acc = runs[0]
    loss = float(acc[:1].view(np.float64)[0])

    # the atomic path (g2v_cbow_fwd_do + g2v_cbow_fwdbwd_csc) and the oracle
    f = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, reduce=reduce)
    f.prepare_csc(wd)
    f.fwdbwd(wd, N)
    torch.cuda.synchronize()
    assert rel_max(dO, f.prepared(wd).dO.cpu().numpy()) < 1e-5
    assert rel_max(g_ih, f.g_ih.cpu().numpy()) < 2e-5 and rel_max(g_ho, f.g_ho.cpu().numpy()) < 2e-5
    assert abs(loss - f.loss_sum(f.acc.cpu())) < 1e-5 * abs(loss)
    assert int(acc[1]) == int(f.acc.cpu()[1])
    if reduce == "sum":
        o_gih, o_gho, o_loss, o_nc = oracle.cbow_grad(rowptr, gene, label, win, N, W0, Wo0)
        assert rel_max(g_ih, o_gih) < 2e-5 and rel_max(g_ho, o_gho) < 2e-5
        assert abs(loss / N - o_loss) < 1e-5 * max(1.0, abs(o_loss))
        assert abs(int(acc[1]) - o_nc) <= 2
    assert (g_ih[V - unused:] == 0).all()

    # the mini-batch forward: same bits for every grid too
    outs = []
    for max_ctas in (1, 17, 0):
        dO = torch.zeros(1000, device="cuda"); g_ho = torch.zeros(D, device="cuda")
        acc = torch.zeros(2, dtype=torch.int64, device="cuda")
        _capi.check(lib.g2v_cbow_fwd_do_det(m.rowptr.data_ptr(), m.gene.data_ptr(), m.label.data_ptr(),
                                            wd.data_ptr() + 4 * 300, 1000, 1e-3, m.W_ih.data_ptr(), m.W_ho.data_ptr(),
                                            dO.data_ptr(), g_ho.data_ptr(), acc.data_ptr(), acc.data_ptr() + 8, V, D,
                                            red, ws.data_ptr(), max_ctas, st), "g2v_cbow_fwd_do_det")
        outs.append(b"".join(x.cpu().numpy().tobytes() for x in (dO, g_ho, acc)))
    assert outs[0] == outs[1] == outs[2]


def _host_loop_without_carry(g2v, g, max_epoch=500):
    """The full-batch loop of train_cbow, enqueued step by step from the host with the carry turned off: every step
    runs its own training forward."""
    import torch
    from g2vec_b200 import cbow
    m = g2v.CbowModel(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["W0"], g["Wo0"], lr=g["lr"],
                      deterministic=True)
    tr_d = torch.from_numpy(np.ascontiguousarray(g["tr"], dtype=np.int32)).cuda()
    va_d = torch.from_numpy(np.ascontiguousarray(g["va"], dtype=np.int32)).cuda()
    m.prepare_csc(tr_d)
    loop = cbow.DeviceLoop(m, None, tr_d, va_d, len(g["tr"]), max_epoch, True)
    assert loop.carried
    loop.carried = False
    loop.attach()
    try:
        for _ in range(max_epoch):
            loop.one(True)
            loop.fetch()
            torch.cuda.synchronize()
            if int(loop.ctl_pin[0]):
                break
    finally:
        loop.detach()
    stop = int(loop.ctl_pin[2])
    W = (loop.result if stop >= 0 else m.W_ih).cpu().numpy()
    n = int(loop.ctl_pin[1])
    return W, m.W_ho.cpu().numpy(), loop.hist_pin[:4 * n].numpy().reshape(n, 4), (stop if stop >= 0 else None)


@pytest.mark.parametrize("name", ["cbow_small.npz", "cbow_ex.npz"])
def test_goldens_and_carried_graph_loop_equals_host_loop_bit_for_bit(g2v, name):
    g = helpers.cbow_golden(name)
    args = (g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"])
    got = {}
    for use_graph in (True, False):
        W, info = g2v.train_cbow(*args, max_epoch=500, seed=g["seed"], log=None, return_info=True, use_graph=use_graph,
                                 deterministic=True)
        assert info["stop_step"] == g["stop_step"], use_graph
        assert rel_max(W, g["W_ref"]) < RTOL_VEC, use_graph
        got[use_graph] = (W, info["model"].W_ho.cpu().numpy(), info["history"], info["stop_step"])
    assert got[True][0].tobytes() == got[False][0].tobytes() and got[True][1].tobytes() == got[False][1].tobytes()
    assert got[True][2:] == got[False][2:]
    W, Wo, hist, stop = _host_loop_without_carry(g2v, g)
    assert stop == got[True][3]
    assert W.tobytes() == got[True][0].tobytes() and Wo.tobytes() == got[True][1].tobytes()
    n_tr, n_va = len(g["tr"]), len(g["va"])
    f32 = np.float32
    want = [(s, float(f32(int(h[2])) / f32(n_va)), float(f32(int(h[3])) / f32(n_tr))) for s, h in enumerate(hist)]
    assert want == got[True][2]


def _minibatch_problem():
    V, N, D, B = 3000, 1200, 128, 256
    rowptr, gene, label = helpers.random_windows(N, V, 1, 30, seed=12)
    W0, Wo0 = helpers.init_weights(V, D, 4)
    tr, _ = oracle.split_indices(N, 0)
    return rowptr, gene, label, V, D, B, W0, Wo0, tr


@pytest.mark.parametrize("reshuffle", [False, True])
@pytest.mark.parametrize("optimizer", ["adam", "sgd", "lazy_adam"])
def test_minibatch_runs_repeat_bit_for_bit_and_match_the_oracle(g2v, optimizer, reshuffle):
    rowptr, gene, label, V, D, B, W0, Wo0, tr = _minibatch_problem()
    lr = 0.5 if optimizer == "sgd" else 0.005
    kw = dict(seed=0, W_ih0=W0, W_ho0=Wo0, early_stop=False, log=None, batch=B, optimizer=optimizer,
              reshuffle=reshuffle, return_info=True, deterministic=True)
    a, ia = g2v.train_cbow(rowptr, gene, label, V, D, lr, max_epoch=2, **kw)
    b, ib = g2v.train_cbow(rowptr, gene, label, V, D, lr, max_epoch=2, **kw)
    assert a.tobytes() == b.tobytes() and ia["history"] == ib["history"]
    assert ia["model"].W_ho.cpu().numpy().tobytes() == ib["model"].W_ho.cpu().numpy().tobytes()
    orders = ro.epoch_orders(tr, 0, 2) if reshuffle else [tr, tr]
    if optimizer == "lazy_adam":
        want, _ = ro.lazy_minibatch_train_orders(rowptr, gene, label, orders, W0, Wo0, lr, B)
    else:
        want, _ = ro.dense_minibatch_train_orders(rowptr, gene, label, orders, W0, Wo0, lr, B, optimizer)
    assert rel_max(a, want) < RTOL_VEC
    one = g2v.train_cbow(rowptr, gene, label, V, D, lr, max_epoch=1, **kw)[0]
    if optimizer == "lazy_adam":
        want1, _ = lazy_adam_oracle.lazy_minibatch_train(rowptr, gene, label, tr, W0, Wo0, lr, B, 1)
    else:
        want1, _ = ro.dense_minibatch_train_orders(rowptr, gene, label, [tr], W0, Wo0, lr, B, optimizer)
    assert rel_max(one, want1) < RTOL_VEC


def test_batch_expansion_matches_the_scatter(g2v):
    import torch
    from g2vec_b200 import _capi
    V, N, B, unused = 600, 1500, 1000, 40
    for D in (128, 100):
        rowptr, gene, label = _windows(N, V, unused, seed=D)
        W0, Wo0 = helpers.init_weights(V, D, 3)
        wd = torch.from_numpy(np.random.RandomState(D).permutation(N).astype(np.int32)).cuda()
        det = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, deterministic=True)
        det.prepare_batches(wd, B)
        ref = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0)
        for lo, nb in ((0, B), (B, N - B)):
            l0 = _capi.launch_count()
            det.fwdbwd(wd, nb, win_begin=lo, n_win=nb)
            torch.cuda.synchronize()
            assert _capi.launch_count() - l0 == 3                 # tiled forward, tile sum, batch expansion
            ref.fwdbwd(wd, nb, win_begin=lo, n_win=nb)
        torch.cuda.synchronize()
        assert rel_max(det.g_ih.cpu().numpy(), ref.g_ih.cpu().numpy()) < 2e-5
        assert rel_max(det.g_ho.cpu().numpy(), ref.g_ho.cpu().numpy()) < 2e-5
        assert (det.g_ih.cpu().numpy()[V - unused:] == 0).all()
        with pytest.raises(RuntimeError, match="prepare_batches"):
            det.fwdbwd(wd, 10, win_begin=3, n_win=10)


def test_large_tables_route_deterministic_runs_to_the_single_pass(g2v, monkeypatch):
    monkeypatch.setenv("G2V_CBOW_SLABS", "3")
    ex = helpers.cbow_golden("cbow_ex.npz")
    args = (ex["rowptr"], ex["gene"], ex["label"], ex["V"], ex["D"], ex["lr"])
    kw = dict(max_epoch=3, seed=ex["seed"], early_stop=False, log=None, return_info=True)
    slab, si = g2v.train_cbow(*args, **kw)
    assert si["model"]._n_slabs == 3
    det, di = g2v.train_cbow(*args, deterministic=True, **kw)
    tr_d = di["windows"][0]
    assert di["model"].prepared(tr_d).slabs == {} and di["model"].route(tr_d) == "csc_det"
    assert rel_max(det, slab) < RTOL_VEC


def _count_calls(monkeypatch, names):
    from g2vec_b200 import _capi
    lib = _capi.load()
    calls = {k: 0 for k in names}

    def count(name, fn):
        def wrapped(*a):
            calls[name] += 1
            return fn(*a)
        return wrapped
    for k in names:
        monkeypatch.setattr(lib, k, count(k, getattr(lib, k)))
    return calls


def test_each_configuration_launches_the_fixed_order_kernels_only(g2v, monkeypatch):
    calls = _count_calls(monkeypatch, ["g2v_cbow_fwdbwd", "g2v_cbow_fwdbwd_csc", "g2v_cbow_fwd_do", "g2v_cbow_loop_tail",
                                       "g2v_cbow_fwdbwd_slabs", "g2v_cbow_fwdbwd_csc_det", "g2v_cbow_fwd_do_det",
                                       "g2v_cbow_loop_tail_det", "g2v_cbow_batch_expand", "g2v_cbow_update",
                                       "g2v_cbow_lazy_adam", "g2v_cbow_batch_plan"])
    g = helpers.cbow_golden("cbow_small.npz")
    args = (g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"])
    kw = dict(max_epoch=6, seed=g["seed"], early_stop=False, log=None, deterministic=True)
    atomic = ("g2v_cbow_fwdbwd", "g2v_cbow_fwdbwd_csc", "g2v_cbow_fwd_do", "g2v_cbow_loop_tail", "g2v_cbow_fwdbwd_slabs")

    def run(expect, **extra):
        for k in calls:
            calls[k] = 0
        g2v.train_cbow(*args, **kw, **extra)
        assert all(calls[k] == 0 for k in atomic), (extra, calls)
        assert all(calls[k] == v for k, v in expect.items()), (extra, calls)
    # full batch: step 0 runs the forward, the tail pass carries every later one (6 tails, 6 expansions)
    run({"g2v_cbow_fwdbwd_csc_det": 6, "g2v_cbow_loop_tail_det": 6, "g2v_cbow_update": 6, "g2v_cbow_fwd_do_det": 0},
        use_graph=False)
    n_b = -(-len(g["tr"]) // 64)
    run({"g2v_cbow_fwd_do_det": 6 * n_b, "g2v_cbow_batch_expand": 6 * n_b, "g2v_cbow_update": 6 * n_b,
         "g2v_cbow_batch_plan": 1, "g2v_cbow_fwdbwd_csc_det": 0}, batch=64)
    run({"g2v_cbow_fwd_do_det": 6 * n_b, "g2v_cbow_batch_expand": 6 * n_b, "g2v_cbow_batch_plan": 6}, batch=64,
        optimizer="sgd", reshuffle=True)
    run({"g2v_cbow_fwd_do_det": 6 * n_b, "g2v_cbow_lazy_adam": 6 * n_b, "g2v_cbow_batch_expand": 0,
         "g2v_cbow_update": 0}, batch=64, optimizer="lazy_adam")


def test_rejected_configurations_and_rank1_full_batch(g2v, monkeypatch):
    from g2vec_b200 import cbow
    g = helpers.cbow_golden("cbow_small.npz")
    args = (g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"])
    with pytest.raises(ValueError):
        g2v.train_cbow(*args, max_epoch=2, log=None, algo="rank1", batch=64, deterministic=True)
    with pytest.raises(ValueError):
        g2v.CbowModel(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["W0"], g["Wo0"], deterministic=True,
                      nvl_group=object())
    kw = dict(max_epoch=5, seed=g["seed"], early_stop=False, log=None, algo="rank1")
    a = g2v.train_cbow(*args, deterministic=True, **kw)
    b = g2v.train_cbow(*args, **kw)
    assert a.tobytes() == b.tobytes()                      # full-batch rank1 is already reproducible: unchanged

    class TwoRanks:
        def get_world_size(self):
            return 2

        def get_rank(self):
            return 0
    monkeypatch.setattr(cbow, "_dist", lambda: TwoRanks())
    with pytest.raises(ValueError):
        g2v.train_cbow(*args, max_epoch=2, log=None, deterministic=True)


def test_command_line_runs_write_identical_files(g2v, tmp_path):
    from g2vec_b200 import cli
    ef, cf, nf, _ = helpers.write_ex_tsv(tmp_path)
    outs = []
    for k in (0, 1):
        prefix = str(tmp_path / ("det%d" % k))
        cli.main([ef, cf, nf, prefix, "-r", "2", "-e", "30", "-n", "20", "--seed", "3", "--deterministic"])
        outs.append([open(prefix + s, "rb").read() for s in ("_vectors.txt", "_lgroups.txt", "_biomarkers.txt")])
    assert outs[0] == outs[1]
    assert len(outs[0][0].splitlines()) == 7524
