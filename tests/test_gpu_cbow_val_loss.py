"""GPU checks of the validation-loss monitor (DESIGN.md §4.19).

Entry points: Q of g2v_cbow_val_loss against the float64 loss of the same float32 logits (emulated in the kernel's lane
order) and of the float64 logits, on odd D and D = 128/256/512, reduce sum and mean, empty and long windows; Q the same
integer for any split of the list into shards, any order, eager or graph-replayed, on the slab and certified routes and
under rank1; the stopped word; the score exchange of simulated ranks (g2v_cbow_loop_score_nvl) and the decisions on it.

Trainer: monitor="val_acc" changes nothing; monitor="val_loss" stops where the CPU oracle (tests/val_loss_oracle.py)
stops and returns its best step's vectors; the plateau rule on the loss; reproducibility; the command line; several
GPUs (skipped on a one-GPU machine)."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from tests import helpers, lr_plateau_oracle as lro, val_loss_oracle as vo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL_VEC = 1e-4
TOP = 1 << 62


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available()
    from g2vec_b200 import _capi
    return {"lib": _capi.load(), "capi": _capi}


@pytest.fixture(scope="module")
def g2v():
    import torch
    assert torch.cuda.is_available()
    import g2vec_b200
    return g2vec_b200


def stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def cu(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def rel_max(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def problem(V, D, N, lmin, lmax, seed):
    rowptr, gene, label = helpers.random_windows(N, V, lmin, lmax, seed)
    W, Wo = helpers.init_weights(V, D, seed)
    return rowptr, gene, label, W, Wo


class Dev:
    """One problem on the device: the windows, the weights and st = {s, t} from g2v_cbow_st_prepare."""

    def __init__(self, env, rowptr, gene, label, W, Wo):
        import torch
        self.lib, self.capi = env["lib"], env["capi"]
        self.rp, self.ge, self.la = cu(rowptr), cu(gene), cu(label)
        self.V, self.D = W.shape
        self.W, self.Wo = cu(W), cu(Wo.reshape(-1))
        self.st = torch.zeros(2 * self.V, dtype=torch.float32, device="cuda")
        self.capi.check(self.lib.g2v_cbow_st_prepare(self.W.data_ptr(), self.Wo.data_ptr(), self.st.data_ptr(), self.V,
                                                     self.D, stream()), "g2v_cbow_st_prepare")

    def Q(self, win, reduce=0, s=None, stride=2, q=None):
        import torch
        q = torch.zeros(1, dtype=torch.int64, device="cuda") if q is None else q
        w = cu(np.asarray(win, np.int32))
        s = self.st if s is None else s
        self.capi.check(self.lib.g2v_cbow_val_loss(self.rp.data_ptr(), self.ge.data_ptr(), self.la.data_ptr(),
                                                   w.data_ptr(), 0, w.numel(), s.data_ptr(), stride, q.data_ptr(),
                                                   self.V, reduce, stream()), "g2v_cbow_val_loss")
        return int(q.cpu()[0])


# ------------------------------------------------------------------------------------------------ 1. the quantity
@pytest.mark.parametrize("reduce", [0, 1])
@pytest.mark.parametrize("D", [33, 128, 256, 512])
def test_q_against_float64(env, D, reduce):
    """Q equals the float64 loss of the float32 logits formed in the kernel's order from the device's s, to one unit per
    window (measured: exact), and the loss of the float64 logits within the logits' own float32 error (|dl/dz| <= 1).
    Windows of 0..200 genes (empty ones, and longer than 8 lanes x many rounds)."""
    rowptr, gene, label, W, Wo = problem(1001, D, 1500, 0, 200, D + reduce)
    d = Dev(env, rowptr, gene, label, W, Wo)
    red = "mean" if reduce else "sum"
    win = np.random.RandomState(D).permutation(1500)[:1200]
    Qd = d.Q(win, reduce)
    s = d.st.cpu().numpy()[0::2]
    z32 = vo.logits32(rowptr, gene, win, s, red)
    y = label[win]
    Q32 = int(vo.q_terms(z32, y).sum())
    z64 = vo.logits64(rowptr, gene, win, W, Wo, red)
    Q64 = int(vo.q_terms(z64, y).sum())
    dz = float(np.abs(z32.astype(np.float64) - z64).sum())
    print("D", D, red, "Q-Q32", Qd - Q32, "Q-Q64", Qd - Q64, "sum|dz|", dz)
    assert abs(Qd - Q32) <= len(win)
    assert abs(Qd - Q64) <= dz * 2 ** 24 + len(win)
    assert dz < 1e-3 * len(win)
    assert (np.diff(rowptr)[win] == 0).any() and (np.diff(rowptr)[win] > 150).any()


def test_saturation_and_non_finite_logits(env):
    """A logit beyond the cap or not finite adds exactly 64 * 2^24."""
    import torch
    rowptr = np.array([0, 1, 2, 3, 4], np.int32)
    gene = np.array([0, 1, 2, 3], np.int32)
    label = np.array([0, 1, 0, 1], np.uint8)
    W, Wo = np.zeros((4, 4), np.float32), np.zeros(4, np.float32)
    d = Dev(env, rowptr, gene, label, W, Wo)
    s = torch.tensor([[100.0, 0], [-100.0, 0], [float("inf"), 0], [float("nan"), 0]], device="cuda").reshape(-1)
    assert d.Q([0, 1, 2, 3], s=s) == 4 * 64 * 2 ** 24
    s = torch.tensor([[0.0, 0], [-100.0, 0], [100.0, 0], [0.0, 0]], device="cuda").reshape(-1)
    # window 0: z = 0 -> ln 2; window 2: z = 100 with y = 0 -> l = 100, capped at 64
    assert d.Q([0, 2], s=s) == int(np.rint(np.log(2.0) * 2 ** 24)) + 64 * 2 ** 24


@pytest.mark.parametrize("D", [33, 128])
def test_q_is_the_same_integer_for_any_split_order_and_grid(env, D):
    """The parts' Q add up to the whole's for random splits (each a different launch grid) and shard_by_nnz deals; the
    list in any order gives the same Q; with s given at stride 1 (rank1's layout) the same Q."""
    from g2vec_b200.cbow import shard_by_nnz
    rowptr, gene, label, W, Wo = problem(2003, D, 20000, 0, 90, 7)
    d = Dev(env, rowptr, gene, label, W, Wo)
    rs = np.random.RandomState(1)
    win = rs.permutation(20000)[:17000]
    for reduce in (0, 1):
        whole = d.Q(win, reduce)
        assert whole > 0
        for k in (2, 3, 7, 50):
            cuts = np.sort(rs.randint(0, len(win) + 1, size=k - 1))
            parts = np.split(win, cuts)
            assert sum(d.Q(p, reduce) for p in parts) == whole, (k, reduce)
        lens = np.diff(rowptr).astype(np.int64)
        for world in (2, 5):
            assert sum(d.Q(shard_by_nnz(win, lens, world, r), reduce) for r in range(world)) == whole
        assert d.Q(win[::-1], reduce) == whole and d.Q(rs.permutation(win), reduce) == whole
        s1 = d.st[0::2].contiguous()
        assert d.Q(win, reduce, s=s1, stride=1) == whole


def test_graph_replay_and_the_stopped_word(env):
    import torch
    rowptr, gene, label, W, Wo = problem(1001, 128, 5000, 0, 60, 3)
    d = Dev(env, rowptr, gene, label, W, Wo)
    win = cu(np.arange(5000, dtype=np.int32))
    eager = d.Q(np.arange(5000))
    q = torch.zeros(1, dtype=torch.int64, device="cuda")
    lib, capi = d.lib, d.capi
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            capi.check(lib.g2v_cbow_val_loss(d.rp.data_ptr(), d.ge.data_ptr(), d.la.data_ptr(), win.data_ptr(), 0, 5000,
                                             d.st.data_ptr(), 2, q.data_ptr(), d.V, 0,
                                             torch.cuda.current_stream().cuda_stream), "capture")
    for k in range(1, 4):
        g.replay()
        torch.cuda.synchronize()
        assert int(q.cpu()[0]) == k * eager
    # an attached, stopped loop: nothing is added
    ctl = torch.zeros(8, dtype=torch.int64, device="cuda")
    capi.check(lib.g2v_cbow_loop_init(ctl.data_ptr(), 4, 1, stream()), "init")
    ctl[0] = 1
    capi.check(lib.g2v_cbow_loop_attach(ctl.data_ptr()), "attach")
    try:
        q.zero_()
        d.Q(np.arange(5000), q=q)
    finally:
        capi.check(lib.g2v_cbow_loop_attach(None), "detach")
    assert int(q.cpu()[0]) == 0
    # refused arguments launch nothing
    l0 = capi.launch_count()
    assert lib.g2v_cbow_val_loss(d.rp.data_ptr(), d.ge.data_ptr(), d.la.data_ptr(), win.data_ptr(), 0, 5000,
                                 d.st.data_ptr(), 3, q.data_ptr(), d.V, 0, stream()) != 0
    assert lib.g2v_cbow_val_loss(d.rp.data_ptr(), d.ge.data_ptr(), d.la.data_ptr(), win.data_ptr(), 0, 5000,
                                 d.st.data_ptr(), 2, None, d.V, 0, stream()) != 0
    assert capi.launch_count() == l0


def _model(g2v, g, algo="rows"):
    from g2vec_b200 import cbow
    return cbow.CbowModel(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["W0"], g["Wo0"], algo=algo)


def test_routes_agree_slab_certified_rank1(g2v, monkeypatch):
    """CbowModel.evaluate(..., loss=True) on one set of weights: the certified route and the gene-slab route (a fresh st)
    give the same Q bit for bit; rank1 (its own s) agrees with rows to the float32 error of s."""
    import torch
    g = helpers.cbow_golden("cbow_ex.npz")
    va = cu(np.asarray(g["va"], np.int32))
    plain = _model(g2v, g)
    plain.evaluate(va, 2, loss=True)
    monkeypatch.setenv("G2V_CBOW_SLABS", "3")
    slab = _model(g2v, g)
    assert slab.prepare_slabs(va) and slab.route(va) == "slabs"
    slab.evaluate(va, 2, loss=True)
    monkeypatch.delenv("G2V_CBOW_SLABS")
    r1 = _model(g2v, g, algo="rank1")
    r1.evaluate(va, 2, loss=True)
    torch.cuda.synchronize()
    Qp, Qs, Qr = int(plain.q.cpu()[0]), int(slab.q.cpu()[0]), int(r1.q.cpu()[0])
    assert Qp == Qs and Qp > 0
    assert int(plain.acc[2].cpu()) == int(slab.acc[2].cpu()) == int(r1.acc[2].cpu())
    s_rows, s_r1 = plain.st.cpu().numpy()[0::2], r1.s.cpu().numpy()
    print("rank1 - rows:", Qr - Qp, "s bits equal:", s_rows.tobytes() == s_r1.tobytes())
    if s_rows.tobytes() == s_r1.tobytes():
        assert Qr == Qp
    z_r, z_p = (vo.logits32(g["rowptr"], g["gene"], g["va"], s) for s in (s_r1, s_rows))
    assert abs(Qr - Qp) <= np.abs(z_r.astype(np.float64) - z_p).sum() * 2 ** 24 + len(g["va"])
    Q64 = vo.Q(g["rowptr"], g["gene"], g["label"], g["va"], g["W0"], g["Wo0"])
    assert abs(vo.mean_loss(Qp, len(g["va"])) - vo.mean_loss(Q64, len(g["va"]))) < 1e-6


# ------------------------------------------------------------------------------------- 2. decisions and the exchange
QTRAJ = [9, 8, 8, 7, 7, 9, 6, 6, 8, 10, 11, 12]        # units of 2^30: ties, a rise, a new best, rises to the end


@pytest.mark.parametrize("rule", ["decide", "best1", "best3"])
@pytest.mark.parametrize("world", [1, 2, 3, 5])
def test_score_exchange_and_decisions(env, world, rule):
    """Each step every simulated rank adds its part of Q with g2v_cbow_loop_score_nvl, then decides with q == NULL; a
    single-rank loop decides on the whole Q through q.  Every rank ends with the single loop's ctl, best and score row
    2^62 - Q; q is cleared; a stopped loop adds and changes nothing; the stop and best steps are the loss rule's."""
    import torch
    lib, capi = env["lib"], env["capi"]
    K = 3 if rule == "best3" else 1
    T = len(QTRAJ)
    rs = np.random.RandomState(world * 11 + K)
    totals = [q * 2 ** 30 for q in QTRAJ] + [5, 5]             # two more steps after max_steps
    i64 = lambda n: torch.zeros(n, dtype=torch.int64, device="cuda")
    off = 4 * (T + 2)
    ctl, q, buf, hist = [i64(8) for _ in range(world + 1)], [i64(1) for _ in range(world + 1)], [], []
    for r in range(world + 1):
        buf.append(i64(off + T + 2))
        capi.check(lib.g2v_cbow_loop_init(ctl[r].data_ptr(), T, 1, stream()), "init")
    best = [torch.tensor([K, -1, 0, 0], dtype=torch.int64, device="cuda") for _ in range(world + 1)]
    tab = torch.tensor([b.data_ptr() for b in buf[:world]], dtype=torch.int64, device="cuda")

    def decide(r, qp):
        sc = buf[r].data_ptr() + 8 * off
        if rule == "decide":
            capi.check(lib.g2v_cbow_loop_decide_score(ctl[r].data_ptr(), None, buf[r].data_ptr(), qp, sc, stream()), "d")
        else:
            capi.check(lib.g2v_cbow_loop_decide_best_score(ctl[r].data_ptr(), best[r].data_ptr(), None,
                                                           buf[r].data_ptr(), qp, sc, stream()), "db")

    for s in range(T + 2):
        stopped = bool(ctl[world].cpu()[0])
        prev = [b.cpu().numpy().copy() for b in buf]
        cuts = np.sort(rs.randint(0, totals[s] + 1, size=world - 1))
        parts = np.diff(np.concatenate([[0], cuts, [totals[s]]])).astype(np.int64)
        for r in range(world):
            q[r].fill_(int(parts[r]))
            capi.check(lib.g2v_cbow_loop_score_nvl(ctl[r].data_ptr(), q[r].data_ptr(), tab.data_ptr(), None, off, world,
                                                   stream()), "score_nvl")
        for r in range(world):
            decide(r, None)
        q[world].fill_(totals[s])
        decide(world, q[world].data_ptr())
        c = [x.cpu().numpy() for x in ctl]
        b = [x.cpu().numpy() for x in best]
        h = [x.cpu().numpy() for x in buf]
        for r in range(world):
            assert (c[r] == c[world]).all() and (b[r] == b[world]).all(), (rule, world, s, r)
            if stopped:
                assert (h[r] == prev[r]).all() and int(q[r].cpu()[0]) == int(parts[r])
            else:
                assert h[r][off + s] == TOP - totals[s] == h[world][off + s]
                assert int(q[r].cpu()[0]) == 0
        if not stopped:
            assert int(q[world].cpu()[0]) == 0
    stop, best_step = vo.apply_rule(totals[:T], K)
    c = ctl[0].cpu().numpy()
    assert c[0] == 1 and c[2] == (-1 if stop is None else stop)
    if rule != "decide":
        assert best[0].cpu().numpy()[1] == best_step
    assert stop is not None


def test_plateau_kernel_on_the_score(env):
    """g2v_cbow_lr_plateau with counts = the score row, stride 1: the loss rule's rates (a tie is no improvement)."""
    import torch
    lib, capi = env["lib"], env["capi"]
    Qs = [q * 2 ** 30 for q in QTRAJ]
    cap = len(Qs)
    head = torch.tensor([1, -1, 0, 0, 0, cap, 0, 0], dtype=torch.int64)
    rates = torch.zeros(4 + cap + (cap & 1), dtype=torch.float32)
    rates[:3] = torch.tensor([0.01, 0.5, 0.0])
    st = torch.cat([head, rates.view(torch.int64)]).cuda()
    score = cu(np.array([TOP - q for q in Qs], np.int64))
    n = cu(np.array([cap], np.int64))
    capi.check(lib.g2v_cbow_lr_plateau(st.data_ptr(), score.data_ptr(), 1, n.data_ptr(), stream()), "lr_plateau")
    from g2vec_b200.cbow import lr_rates
    got, cuts = lr_rates(st.cpu())
    used, want_cuts, _ = vo.rates(Qs, 0.01, 1, 0.5)
    assert got == [float(r) for r in used] and cuts == want_cuts and cuts


# ------------------------------------------------------------------------------------------------ 3. the trainer
def _args(g):
    return (g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"])


def _record_calls(monkeypatch):
    from g2vec_b200 import cbow
    seen = []
    real = cbow.CbowModel._launch

    def launch(self, name, *a):
        seen.append(name)
        return real(self, name, *a)
    monkeypatch.setattr(cbow.CbowModel, "_launch", launch)
    return seen


OFF_CONFIGS = [
    ("cbow_ex.npz", dict(), False),
    ("cbow_ex.npz", dict(use_graph=False), False),
    ("cbow_ex.npz", dict(early_stop=True, patience=13), False),
    ("cbow_ex.npz", dict(deterministic=True, lr_patience=1), True),
    ("cbow_ex.npz", dict(slabs=True), False),
    ("cbow_ex.npz", dict(algo="rank1"), True),
    ("cbow_small.npz", dict(batch=64, lr_patience=2), False),
    ("cbow_small.npz", dict(batch=64, reshuffle=True, optimizer="lazy_adam", deterministic=True), True),
]


@pytest.mark.parametrize("golden,kw,exact", OFF_CONFIGS)
def test_val_acc_changes_nothing(g2v, monkeypatch, golden, kw, exact):
    from g2vec_b200 import _capi
    kw = dict(kw)
    if kw.pop("slabs", False):
        monkeypatch.setenv("G2V_CBOW_SLABS", "3")
    kw.setdefault("early_stop", False)
    g = helpers.cbow_golden(golden)
    seen = _record_calls(monkeypatch)
    runs = []
    for extra in ({}, {"monitor": "val_acc"}):
        del seen[:]
        lines = []
        l0 = _capi.launch_count()
        W, info = g2v.train_cbow(*_args(g), max_epoch=12, seed=g["seed"], log=lines.append, return_info=True, **kw,
                                 **extra)
        runs.append((W, info, _capi.launch_count() - l0, list(seen), [l.split(" (")[0] for l in lines]))
    (W0, i0, n0, s0, l0_), (W1, i1, n1, s1, l1_) = runs
    assert n1 == n0 and s1 == s0 and l1_ == l0_
    assert not any("val_loss" in x or "score" in x or "st_prepare" in x for x in s0)
    assert "val_loss" not in i0 and "val_loss" not in i1
    if exact:
        assert W1.tobytes() == W0.tobytes() and i1["history"] == i0["history"] and i1["lr"] == i0["lr"]
    else:
        assert rel_max(W1, W0) < 1e-5


_oracle = {}


def oracle_run(name, patience):
    if (name, patience) not in _oracle:
        g = helpers.cbow_golden(name)
        _oracle[(name, patience)] = vo.cbow_train(g["rowptr"], g["gene"], g["label"], g["tr"], g["va"], g["W0"],
                                                  g["Wo0"], g["lr"], max_steps=80, patience=patience)
    return _oracle[(name, patience)]


@pytest.mark.parametrize("name,patience,want", [("cbow_small.npz", 1, (25, 24)), ("cbow_ex.npz", 1, (11, 10)),
                                                ("cbow_small.npz", 3, (27, 24)), ("cbow_ex.npz", 3, (13, 10))])
@pytest.mark.parametrize("kw", [dict(), dict(use_graph=False), dict(keep_best=True), dict(algo="rank1"),
                                dict(slabs=True), dict(deterministic=True)],
                         ids=["carried-graph", "carried-eager", "keep-best", "rank1", "slabs", "deterministic"])
def test_golden_stop_and_best_steps_and_vectors(g2v, monkeypatch, name, patience, want, kw):
    from g2vec_b200 import cbow
    kw = dict(kw)
    if kw.pop("keep_best", False):
        monkeypatch.setattr(cbow.DeviceLoop, "keep_best_from", 1)
    if kw.pop("slabs", False):
        if name != "cbow_ex.npz":
            pytest.skip("the slab route is tested on cbow_ex")
        monkeypatch.setenv("G2V_CBOW_SLABS", "3")
    g = helpers.cbow_golden(name)
    W_want, _, Qs, stop, best = oracle_run(name, patience)
    assert (stop, best) == want
    lines = []
    W, info = g2v.train_cbow(*_args(g), max_epoch=80, seed=g["seed"], W_ih0=g["W0"], W_ho0=g["Wo0"], log=lines.append,
                             return_info=True, patience=patience, monitor="val_loss", **kw)
    assert (info["stop_step"], info["best_step"]) == want
    err = rel_max(W, W_want)
    n_va = len(g["va"])
    dl = max(abs(a - vo.mean_loss(b, n_va)) for a, b in zip(info["val_loss"], Qs))
    print(name, patience, kw, "rel", err, "max |loss - oracle|", dl)
    assert err < RTOL_VEC and dl < 1e-5
    assert len(info["val_loss"]) == want[0] + 1
    assert lines[-2].startswith("    - Epoch(stop): %03d\t" % want[1]) and "\tLOSS[val]=%.6f (" % \
        info["val_loss"][want[1]] in lines[-2]
    assert all("\tLOSS[val]=" in l for l in lines if l.startswith("    - Epoch"))


def test_minibatch_loop_decides_on_the_loss(g2v):
    """Mini-batches (host decision after each epoch's sync): the stop and best steps are the rule's on the returned loss
    trajectory, and the returned vectors are those of a run cut at the best epoch."""
    g = helpers.cbow_golden("cbow_small.npz")
    kw = dict(seed=g["seed"], W_ih0=g["W0"], W_ho0=g["Wo0"], log=None, return_info=True, batch=64, deterministic=True)
    W, info = g2v.train_cbow(*_args(g), max_epoch=60, patience=2, monitor="val_loss", **kw)
    n_va = len(g["va"])
    Qs = [int(round(l * n_va * 2 ** 24)) for l in info["val_loss"]]
    assert (info["stop_step"], info["best_step"]) == vo.apply_rule(Qs, 2)
    assert info["stop_step"] is not None
    W_cut, _ = g2v.train_cbow(*_args(g), max_epoch=info["best_step"] + 1, early_stop=False, **kw)
    assert W.tobytes() == W_cut.tobytes()


@pytest.mark.parametrize("batch,optimizer", [(0, "adam"), (64, "lazy_adam")])
def test_plateau_fires_on_the_loss(g2v, batch, optimizer):
    g = helpers.cbow_golden("cbow_ex.npz" if batch == 0 else "cbow_small.npz")
    epochs = 30
    W, info = g2v.train_cbow(*_args(g), max_epoch=epochs, seed=g["seed"], W_ih0=g["W0"], W_ho0=g["Wo0"], log=None,
                             return_info=True, batch=batch, optimizer=optimizer, early_stop=False, lr_patience=1,
                             lr_factor=0.5, monitor="val_loss")
    n_va = len(g["va"])
    Qs = [int(round(l * n_va * 2 ** 24)) for l in info["val_loss"]]
    used, cuts, _ = vo.rates(Qs, g["lr"], 1, 0.5)
    assert info["lr"] == [float(r) for r in used] and info["lr_reductions"] == cuts and cuts
    if batch == 0:
        # the oracle's trajectory cuts at the same steps, and the vectors follow the float64 trainer at those rates
        o_used, o_cuts, _ = vo.rates(_trajectory_with_rates(g, used), g["lr"], 1, 0.5)
        assert o_cuts == cuts
        want, _ = lro.adam64_train(g["rowptr"], g["gene"], g["label"], [g["tr"]] * epochs, g["W0"], g["Wo0"], used)
        assert rel_max(W, want) < RTOL_VEC


def _trajectory_with_rates(g, rates):
    """Q per step of float32 oracle Adam (oracle.cbow_grad) driven at the given per-step rates."""
    import oracle
    W = np.array(g["W0"], np.float32, copy=True)
    Wo = np.array(g["Wo0"], np.float32, copy=True).reshape(-1)
    m, v, mo, vo_ = np.zeros_like(W), np.zeros_like(W), np.zeros_like(Wo), np.zeros_like(Wo)
    Qs = []
    for t, lr in enumerate(rates):
        gi, gh, _, _ = oracle.cbow_grad(g["rowptr"], g["gene"], g["label"], g["tr"], len(g["tr"]), W, Wo)
        oracle.adam_(W, m, v, gi, float(lr), t + 1)
        oracle.adam_(Wo, mo, vo_, gh, float(lr), t + 1)
        Qs.append(vo.Q(g["rowptr"], g["gene"], g["label"], g["va"], W, Wo))
    return Qs


def test_deterministic_runs_repeat(g2v):
    g = helpers.cbow_golden("cbow_small.npz")
    for kw in (dict(), dict(batch=64, reshuffle=True), dict(algo="rank1")):
        outs = []
        for _ in range(2):
            W, info = g2v.train_cbow(*_args(g), max_epoch=30, seed=g["seed"], log=None, return_info=True,
                                     deterministic=kw.get("algo") != "rank1", patience=3, monitor="val_loss", **kw)
            outs.append((W.tobytes(), info["model"].W_ho.cpu().numpy().tobytes(), info["val_loss"],
                         info["stop_step"], info["best_step"]))
        assert outs[0] == outs[1], kw


def test_command_line(g2v, tmp_path, capsys):
    from g2vec_b200 import cli
    ef, cf, nf, _ = helpers.write_ex_tsv(tmp_path)
    prefix = str(tmp_path / "loss")
    cli.main([ef, cf, nf, prefix, "-r", "2", "-n", "20", "--seed", "3", "--deterministic", "--monitor", "val_loss",
              "--patience", "2"])
    out = capsys.readouterr().out
    files = [open(prefix + s).read() for s in ("_vectors.txt", "_lgroups.txt", "_biomarkers.txt")]
    assert all(len(f) > 0 for f in files)
    epoch = [l for l in out.splitlines() if l.startswith("    - Epoch")]
    assert epoch and all("\tLOSS[val]=" in l for l in epoch)
    assert any(l.startswith("    - Epoch(stop)") or l.startswith("    - Epoch(best)") for l in epoch) or len(epoch) > 50


def test_several_gpus_agree_on_the_loss(g2v, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    world = min(torch.cuda.device_count(), 4)
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out = str(tmp_path / "mgpu_val_loss.npz")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "mgpu_val_loss_worker.py"), out]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    z = np.load(out)
    (rowptr, gene, label), _ = helpers.ex_windows(reps=2)
    W0, Wo0 = helpers.init_weights(7523, 128, 0)
    W1, one = g2v.train_cbow(rowptr, gene, label, 7523, 128, 0.005, max_epoch=30, seed=0, W_ih0=W0, W_ho0=Wo0,
                             log=None, return_info=True, patience=3, lr_patience=1, lr_factor=0.5, monitor="val_loss")
    for k in ("nvl", "nccl"):
        loss = z[k + "_loss"]                    # [world, steps]: every rank's record
        assert (loss == loss[0]).all(), k
        n_va = one["n_val"]
        Qs = [int(round(l * n_va * 2 ** 24)) for l in loss[0]]
        assert tuple(z[k + "_steps"]) == tuple(-1 if x is None else x for x in vo.apply_rule(Qs, 3)), k
        assert np.abs(loss[0][:len(one["val_loss"])] - one["val_loss"][:len(loss[0])]).max() < 1e-5, k
    assert str(z["exchange"][1]).startswith("nccl")
