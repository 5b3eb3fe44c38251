"""GPU checks of the reduce-on-plateau learning rate (DESIGN.md §4.17): the Adam tick from a device rate against
g2v_cbow_adam_tick and TF1's float32 formula; the decision kernel against the CPU rule (tests/lr_plateau_oracle.py) in
both of its forms and from a captured CUDA graph; a schedule that never fires gives the bits of a run without it; a
firing schedule gives the rule's rates on the run's own validation counts and the vectors of a float64 Adam trainer
fed those rates, in every loop that trains with Adam; early stopping keeps its rule; the command line; N GPUs."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from tests import helpers, lr_plateau_oracle as lro, patience_oracle, reshuffle_oracle

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL_VEC = 1e-4
F32 = np.float32
NEW = ("g2v_cbow_lr_plateau", "g2v_cbow_adam_tick_lr")


@pytest.fixture(scope="module")
def g2v():
    import torch
    assert torch.cuda.is_available()
    import g2vec_b200
    return g2vec_b200


def rel_max(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _args(g):
    return (g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"])


def _stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


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


# ---------------------------------------------------------------------------------------------- 1. the Adam tick
def test_adam_tick_from_a_device_rate(g2v):
    import torch
    from g2vec_b200 import _capi
    lib, s = _capi.load(), _stream()
    n = 1000
    a = torch.tensor([1.0, 1.0, 0.0, 0.0], dtype=torch.float32, device="cuda")
    b = a.clone()
    rate = torch.tensor([0.005], dtype=torch.float32, device="cuda")
    ha, hb = torch.empty(n, 3, device="cuda"), torch.empty(n, 3, device="cuda")
    for t in range(n):
        _capi.check(lib.g2v_cbow_adam_tick(a.data_ptr(), 0.005, 0.9, 0.999, s), "g2v_cbow_adam_tick")
        _capi.check(lib.g2v_cbow_adam_tick_lr(b.data_ptr(), rate.data_ptr(), 0.9, 0.999, s), "g2v_cbow_adam_tick_lr")
        ha[t].copy_(a[:3]); hb[t].copy_(b[:3])
    assert torch.equal(ha.view(torch.int32), hb.view(torch.int32))
    # the rate changed between steps: TF1's float32 alpha_t = lr_t sqrt(1 - beta2^t) / (1 - beta1^t), powers untouched
    c = torch.tensor([1.0, 1.0, 0.0, 0.0], dtype=torch.float32, device="cuda")
    rates = [F32(0.005)] * 300 + [F32(0.0005)] * 300 + [F32(3e-5)] * 150 + [F32(0.01)] * 250
    hc = torch.empty(n, dtype=torch.float32, device="cuda")
    for t in range(n):
        if t == 0 or rates[t] != rates[t - 1]:
            rate.fill_(float(rates[t]))
        _capi.check(lib.g2v_cbow_adam_tick_lr(c.data_ptr(), rate.data_ptr(), 0.9, 0.999, s), "g2v_cbow_adam_tick_lr")
        hc[t].copy_(c[2])
    b1p = b2p = F32(1)
    want = np.empty(n, np.float32)
    for t in range(n):
        b1p, b2p = F32(b1p * F32(0.9)), F32(b2p * F32(0.999))
        want[t] = F32(F32(rates[t] * np.sqrt(F32(F32(1) - b2p))) / F32(F32(1) - b1p))
    assert (hc.cpu().numpy().view(np.int32) == want.view(np.int32)).all()


# ---------------------------------------------------------------------------------------- 2. the decision kernel
def _state(K, lr, factor, min_lr, cap):
    import torch
    head = torch.tensor([K, -1, 0, 0, 0, cap, 0, 0], dtype=torch.int64)
    f = torch.zeros(4 + cap + (cap & 1), dtype=torch.float32)
    f[:3] = torch.tensor([lr, factor, min_lr])
    return torch.cat([head, f.view(torch.int64)]).cuda()


def _check_state(st, counts, K, lr, factor, min_lr):
    from g2vec_b200 import cbow
    used, cuts, last = lro.rates(counts, lr, K, factor, min_lr)
    h = st.cpu()
    got_rates, got_cuts = cbow.lr_rates(h)
    assert int(h[4]) == len(counts) and int(h[3]) == len(cuts)
    assert np.array(got_rates, np.float32).view(np.int32).tolist() == np.array(used, np.float32).view(np.int32).tolist()
    assert got_cuts == cuts
    assert h.numpy()[8:].view(np.float32)[0].view(np.int32) == np.float32(last).view(np.int32)


# long plateaus, ties, a floor, counts that improve again; K = 1, 2, 3 and one larger than the run
_COUNTS = [5, 7, 7, 7, 6, 7, 8, 8, 8, 8, 8, 8, 8, 8, 8, 9, 3, 3, 9, 10, 10, 1, 2, 2, 2, 2, 2, 2, 2, 2, 11, 11, 11, 11,
           11, 11, 11, 11, 11, 11, 11, 12]


@pytest.mark.parametrize("K,factor,min_lr", [(1, 0.5, 0.0), (2, 0.1, 0.0), (3, 0.5, 1e-3), (1, 0.3, 4e-3), (100, 0.5, 0.0)])
def test_decision_kernel_on_counts_in_hist_and_acc(g2v, K, factor, min_lr):
    import torch
    from g2vec_b200 import _capi
    lib, s = _capi.load(), _stream()
    n = len(_COUNTS)
    # device-loop form: the count of step k at hist[4k + 2], the steps decided in ctl[1]
    hist = torch.zeros(4 * n, dtype=torch.int64, device="cuda")
    hist[2::4] = torch.tensor(_COUNTS, dtype=torch.int64)
    ctl = torch.zeros(8, dtype=torch.int64, device="cuda")
    st = _state(K, 0.01, factor, min_lr, n)
    k = 0
    for step_to in list(range(1, 20)) + [23, 23, 23, 30, 31, 31] + list(range(32, n + 1)):
        ctl[1] = step_to                         # several steps at once, and calls that decide nothing (a stopped loop)
        _capi.check(lib.g2v_cbow_lr_plateau(st.data_ptr(), hist.data_ptr() + 16, 4, ctl.data_ptr() + 8, s), "plateau")
        k = step_to
    assert k == n
    _check_state(st, _COUNTS, K, 0.01, factor, min_lr)
    # host-driven form: one step per call from acc[2]
    acc = torch.zeros(6, dtype=torch.int64, device="cuda")
    st2 = _state(K, 0.01, factor, min_lr, n)
    for v in _COUNTS:
        acc[2] = v
        _capi.check(lib.g2v_cbow_lr_plateau(st2.data_ptr(), acc.data_ptr() + 16, 0, None, s), "plateau")
    _check_state(st2, _COUNTS, K, 0.01, factor, min_lr)
    # a record shorter than the run: the rule goes on, only the record stops
    st3 = _state(K, 0.01, factor, min_lr, 10)
    for v in _COUNTS:
        acc[2] = v
        _capi.check(lib.g2v_cbow_lr_plateau(st3.data_ptr(), acc.data_ptr() + 16, 0, None, s), "plateau")
    h3 = st3.cpu()
    _, cuts, last = lro.rates(_COUNTS, 0.01, K, factor, min_lr)
    assert int(h3[4]) == n and int(h3[3]) == len(cuts) and h3[8:].view(torch.float32)[0].item() == float(last)


def test_decision_kernel_replayed_from_a_captured_graph(g2v):
    import torch
    from g2vec_b200 import _capi
    lib = _capi.load()
    n = len(_COUNTS)
    hist = torch.zeros(4 * n, dtype=torch.int64, device="cuda")
    hist[2::4] = torch.tensor(_COUNTS, dtype=torch.int64)
    ctl = torch.zeros(8, dtype=torch.int64, device="cuda")
    st = _state(2, 0.005, 0.5, 0.0, n)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            for _ in range(3):                   # three steps per replay, as a loop decides them
                ctl[1:2].add_(1)
                _capi.check(lib.g2v_cbow_lr_plateau(st.data_ptr(), hist.data_ptr() + 16, 4, ctl.data_ptr() + 8,
                                                    side.cuda_stream), "plateau")
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert int(st.cpu()[4]) == 0                 # capture records, it does not execute
    for _ in range(n // 3):
        g.replay()
    torch.cuda.synchronize()
    _check_state(st, _COUNTS[:3 * (n // 3)], 2, 0.005, 0.5, 0.0)


# ------------------------------------------------------------------------ 3. a schedule that never fires changes nothing
_NEVER = dict(lr_patience=10_000, lr_factor=0.5)


def _same_run(g2v, monkeypatch, args, **kw):
    calls = _count_calls(monkeypatch, NEW)
    W0, i0 = g2v.train_cbow(*args, log=None, return_info=True, **kw)
    assert calls == {k: 0 for k in NEW}          # off: neither new entry point runs
    W1, i1 = g2v.train_cbow(*args, log=None, return_info=True, **_NEVER, **kw)
    assert calls["g2v_cbow_lr_plateau"] > 0 and calls["g2v_cbow_adam_tick_lr"] > 0
    assert W1.tobytes() == W0.tobytes()
    assert i1["history"] == i0["history"] and i1["stop_step"] == i0["stop_step"] and i1["best_step"] == i0["best_step"]
    assert i1["lr"] == i0["lr"] == [float(F32(args[5]))] * len(i0["history"])
    assert i1["lr_reductions"] == i0["lr_reductions"] == []
    return i0


@pytest.mark.parametrize("use_graph", [True, False])
@pytest.mark.parametrize("algo", ["rows", "rank1"])
def test_never_firing_schedule_gives_the_same_bits_full_batch(g2v, monkeypatch, algo, use_graph):
    g = helpers.cbow_golden("cbow_ex.npz")
    info = _same_run(g2v, monkeypatch, _args(g), max_epoch=500, seed=g["seed"], algo=algo, use_graph=use_graph,
                     deterministic=algo == "rows")
    assert info["stop_step"] == g["stop_step"]


@pytest.mark.parametrize("optimizer", ["adam", "lazy_adam"])
def test_never_firing_schedule_gives_the_same_bits_reshuffled_minibatch(g2v, monkeypatch, optimizer):
    g = helpers.cbow_golden("cbow_small.npz")
    _same_run(g2v, monkeypatch, _args(g), max_epoch=20, seed=g["seed"], batch=64, reshuffle=True, optimizer=optimizer,
              deterministic=True, patience=3)


# ----------------------------------------------------------------------------------------------- 4. a firing schedule
def _check_firing(g2v, g, lists_of, batch=0, lazy=False, epochs=30, **kw):
    """Train with the schedule; the rates are the rule's on the run's own counts and W_ih is the float64 trainer's fed
    those rates (up to the step whose weights are returned)."""
    W, info = g2v.train_cbow(*_args(g), max_epoch=epochs, seed=g["seed"], W_ih0=g["W0"], W_ho0=g["Wo0"], log=None,
                             return_info=True, batch=batch, **kw)
    counts = lro.val_counts(info)
    used, cuts, _ = lro.rates(counts, g["lr"], kw["lr_patience"], kw["lr_factor"])
    assert info["lr"] == [float(r) for r in used] and info["lr_reductions"] == cuts
    assert cuts, "the schedule never fired"
    n = info["best_step"] + 1
    want, _ = lro.adam64_train(g["rowptr"], g["gene"], g["label"], lists_of(n), g["W0"], g["Wo0"], used[:n],
                               batch=batch, lazy=lazy)
    err = rel_max(W, want)
    print("steps", len(counts), "returned", n, "cuts", cuts, "rel", err)
    assert err < RTOL_VEC
    return info


@pytest.mark.parametrize("K", [1, 2])
@pytest.mark.parametrize("algo,deterministic,keep_best", [("rows", False, False), ("rows", False, True),
                                                          ("rows", True, False), ("rank1", False, False)])
def test_firing_schedule_full_batch(g2v, K, algo, deterministic, keep_best):
    g = helpers.cbow_golden("cbow_ex.npz")
    # keep_best: early stopping whose patience outlasts the run takes the keep-best kernels and returns the best step
    es = dict(early_stop=True, patience=31) if keep_best else dict(early_stop=False)
    info = _check_firing(g2v, g, lambda n: [g["tr"]] * n, algo=algo, deterministic=deterministic, lr_patience=K,
                         lr_factor=0.5, **es)
    assert len(info["history"]) == 30 and info["stop_step"] is None and info["graph"]


@pytest.mark.parametrize("K", [1, 2])
@pytest.mark.parametrize("optimizer,reshuffle", [("lazy_adam", False), ("lazy_adam", True), ("adam", True)])
def test_firing_schedule_minibatch(g2v, K, optimizer, reshuffle):
    g = helpers.cbow_golden("cbow_small.npz")
    lists = (lambda n: reshuffle_oracle.epoch_orders(g["tr"], g["seed"], n)) if reshuffle else (lambda n: [g["tr"]] * n)
    _check_firing(g2v, g, lists, batch=64, lazy=optimizer == "lazy_adam", epochs=12, optimizer=optimizer,
                  reshuffle=reshuffle, deterministic=optimizer == "adam", early_stop=False, lr_patience=K, lr_factor=0.5)


# ----------------------------------------------------------------------------------- 5. early stopping keeps its rule
@pytest.mark.parametrize("use_graph", [True, False])
def test_early_stopping_follows_its_own_rule(g2v, use_graph):
    g = helpers.cbow_golden("cbow_ex.npz")
    kw = dict(seed=g["seed"], deterministic=True, use_graph=use_graph, lr_patience=1, lr_factor=0.5)
    W, info = g2v.train_cbow(*_args(g), max_epoch=500, patience=3, log=None, return_info=True, **kw)
    counts = lro.val_counts(info)
    assert (info["stop_step"], info["best_step"]) == patience_oracle.apply_rule(counts, 3)
    assert info["stop_step"] is not None
    used, cuts, _ = lro.rates(counts, g["lr"], 1, 0.5)
    assert info["lr"] == [float(r) for r in used] and info["lr_reductions"] == cuts and cuts
    want = g2v.train_cbow(*_args(g), max_epoch=info["best_step"] + 1, early_stop=False, log=None, **kw)
    assert W.tobytes() == want.tobytes()


# ------------------------------------------------------------------------------------------------ 6. the command line
def test_command_line(g2v, tmp_path, monkeypatch, capsys):
    from g2vec_b200 import cbow, cli
    ef, cf, nf, _ = helpers.write_ex_tsv(tmp_path)
    seen = []
    train = cbow.train_cbow

    def keep_info(*a, **k):
        W, info = train(*a, return_info=True, **k)
        seen.append(info)
        return W
    monkeypatch.setattr(cbow, "train_cbow", keep_info)
    base = [ef, cf, nf, None, "-r", "2", "-n", "20", "--seed", "3", "--deterministic"]
    files = {}
    for name, extra in (("off", []), ("never", ["--lr-patience", "10000"]),
                        ("fire", ["--lr-patience", "1", "--lr-factor", "0.5", "--patience", "4"])):
        prefix = str(tmp_path / name)
        cli.main([prefix if a is None else a for a in base] + extra)
        out = capsys.readouterr().out
        files[name] = [open(prefix + s, "rb").read() for s in ("_vectors.txt", "_lgroups.txt", "_biomarkers.txt")]
        lines = [l for l in out.splitlines() if "learning rate ->" in l]
        info = seen[-1]
        if name != "fire":
            assert lines == [] and info["lr_reductions"] == []
        else:
            assert info["lr_reductions"], "the schedule never fired"
            assert lines == ["    - Epoch: %03d\tlearning rate -> %g" % (s, info["lr"][s + 1] if s + 1 < len(info["lr"])
                                                                            else info["lr"][s] * 0.5)
                             for s in info["lr_reductions"]]
    assert files["never"] == files["off"]
    assert all(len(f) > 0 for f in files["fire"])


# ----------------------------------------------------------------------------------------------------- 7. N GPUs
def test_several_gpus_hold_the_same_rates_and_match_one(g2v, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    world = min(torch.cuda.device_count(), 4)
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out = str(tmp_path / "mgpu_lr_plateau.npz")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "mgpu_lr_plateau_worker.py"), out]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    z = np.load(out)
    (rowptr, gene, label), _ = helpers.ex_windows(reps=2)
    W0, Wo0 = helpers.init_weights(7523, 128, 0)
    W1, one = g2v.train_cbow(rowptr, gene, label, 7523, 128, 0.005, max_epoch=20, seed=0, W_ih0=W0, W_ho0=Wo0,
                             log=None, return_info=True, early_stop=False, lr_patience=1, lr_factor=0.5)
    for k in ("nvl", "nccl"):
        rates = z[k + "_lr"]                     # [world, steps]: every rank's record
        assert (rates == rates[0]).all(), k
        used, _, _ = lro.rates(z[k + "_val"], 0.005, 1, 0.5)
        assert rates[0].tolist() == [float(r) for r in used], k
        assert rel_max(z[k + "_W"], W1) < RTOL_VEC, k
    assert str(z["exchange"][1]).startswith("nccl")
