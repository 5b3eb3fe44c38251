"""GPU checks of early stopping with patience (DESIGN.md §4.15): the default rule keeps its launches and results; the
keep-best kernels forced onto patience 1 give the default path's bits; patience runs agree with the CPU restatement
(tests/patience_oracle.py); the returned vectors are the best step's, bit for bit, in every loop; a run that reaches
max_epoch returns the best step's weights; the command line; N GPUs against one."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from tests import helpers, patience_oracle

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL_VEC = 1e-4
NEW = ("g2v_cbow_loop_decide_best", "g2v_cbow_loop_keep_best")
OLD = ("g2v_cbow_loop_decide", "g2v_cbow_loop_begin")


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


@pytest.mark.parametrize("use_graph", [True, False])
def test_default_rule_makes_the_same_launches_and_returns_the_golden_result(g2v, monkeypatch, use_graph):
    from g2vec_b200 import _capi
    calls = _count_calls(monkeypatch, NEW + OLD)
    g = helpers.cbow_golden("cbow_small.npz")
    runs = []
    for kw in ({}, {"patience": 1}):
        for k in calls:
            calls[k] = 0
        l0 = _capi.launch_count()
        W, info = g2v.train_cbow(*_args(g), max_epoch=500, seed=g["seed"], log=None, return_info=True,
                                 deterministic=True, use_graph=use_graph, **kw)
        n_launch = _capi.launch_count() - l0                 # with graphs: the eager step and the captures
        assert info["stop_step"] == g["stop_step"] and info["best_step"] == g["stop_step"] - 1
        assert rel_max(W, g["W_ref"]) < RTOL_VEC
        assert calls["g2v_cbow_loop_decide_best"] == calls["g2v_cbow_loop_keep_best"] == 0
        assert calls["g2v_cbow_loop_decide"] == calls["g2v_cbow_loop_begin"] > 0
        if not use_graph:                 # eager: step 0, then whole chunks of 5 (the steps after the stop are no-ops)
            assert calls["g2v_cbow_loop_decide"] == 1 + 5 * -(-g["stop_step"] // 5)
        runs.append((W, info["history"], n_launch, calls["g2v_cbow_loop_decide"]))
    assert runs[0][0].tobytes() == runs[1][0].tobytes() and runs[0][1] == runs[1][1]
    assert runs[0][2] == runs[1][2] and runs[0][3] == runs[1][3]       # the same launches, step for step


@pytest.mark.parametrize("use_graph", [True, False])
def test_keep_best_kernels_at_patience_one_equal_the_default_path_bit_for_bit(g2v, monkeypatch, use_graph):
    from g2vec_b200 import cbow
    g = helpers.cbow_golden("cbow_ex.npz")
    kw = dict(max_epoch=500, seed=g["seed"], log=None, return_info=True, deterministic=True, use_graph=use_graph)
    W0, i0 = g2v.train_cbow(*_args(g), **kw)
    calls = _count_calls(monkeypatch, NEW + OLD)
    monkeypatch.setattr(cbow.DeviceLoop, "keep_best_from", 1)
    W1, i1 = g2v.train_cbow(*_args(g), patience=1, **kw)
    assert calls["g2v_cbow_loop_decide"] == 0
    assert calls["g2v_cbow_loop_decide_best"] == calls["g2v_cbow_loop_keep_best"] == calls["g2v_cbow_loop_begin"] > 0
    assert i1["stop_step"] == i0["stop_step"] == g["stop_step"]
    assert i1["best_step"] == i0["best_step"] == g["stop_step"] - 1
    assert i1["history"] == i0["history"]
    assert W1.tobytes() == W0.tobytes()


_oracle_runs = {}


def _oracle(name, patience):
    key = (name, patience)
    if key not in _oracle_runs:
        g = helpers.cbow_golden(name)
        _oracle_runs[key] = patience_oracle.cbow_train(g["rowptr"], g["gene"], g["label"], g["tr"], g["va"], g["W0"],
                                                       g["Wo0"], g["lr"], max_steps=500, patience=patience)
    return _oracle_runs[key]


@pytest.mark.parametrize("name,patience,stop,best", [("cbow_ex.npz", 5, 23, 18), ("cbow_small.npz", 10, 53, 43)])
@pytest.mark.parametrize("algo,use_graph", [("rows", True), ("rows", False), ("rank1", True)])
def test_patience_runs_match_the_oracle(g2v, name, patience, stop, best, algo, use_graph):
    g = helpers.cbow_golden(name)
    W_o, hist_o, stop_o, best_o = _oracle(name, patience)
    assert (stop_o, best_o) == (stop, best)
    lines = []
    W, info = g2v.train_cbow(*_args(g), max_epoch=500, seed=g["seed"], log=lines.append, return_info=True, algo=algo,
                             use_graph=use_graph, patience=patience)
    assert (info["stop_step"], info["best_step"]) == (stop, best)
    assert len(info["history"]) == len(hist_o)
    n_va, n_tr = len(g["va"]), len(g["tr"])
    for (s, av, at), (so, avo, ato) in zip(info["history"], hist_o):
        assert s == so and abs(av - avo) <= 2.0 / n_va + 1e-7
        assert (at is None and s == stop) or abs(at - ato) <= 2.0 / n_tr + 1e-7   # rank1: no ACC[tr] at the stop
    assert rel_max(W, W_o) < RTOL_VEC
    assert lines[-2].startswith("    - Epoch(stop): %03d\tACC[val]=%.4f\tACC[tr]=%.4f"
                                % (best, info["history"][best][1], info["history"][best][2]))


def _best_is_best(g2v, args, patience, max_epoch, **kw):
    """A patience run's vectors == W_ih of a run without early stopping over best_step + 1 steps, bit for bit."""
    W, info = g2v.train_cbow(*args, max_epoch=max_epoch, patience=patience, return_info=True, log=None, **kw)
    best = info["best_step"]
    want = g2v.train_cbow(*args, max_epoch=best + 1, early_stop=False, log=None, **kw)
    assert W.tobytes() == want.tobytes(), (info["stop_step"], best)
    # best_step is the last step with the highest validation count up to where the run ended
    n = np.array([h[1] for h in info["history"]])
    assert best == len(n) - 1 - int(np.argmax(n[::-1]))
    if info["stop_step"] is not None:
        assert info["stop_step"] == best + patience == len(n) - 1
    return info


@pytest.mark.parametrize("use_graph", [True, False])
@pytest.mark.parametrize("algo", ["rows", "rank1"])
def test_full_batch_result_is_the_best_step_bit_for_bit(g2v, algo, use_graph):
    # cbow_small, patience 10: stop 53 in the graph chunk of steps 51..55, best 43 in the chunk 41..45
    g = helpers.cbow_golden("cbow_small.npz")
    kw = dict(seed=g["seed"], use_graph=use_graph, algo=algo, deterministic=algo == "rows")
    info = _best_is_best(g2v, _args(g), 10, 500, **kw)
    assert (info["stop_step"], info["best_step"]) == (53, 43)
    ex = helpers.cbow_golden("cbow_ex.npz")
    info = _best_is_best(g2v, _args(ex), 5, 500, **dict(kw, seed=ex["seed"]))
    assert (info["stop_step"], info["best_step"]) == (23, 18)


@pytest.mark.parametrize("optimizer", ["adam", "lazy_adam"])
def test_reshuffled_minibatch_result_is_the_best_epoch_bit_for_bit(g2v, optimizer):
    g = helpers.cbow_golden("cbow_small.npz")
    for patience in (2, 4):
        info = _best_is_best(g2v, _args(g), patience, 40, seed=g["seed"], batch=64, reshuffle=True,
                             optimizer=optimizer, deterministic=True)
        print(optimizer, patience, "stop", info["stop_step"], "best", info["best_step"])


def test_a_run_that_reaches_max_epoch_returns_the_best_step(g2v):
    g = helpers.cbow_golden("cbow_ex.npz")
    kw = dict(seed=g["seed"], deterministic=True)
    # patience 10, 25 steps: best 18, steps 19..24 below it when the run ends
    lines = []
    W, info = g2v.train_cbow(*_args(g), max_epoch=25, patience=10, log=lines.append, return_info=True, **kw)
    assert info["stop_step"] is None and info["best_step"] == 18
    want = g2v.train_cbow(*_args(g), max_epoch=19, early_stop=False, log=None, **kw)
    last = g2v.train_cbow(*_args(g), max_epoch=25, early_stop=False, log=None, **kw)
    assert W.tobytes() == want.tobytes() and W.tobytes() != last.tobytes()
    h = info["history"][18]
    assert lines[-2] == "    - Epoch(best): 018\tACC[val]=%.4f\tACC[tr]=%.4f" % (h[1], h[2])
    # 11 steps: every step improves, the last one (in the second graph chunk) sets `stopped` and is the best
    lines = []
    W, info = g2v.train_cbow(*_args(g), max_epoch=11, patience=10, log=lines.append, return_info=True, **kw)
    assert info["stop_step"] is None and info["best_step"] == 10 and info["graph"]
    want = g2v.train_cbow(*_args(g), max_epoch=11, early_stop=False, log=None, **kw)
    assert W.tobytes() == want.tobytes()
    assert not any("Epoch(best)" in l or "Epoch(stop)" in l for l in lines)


def test_command_line_patience_writes_the_best_epochs_vectors(g2v, tmp_path, monkeypatch, capsys):
    from g2vec_b200 import cbow, cli
    ef, cf, nf, _ = helpers.write_ex_tsv(tmp_path)
    seen = {}
    train = cbow.train_cbow

    def keep_info(*a, **k):
        W, seen["info"] = train(*a, return_info=True, **k)
        return W
    monkeypatch.setattr(cbow, "train_cbow", keep_info)
    prefix = str(tmp_path / "pat")
    cli.main([ef, cf, nf, prefix, "-r", "2", "-n", "20", "--seed", "3", "--patience", "5"])
    out = capsys.readouterr().out
    for s in ("_vectors.txt", "_lgroups.txt", "_biomarkers.txt"):
        assert os.path.getsize(prefix + s) > 0
    info = seen["info"]
    assert info["stop_step"] is not None and info["stop_step"] == info["best_step"] + 5
    h = info["history"][info["best_step"]]
    assert "    - Epoch(stop): %03d\tACC[val]=%.4f\tACC[tr]=%.4f" % h in out
    assert "Namespace(" in out and "patience=5" in out


def test_several_gpus_stop_and_keep_the_same_steps_as_one(g2v, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    world = min(torch.cuda.device_count(), 4)
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out = str(tmp_path / "mgpu_patience.npz")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "mgpu_patience_worker.py"), out]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    z = np.load(out)
    (rowptr, gene, label), _ = helpers.ex_windows(reps=2)
    W0, Wo0 = helpers.init_weights(7523, 128, 0)
    W1, one = g2v.train_cbow(rowptr, gene, label, 7523, 128, 0.005, max_epoch=60, seed=0, W_ih0=W0, W_ho0=Wo0,
                             log=None, return_info=True, patience=5)
    for k in ("nvl", "nccl"):
        assert (int(z[k + "_stop"]), int(z[k + "_best"])) == (one["stop_step"] if one["stop_step"] is not None else -1,
                                                              one["best_step"]), k
        assert rel_max(z[k + "_W"], W1) < RTOL_VEC, k
    assert str(z["exchange"][1]).startswith("nccl")
