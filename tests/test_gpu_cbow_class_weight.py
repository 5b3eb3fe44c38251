"""GPU checks of the class weights of the training loss (DESIGN.md §4.20).

Entry points: each of the ten *_cw entry points with w = (1, 1) gives the bits of its plain form (dO or c on every
route; g_ih, g_ho and the loss on the fixed-order routes; the atomic routes' g_ih / g_ho within the reorder bound);
with dyadic weights (0.25, 4) and with (0.37, 1.9) every output is within the per-element float64 bound of
tests/f64_reference.py weighted by w_y (tests/class_weight_oracle.WeightedStep), for D in {128, 256, 512, 100}, sum
and mean, batch slices, empty windows and one-label lists, the gene-slab route included; bad weights launch nothing.

Trainer: train_cbow(class_weight=...) against the float64 trainer of tests/class_weight_oracle.py in the full-batch
loops (carried graph and eager, rank1) and the mini-batch loops (adam, lazy_adam, reshuffle); deterministic runs
repeat and (1, 1) is bit-identical to no weights; "balanced" from the split; the command line."""
import numpy as np
import pytest

from tests import class_weight_oracle as cwo, f64_reference as f64, helpers, reshuffle_oracle
from tests.test_gpu_cbow_f64 import Problem, assert_within

pytestmark = pytest.mark.gpu
F32 = np.float32
RTOL_VEC = 1e-4
CW_DYADIC, CW_REAL = (0.25, 4.0), (float(F32(0.37)), float(F32(1.9)))


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available()
    from g2vec_b200 import _capi
    p = torch.cuda.get_device_properties(0)
    return {"lib": _capi.load(), "capi": _capi, "sm": p.multi_processor_count}


@pytest.fixture(scope="module")
def g2v():
    import torch
    assert torch.cuda.is_available()
    import g2vec_b200
    return g2vec_b200


def stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def z(*shape, dtype=None):
    import torch
    return torch.zeros(*shape, dtype=dtype or torch.float32, device="cuda")


def bits(t):
    return t.detach().cpu().numpy().tobytes()


def rel_max(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


ROUTES = ["fwdbwd", "fwdbwd_csc", "fwd_do", "fwdbwd_csc_det", "fwd_do_det", "loop_tail", "loop_tail_det",
          "fwdbwd_slabs", "r1_windows", "r1_windows_csc"]
FIXED_ORDER = {"fwdbwd_csc_det", "fwd_do_det", "loop_tail_det", "r1_windows_csc"}


def run(env, P, route, cw, lo=0, n=None):
    """One call of g2v_cbow_<route> (cw None) or its _cw form over list positions [lo, lo + n) of P.win; returns its
    outputs as NumPy: dO (per position, times the scale where the entry point stores it so), c, g_ih, g_ho, loss,
    correct count."""
    import torch
    lib, d = env["lib"], P.d
    n = P.n - lo if n is None else n
    V, D, red = P.V, P.D, 1 if P.reduce == "mean" else 0
    inv_n = float(F32(1) / F32(P.N))
    out = {"dO": z(max(n, 1)), "g_ih": z(V, D), "g_ho": z(D), "c": z(V), "acc": z(6, dtype=torch.int64)}
    acc = out["acc"].data_ptr()
    win_ptr = d["win"].data_ptr() + 4 * lo
    ws = z(max(int(lib.g2v_cbow_det_workspace_bytes(max(n, 1), D)), 4) // 4 + 64)
    common = (d["rowptr"].data_ptr(), d["gene"].data_ptr(), d["label"].data_ptr())
    W, Wo = d["W"].data_ptr(), d["Who"].data_ptr()
    extra = tuple(cw) if cw is not None else ()
    name = "g2v_cbow_" + route + ("_cw" if cw is not None else "")
    fn = getattr(lib, name)
    if route in ("fwdbwd_csc", "fwdbwd_csc_det", "r1_windows_csc"):
        assert lo == 0 and n == P.n                            # the CSC is of the whole list
    if route == "fwdbwd":
        rc = fn(*common, d["win"].data_ptr(), lo, n, inv_n, W, Wo, out["g_ih"].data_ptr(), out["g_ho"].data_ptr(), acc,
                acc + 8, V, D, red, *extra, stream())
    elif route in ("fwdbwd_csc", "fwdbwd_csc_det"):
        args = (*common, win_ptr, n, inv_n, W, Wo, d["cscptr"].data_ptr(), d["pos"].data_ptr(), out["dO"].data_ptr(),
                out["g_ih"].data_ptr(), out["g_ho"].data_ptr(), acc, acc + 8, V, D, red)
        rc = fn(*args, *((ws.data_ptr(), 0) if route.endswith("det") else ()), *extra, stream())
    elif route in ("fwd_do", "fwd_do_det"):
        args = (*common, win_ptr, n, inv_n, W, Wo, out["dO"].data_ptr(), out["g_ho"].data_ptr(), acc, acc + 8, V, D, red)
        rc = fn(*args, *((ws.data_ptr(), 0) if route.endswith("det") else ()), *extra, stream())
    elif route in ("loop_tail", "loop_tail_det"):
        ctl = z(8, dtype=torch.int64)
        env["capi"].check(lib.g2v_cbow_loop_init(ctl.data_ptr(), 10, 1, stream()), "g2v_cbow_loop_init")
        args = (ctl.data_ptr(), *common, win_ptr, n, inv_n, W, Wo, out["dO"].data_ptr(), out["g_ho"].data_ptr(), acc,
                V, D, red)
        rc = fn(*args, *((ws.data_ptr(), 0) if route.endswith("det") else ()), *extra, stream())
        out["ctl"] = ctl
    elif route == "fwdbwd_slabs":
        S = 3
        sws = z(int(lib.g2v_cbow_slab_workspace_bytes(n, D, S)) // 4 + 64)
        env["capi"].check(lib.g2v_cbow_slab_setup(d["rowptr"].data_ptr(), d["gene"].data_ptr(), d["win"].data_ptr(),
                                                  lo, n, V, S, sws.data_ptr(), stream()), "g2v_cbow_slab_setup")
        rc = fn(d["gene"].data_ptr(), d["label"].data_ptr(), d["win"].data_ptr(), lo, n, inv_n, W, Wo,
                out["g_ih"].data_ptr(), out["g_ho"].data_ptr(), acc, acc + 8, V, D, red, S, sws.data_ptr(), *extra,
                stream())
    else:
        s = z(V)
        env["capi"].check(lib.g2v_cbow_r1_prepare(W, Wo, s.data_ptr(), V, D, stream()), "g2v_cbow_r1_prepare")
        if route == "r1_windows":
            rc = fn(*common, d["win"].data_ptr(), lo, n, inv_n, s.data_ptr(), out["c"].data_ptr(), acc, acc + 8, V,
                    red, *extra, stream())
        else:
            rc = fn(*common, win_ptr, n, inv_n, s.data_ptr(), d["cscptr"].data_ptr(), d["pos"].data_ptr(),
                    out["dO"].data_ptr(), out["c"].data_ptr(), acc, acc + 8, V, red, *extra, stream())
    env["capi"].check(rc, name)
    torch.cuda.synchronize()
    a = out["acc"].cpu().numpy()
    slot = 4 if route.startswith("loop_tail") else 0
    res = {k: out[k].cpu().numpy() for k in ("dO", "g_ih", "g_ho", "c")}
    res["dO"] = res["dO"][:n]
    res["loss"] = float(a[slot:slot + 1].view(np.float64)[0])
    res["correct"] = int(a[slot + 1])
    if route.startswith("loop_tail"):
        assert int(out["ctl"].cpu()[6]) == 1                      # the carry is pending
    return res


OUTPUTS = {"fwdbwd": ("g_ih", "g_ho", "loss"), "fwdbwd_csc": ("dO", "g_ih", "g_ho", "loss"),
           "fwd_do": ("dO", "g_ho", "loss"), "fwdbwd_csc_det": ("dO", "g_ih", "g_ho", "loss"),
           "fwd_do_det": ("dO", "g_ho", "loss"), "loop_tail": ("dO", "g_ho", "loss"),
           "loop_tail_det": ("dO", "g_ho", "loss"), "fwdbwd_slabs": ("g_ih", "g_ho", "loss"),
           "r1_windows": ("c", "loss"), "r1_windows_csc": ("dO", "c", "loss")}


def _problem(env, D, reduce, mode="realistic", n_list=3000, V=1001, one_label=None):
    P = Problem(D, V, n_list, mode, reduce, seed=D + (7 if reduce == "mean" else 0), sm=env["sm"])
    if one_label is not None:
        import torch
        P.label[:] = one_label
        P.d["label"] = torch.from_numpy(P.label.astype(np.uint8)).cuda()
    return P


def _expected(env, P, cw, lo=0, n=None):
    n = P.n - lo if n is None else n
    chain = f64.atomic_chain(n, env["sm"]) + f64.det_chain(n) + 64
    return cwo.WeightedStep(P.rowptr, P.gene, P.label, P.win[lo:lo + n], P.N, P.W, P.Who, cw, reduce=P.reduce,
                            chain=chain)


def _check(route, got, r, what):
    """Every output of a weighted call within the weighted float64 bound."""
    for k in OUTPUTS[route]:
        if k == "loss":
            assert abs(got["loss"] - r.loss_terms.sum()) <= r.loss_err, (what, got["loss"], r.loss_terms.sum())
        elif k == "dO":                                         # stored as dO * scale
            assert_within(got["dO"], r.dO * r.s, r.dO_err * r.s + f64.U * np.abs(r.dO * r.s), what + " dO")
        elif k == "c":
            assert_within(got["c"], r.c, r.c_err + 4 * f64.U * np.abs(r.c) + 1e-30, what + " c")
        elif k == "g_ih":
            assert_within(got["g_ih"], r.g_ih(), r.g_ih_err(), what + " g_ih")
        elif k == "g_ho":
            assert_within(got["g_ho"], r.g_ho, r.g_ho_err, what + " g_ho")
    lo_c, hi_c, _ = r.count_band()
    assert lo_c <= got["correct"] <= hi_c, (what, got["correct"], lo_c, hi_c)


# ---------------------------------------------------------------------------------------------- 1. identity
@pytest.mark.parametrize("D,reduce", [(128, "sum"), (512, "mean"), (100, "sum")])
@pytest.mark.parametrize("route", ROUTES)
def test_unit_weights_are_the_plain_entry_point(env, route, D, reduce):
    if route == "fwdbwd_slabs" and D == 100:
        pytest.skip("the gene-slab route has D in {128, 256, 512} only")
    P = _problem(env, D, reduce)
    plain, unit = run(env, P, route, None), run(env, P, route, (1.0, 1.0))
    assert plain["correct"] == unit["correct"]
    # dO per position on every route; c, g_ih, g_ho and the loss where the order is fixed (r1_windows adds c atomically)
    exact = {"dO"} | ({"c", "g_ih", "g_ho", "loss"} if route in FIXED_ORDER else set())
    if route in ("fwdbwd_csc", "fwdbwd_csc_det"):
        exact.add("g_ih")                                       # written once per row from the same dO
    r = _expected(env, P, (1.0, 1.0))
    for k in OUTPUTS[route]:
        if k in exact:
            assert np.asarray(plain[k]).tobytes() == np.asarray(unit[k]).tobytes(), (route, k)
    # the atomic outputs: within the reorder bound of each other
    _check(route, unit, r, route)
    _check(route, plain, r, route)


# ---------------------------------------------------------------------------------------------- 2. accuracy
@pytest.mark.parametrize("D,reduce,mode", [(128, "sum", "dyadic"), (256, "mean", "realistic"), (512, "sum", "realistic"),
                                           (100, "mean", "realistic"), (100, "sum", "dyadic")])
@pytest.mark.parametrize("cw", [CW_DYADIC, CW_REAL], ids=["dyadic-w", "real-w"])
@pytest.mark.parametrize("route", ROUTES)
def test_weighted_entry_points_against_float64(env, route, D, reduce, mode, cw):
    if route == "fwdbwd_slabs" and D == 100:
        pytest.skip("the gene-slab route has D in {128, 256, 512} only")
    P = _problem(env, D, reduce, mode)
    assert (np.diff(P.rowptr)[P.win] == 0).any()                # empty windows in the list
    got = run(env, P, route, cw)
    r = _expected(env, P, cw)
    _check(route, got, r, "%s D=%d %s %s" % (route, D, reduce, cw))
    if cw == CW_DYADIC:                                         # a power-of-two weight scales dO exactly
        plain = run(env, P, route, None)
        if "dO" in OUTPUTS[route]:
            w = np.where(P.label[P.win] != 0, F32(4), F32(0.25))
            assert np.array_equal(got["dO"], plain["dO"] * w)


@pytest.mark.parametrize("route", ["fwdbwd", "r1_windows", "fwd_do", "fwd_do_det", "fwdbwd_slabs"])
def test_batch_slices(env, route):
    P = _problem(env, 128, "sum")
    for lo, n in ((0, 64), (640, 64), (2999, 1), (1000, 1999)):
        got = run(env, P, route, CW_REAL, lo, n)
        _check(route, got, _expected(env, P, CW_REAL, lo, n), "%s [%d, %d)" % (route, lo, lo + n))


@pytest.mark.parametrize("label", [0, 1])
@pytest.mark.parametrize("route", ROUTES)
def test_one_label_lists(env, route, label):
    P = _problem(env, 256, "sum", one_label=label)
    got = run(env, P, route, CW_REAL)
    _check(route, got, _expected(env, P, CW_REAL), "%s label %d" % (route, label))
    # only w_label acts: the result is the unit-weight result times it (to the rounding of one product)
    unit = run(env, P, route, (1.0, 1.0))
    w = CW_REAL[label]
    assert abs(got["loss"] - w * unit["loss"]) <= 1e-5 * abs(w * unit["loss"]) + 1e-12


@pytest.mark.parametrize("bad", [0.0, -1.0, float("inf"), float("nan")])
def test_bad_weights_launch_nothing(env, bad):
    P = _problem(env, 128, "sum", n_list=200)
    for route in ROUTES:
        for cw in ((bad, 1.0), (1.0, bad)):
            l0 = env["capi"].launch_count()
            with pytest.raises(RuntimeError, match="class weights"):
                run(env, P, route, cw)
            assert env["capi"].launch_count() - l0 <= 2, route   # only the setup calls of run() itself


# ------------------------------------------------------------------------------------------ 3. the trainer
def _args(g):
    return (g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"])


@pytest.mark.parametrize("kw", [dict(), dict(use_graph=False), dict(algo="rank1"), dict(algo="rank1", use_graph=False),
                                dict(deterministic=True), dict(batch=64), dict(batch=64, optimizer="lazy_adam"),
                                dict(batch=64, reshuffle=True), dict(batch=64, reshuffle=True, optimizer="lazy_adam")],
                         ids=["carried-graph", "carried-eager", "rank1", "rank1-eager", "deterministic", "adam-b64",
                              "lazy-b64", "adam-b64-reshuffle", "lazy-b64-reshuffle"])
@pytest.mark.parametrize("cw", ["balanced", CW_REAL])
def test_trainer_against_float64(g2v, kw, cw):
    g = helpers.cbow_golden("cbow_small.npz")
    steps = 10
    W, info = g2v.train_cbow(*_args(g), max_epoch=steps, seed=g["seed"], W_ih0=g["W0"], W_ho0=g["Wo0"], log=None,
                             return_info=True, early_stop=False, class_weight=cw, **kw)
    want_cw = cwo.balanced(g["label"][g["tr"]]) if cw == "balanced" else cw
    assert info["class_weight"] == want_cw
    batch = kw.get("batch", 0)
    lists = (reshuffle_oracle.epoch_orders(g["tr"], g["seed"], steps) if kw.get("reshuffle")
             else [g["tr"]] * steps)
    want, want_o = cwo.train64(g["rowptr"], g["gene"], g["label"], lists, g["W0"], g["Wo0"], [g["lr"]] * steps,
                               want_cw, batch=batch, optimizer=kw.get("optimizer", "adam"))
    unweighted, _ = cwo.train64(g["rowptr"], g["gene"], g["label"], lists, g["W0"], g["Wo0"], [g["lr"]] * steps,
                                (1, 1), batch=batch, optimizer=kw.get("optimizer", "adam"))
    err = rel_max(W, want)
    print(kw, cw, "rel", err, "weight effect", rel_max(unweighted, want))
    assert err < RTOL_VEC
    if cw == CW_REAL:
        assert rel_max(unweighted, want) > 10 * RTOL_VEC             # the weights are visible at this bar
    assert rel_max(info["model"].W_ho.cpu().numpy(), want_o) < RTOL_VEC


def test_early_stop_runs_and_keeps_the_validation_rule(g2v):
    """With early stopping the weighted run stops where the oracle's validation counts say it must."""
    g = helpers.cbow_golden("cbow_small.npz")
    W, info = g2v.train_cbow(*_args(g), max_epoch=200, seed=g["seed"], W_ih0=g["W0"], W_ho0=g["Wo0"], log=None,
                             return_info=True, class_weight="balanced", deterministic=True)
    stop = info["stop_step"]
    assert stop is not None
    hist = info["history"]
    n_steps = len(hist)
    # the oracle trainer to the same step, and its validation counts step by step
    counts = []
    for k in range(1, n_steps + 1):                            # a step's counts are taken after its update
        Wk, Wok = cwo.train64(g["rowptr"], g["gene"], g["label"], [g["tr"]] * k, g["W0"], g["Wo0"], [g["lr"]] * k,
                              info["class_weight"])
        X, _ = f64.incidence(g["rowptr"], g["gene"], g["va"], g["V"])
        o = X @ (Wk @ Wok)
        counts.append(int(((o > 0) == (g["label"][g["va"]] != 0)).sum()))
    got = [int(round(h[1] * len(g["va"]))) for h in hist]
    assert all(abs(a - b) <= 2 for a, b in zip(got, counts)), (got, counts)
    want_best, _ = cwo.train64(g["rowptr"], g["gene"], g["label"], [g["tr"]] * (info["best_step"] + 1), g["W0"],
                               g["Wo0"], [g["lr"]] * (info["best_step"] + 1), info["class_weight"])
    assert rel_max(W, want_best) < RTOL_VEC


# ---------------------------------------------------------------------------------------- 4. reproducibility
@pytest.mark.parametrize("kw", [dict(), dict(batch=64, reshuffle=True), dict(batch=64, optimizer="lazy_adam"),
                                dict(algo="rank1")])
def test_deterministic_runs_repeat_and_unit_weights_are_off(g2v, kw):
    g = helpers.cbow_golden("cbow_small.npz")
    det = kw.get("algo") != "rank1"
    runs = []
    for cw in (CW_REAL, CW_REAL, (1, 1), None):
        W, info = g2v.train_cbow(*_args(g), max_epoch=8, seed=g["seed"], log=None, return_info=True,
                                 deterministic=det, early_stop=False, class_weight=cw, **kw)
        runs.append((W.tobytes(), bits(info["model"].W_ho), info["history"]))
    assert runs[0] == runs[1]
    assert runs[2] == runs[3]
    assert runs[0][0] != runs[3][0]


# ----------------------------------------------------------------------------------------- 5. command line
def test_command_line(g2v, tmp_path, capsys):
    from g2vec_b200 import cli
    ef, cf, nf, _ = helpers.write_ex_tsv(tmp_path)
    base = [ef, cf, nf, None, "-r", "2", "-n", "20", "--seed", "3", "--deterministic"]
    files, logs = {}, {}
    for name, extra in (("off", []), ("unit", ["--class-weight", "1,1"]), ("balanced", ["--class-weight", "balanced"])):
        prefix = str(tmp_path / name)
        cli.main([prefix if a is None else a for a in base] + extra)
        logs[name] = capsys.readouterr().out
        files[name] = [open(prefix + s, "rb").read() for s in ("_vectors.txt", "_lgroups.txt", "_biomarkers.txt")]
    assert files["unit"] == files["off"]
    assert "class weights:" not in logs["off"] and "class weights: w0=1 w1=1" in logs["unit"]
    lines = logs["balanced"].splitlines()
    i = next(k for k, ln in enumerate(lines) if "Start training" in ln)
    assert lines[i + 1].strip().startswith("class weights: w0=")
    assert all(len(f) > 0 for f in files["balanced"]) and files["balanced"][0] != files["off"][0]
    # the same writers: the same line structure as the unweighted run's files
    for a, b in zip(files["balanced"], files["off"]):
        la, lb = a.decode().splitlines(), b.decode().splitlines()
        assert len(la) == len(lb) and [len(x.split("\t")) for x in la] == [len(x.split("\t")) for x in lb]
    for bad in ("0,1", "nan,1", "1e40,1", "a,b"):
        with pytest.raises(SystemExit) as e:
            cli.main([str(tmp_path / "bad") if a is None else a for a in base] + ["--class-weight=" + bad])
        assert e.value.code == 2 and "--class-weight" in capsys.readouterr().err


# ------------------------------------------------------------------------------------------ 6. several GPUs
def test_torchrun_ranks_match_one_gpu(tmp_path):
    import os
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mgpu_class_weight_worker.py")
    out = str(tmp_path / "W.npy")
    subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node=2",
                           worker, out], cwd=os.path.dirname(os.path.dirname(worker)))
    g = helpers.cbow_golden("cbow_small.npz")
    import g2vec_b200
    one = g2vec_b200.train_cbow(*_args(g), max_epoch=10, seed=g["seed"], log=None, early_stop=False,
                                class_weight="balanced")
    assert rel_max(np.load(out), one) < 1e-4
