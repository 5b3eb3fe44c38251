"""GPU checks of decoupled weight decay (DESIGN.md §4.18).

Entry points: each *_wd entry point at λ = 0 gives its counterpart's bits with the same launch count; at λ > 0 the
fused decay equals a float32 torch decay W - (λ W) followed by the counterpart at λ = 0, bit for bit (dense, lazy);
rows with g = m = v = 0 end at fl(w - fl(λ w)); lazy leaves untouched rows byte-identical; the multi-GPU exchange on
simulated ranks equals the dense update bit for bit; rank-1 takes g_ho from the pre-decay W_ih, decays rows with
c[g] = 0 under SGD and refreshes s; a CUDA graph replays the eager bits; bad λ is refused with nothing launched.

Trainer: λ = 0 (given or not) makes the same calls and gives the same bits; λ > 0 stays within 1e-4 max|W| of the
float64 AdamW / SGDW / lazy AdamW trainer (tests/weight_decay_oracle.py) in every full-batch and mini-batch loop;
full-batch lazy_adam against adam; reproducibility; the plateau schedule; the command line."""
import numpy as np
import pytest

from tests import helpers, lr_plateau_oracle as lro, reshuffle_oracle, weight_decay_oracle as wdo
from tests.test_gpu_cbow_exchange import Ranks, dyadic_grads, owned, hyper_at

pytestmark = pytest.mark.gpu
F32 = np.float32
LR, B1, B2, EPS = 0.005, 0.9, 0.999, 1e-8
ADAM, SGD = 0, 1
RTOL_VEC = 1e-4
LAM = float(F32(0.01))


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


def bits(t):
    return t.detach().cpu().numpy().tobytes()


def rel_max(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def torch_decay(t, lam):
    """The composed form's decay: a float32 torch W - (λ W), in place."""
    t.copy_(t - (lam * t))


def launches(env, fn):
    """Run fn (which returns a C ABI return code), check it, and return the launches it made."""
    import torch
    l0 = env["capi"].launch_count()
    env["capi"].check(fn(), "call")
    torch.cuda.synchronize()
    return env["capi"].launch_count() - l0


# ------------------------------------------------------------------------------------------------ 1. dense update
DENSE_SHAPES = [(4, 1001), (128, 1001), (129, 999), (512, 257)]     # odd V; 129 * 999 leaves a scalar tail of W_ih
VARIANTS = [("adam_host", ADAM, 3), ("adam_dev", ADAM, 3), ("sgd", SGD, 1)]


class Dense:
    """Buffers of one g2v_cbow_update call (W_ih [V, D], W_ho, m, v, their [D] parts, the gradients)."""

    def __init__(self, V, D, seed, t):
        rs = np.random.RandomState(seed)
        self.V, self.D = V, D
        self.h = {"W": rs.randn(V * D).astype(F32), "Wo": rs.randn(D).astype(F32),
                  "g": (rs.randn(V * D) * 1e-2).astype(F32), "go": (rs.randn(D) * 1e-2).astype(F32)}
        for k, n in (("m", V * D), ("v", V * D), ("mo", D), ("vo", D)):
            self.h[k] = ((rs.randn(n) * 1e-3) if k[0] == "m" else (rs.rand(n) * 1e-6)).astype(F32) if t > 1 \
                else np.zeros(n, F32)
        self.h["g"][::7] = 0
        self.h["g"][-1] = F32(0.25)
        # rows 0, 5, 10, ...: zero gradient and zero moments
        zr = np.zeros((V, D), bool); zr[::5] = True; zr = zr.reshape(-1)
        for k in ("g", "m", "v"):
            self.h[k][zr] = 0
        self.zero_rows = zr

    def device(self):
        return {k: cu(v.copy()) for k, v in self.h.items()}

    def call(self, lib, d, opt, t, hyper, wd=None):
        p = lambda k: d[k].data_ptr() if opt == ADAM else None
        dev = hyper is not None
        args = [d["W"].data_ptr(), d["Wo"].data_ptr(), p("m"), p("v"), p("mo"), p("vo"), d["g"].data_ptr(),
                d["go"].data_ptr(), self.V, self.D, opt, LR, B1, B2, EPS]
        tail = [0 if dev else t, hyper.data_ptr() if dev else None, stream()]
        if wd is None:
            return lib.g2v_cbow_update(*args, *tail)
        return lib.g2v_cbow_update_wd(*args, wd, *tail)


@pytest.mark.parametrize("D,V", DENSE_SHAPES)
def test_update_wd_at_zero_is_the_update(env, D, V):
    P = Dense(V, D, D + V, 3)
    for name, opt, t in VARIANTS:
        hyper = hyper_at(t) if name == "adam_dev" else None
        a, b = P.device(), P.device()
        na = launches(env, lambda: P.call(env["lib"], a, opt, t, hyper))
        nb = launches(env, lambda: P.call(env["lib"], b, opt, t, hyper, wd=0.0))
        assert na == nb == 1
        for k in a:
            assert bits(a[k]) == bits(b[k]), (name, k)
        assert float(b["g"].abs().max()) == 0.0 and float(b["go"].abs().max()) == 0.0


@pytest.mark.parametrize("lam", [LAM, float(F32(0.3))])
@pytest.mark.parametrize("D,V", DENSE_SHAPES)
def test_update_wd_is_decay_then_update_bit_for_bit(env, D, V, lam):
    P = Dense(V, D, 7 * D + V, 3)
    for name, opt, t in VARIANTS:
        hyper = hyper_at(t) if name == "adam_dev" else None
        fused, comp = P.device(), P.device()
        assert launches(env, lambda: P.call(env["lib"], fused, opt, t, hyper, wd=lam)) == 1
        torch_decay(comp["W"], lam)
        torch_decay(comp["Wo"], lam)
        assert bits(comp["W"]) == wdo.decay32(P.h["W"], lam).tobytes()        # torch's decay is the kernels' rule
        launches(env, lambda: P.call(env["lib"], comp, opt, t, hyper))
        for k in fused:
            assert bits(fused[k]) == bits(comp[k]), (name, k)
        # g = m = v = 0: the step adds nothing, the element ends at fl(w - fl(λ w))
        W = fused["W"].cpu().numpy()
        assert W[P.zero_rows].tobytes() == wdo.decay32(P.h["W"][P.zero_rows], lam).tobytes(), name
        assert W[P.zero_rows].tobytes() != P.h["W"][P.zero_rows].tobytes()


# -------------------------------------------------------------------------------------------------- 2. lazy Adam
def _lazy_problem(V, D, seed):
    rs = np.random.RandomState(seed)
    rows = np.sort(rs.choice(V, size=V // 3, replace=False)).astype(np.int32)
    k = rs.randint(1, 5, len(rows))
    segptr = np.zeros(len(rows) + 1, np.int32); segptr[1:] = np.cumsum(k)
    n_b = 200
    pos = rs.randint(0, n_b, int(segptr[-1])).astype(np.int32)
    dO = (rs.randn(n_b) * 1e-2).astype(F32)
    h = {"W": rs.randn(V, D).astype(F32), "m": (rs.randn(V, D) * 1e-3).astype(F32),
         "v": (rs.rand(V, D) * 1e-6).astype(F32), "Wo": rs.randn(D).astype(F32),
         "mo": (rs.randn(D) * 1e-3).astype(F32), "vo": (rs.rand(D) * 1e-6).astype(F32),
         "go": (rs.randn(D) * 1e-2).astype(F32)}
    return rows, segptr, pos, dO, h


def _lazy_call(lib, plan, d, V, D, t, wd=None):
    rows, segptr, pos, dO = plan
    args = [rows.data_ptr(), segptr.data_ptr(), pos.data_ptr(), dO.data_ptr(), rows.shape[0], d["W"].data_ptr(),
            d["m"].data_ptr(), d["v"].data_ptr(), d["Wo"].data_ptr(), d["mo"].data_ptr(), d["vo"].data_ptr(),
            d["go"].data_ptr(), V, D, LR, B1, B2, EPS]
    tail = [t, None, stream()]
    if wd is None:
        return lib.g2v_cbow_lazy_adam(*args, *tail)
    return lib.g2v_cbow_lazy_adam_wd(*args, wd, *tail)


@pytest.mark.parametrize("D", [4, 128, 129])
def test_lazy_adam_wd(env, D):
    V, t = 1001, 2
    rows, segptr, pos, dO, h = _lazy_problem(V, D, D)
    plan = tuple(cu(x) for x in (rows, segptr, pos, dO))
    new = lambda: {k: cu(v.copy()) for k, v in h.items()}
    # λ = 0: the counterpart's bits and launches
    a, b = new(), new()
    na = launches(env, lambda: _lazy_call(env["lib"], plan, a, V, D, t))
    nb = launches(env, lambda: _lazy_call(env["lib"], plan, b, V, D, t, wd=0.0))
    assert na == nb == 2
    assert all(bits(a[k]) == bits(b[k]) for k in a)
    # λ > 0: the rows as "decay the listed rows in torch, then the λ = 0 call", W_ho as "decay W_ho, then the λ = 0
    # call" -- the rows' gradient c * W_ho reads W_ho before the step, so each composition decays one of the two
    import torch
    fused, comp, comp_o = new(), new(), new()
    assert launches(env, lambda: _lazy_call(env["lib"], plan, fused, V, D, t, wd=LAM)) == 2
    ri = plan[0].long()
    comp["W"][ri] = comp["W"][ri] - (LAM * comp["W"][ri])
    torch_decay(comp_o["Wo"], LAM)
    launches(env, lambda: _lazy_call(env["lib"], plan, comp, V, D, t))
    launches(env, lambda: _lazy_call(env["lib"], plan, comp_o, V, D, t))
    for k in ("W", "m", "v"):
        assert bits(fused[k]) == bits(comp[k]), k
    for k in ("Wo", "mo", "vo", "go"):
        assert bits(fused[k]) == bits(comp_o[k]), k
    untouched = np.setdiff1d(np.arange(V), rows)
    for k in ("W", "m", "v"):
        assert fused[k].cpu().numpy()[untouched].tobytes() == h[k][untouched].tobytes(), k
    assert bits(fused["Wo"]) != bits(a["Wo"])                     # W_ho is decayed
    # an empty row list: only W_ho is stepped (and decayed)
    e, f = new(), new()
    empty = (torch.zeros(1, dtype=torch.int32, device="cuda"),) * 3 + (plan[3],)
    call0 = lambda d, wd=None: _lazy_call(env["lib"], (empty[0][:0],) + empty[1:], d, V, D, t, wd)
    assert launches(env, lambda: call0(e, LAM)) == 1
    torch_decay(f["Wo"], LAM)
    launches(env, lambda: call0(f))
    assert all(bits(e[k]) == bits(f[k]) for k in e) and bits(e["W"]) == h["W"].tobytes()


# ------------------------------------------------------------------------------- 3. multi-GPU exchange, simulated
NVL_WORLDS = [1, 2, 3, 5, 8]
NVL_SHAPES = [(1, 1), (2, 1), (4, 1), (6, 1), (1000, 3), (1001, 3), (1000, 33), (999, 33)]


def _nvl_call(lib, R, rank, opt, t, wd, alpha_dev=None):
    adam = opt == ADAM
    args = [R.g_tab.data_ptr(), R.w_tab.data_ptr(), None, None, R.m[rank].data_ptr() if adam else None,
            R.v[rank].data_ptr() if adam else None, R.n, rank, R.world, opt, LR, B1, B2, EPS]
    tail = [t, alpha_dev, stream()]
    if wd is None:
        return lib.g2v_cbow_update_nvl(*args, *tail)
    return lib.g2v_cbow_update_nvl_wd(*args, wd, *tail)


def _dense_flat(env, V, D, W, m, v, g, opt, t, alpha_dev, wd):
    k = 4 * V * D
    p = lambda x, off=0: x.data_ptr() + off if opt == ADAM else None
    env["capi"].check(env["lib"].g2v_cbow_update_wd(W.data_ptr(), W.data_ptr() + k, p(m), p(v), p(m, k), p(v, k),
                                                    g.data_ptr(), g.data_ptr() + k, V, D, opt, LR, B1, B2, EPS, wd, t,
                                                    alpha_dev, stream()), "g2v_cbow_update_wd")


def test_nvl_cases_reach_every_residue_and_idle_ranks():
    ns = [(w, (V + 1) * D) for w in NVL_WORLDS for V, D in NVL_SHAPES]
    assert {n % 4 for _, n in ns} == {0, 1, 2, 3}
    assert any(n // 4 < w for w, n in ns)


@pytest.mark.parametrize("V,D", NVL_SHAPES)
@pytest.mark.parametrize("world", NVL_WORLDS)
def test_update_nvl_wd_is_the_dense_update_bit_for_bit(env, world, V, D):
    import torch
    n = (V + 1) * D
    R = Ranks(world, n)
    rs = np.random.RandomState(n % 100003 * 8 + world + 5)
    W0 = rs.randn(n).astype(F32)
    own = [torch.from_numpy(owned(n, world, r)).cuda() for r in range(world)]
    for kind, t, dev, wd in (("adam", 1, False, LAM), ("adam", 3, False, LAM), ("adam", 2, True, LAM),
                             ("sgd", 1, False, LAM), ("adam", 3, False, 0.0), ("sgd", 1, False, 0.0)):
        what = "%s t=%d dev=%s wd=%g world=%d n=%d" % (kind, t, dev, wd, world, n)
        opt = ADAM if kind == "adam" else SGD
        gs, gsum = dyadic_grads(world, n, rs)
        m0 = (rs.randn(n) * 1e-3).astype(F32) if t > 1 else np.zeros(n, F32)
        v0 = (rs.rand(n) * 1e-6).astype(F32) if t > 1 else np.zeros(n, F32)
        hyper = hyper_at(t) if dev else None
        ad = hyper.data_ptr() if dev else None
        R.load(W0, m0, v0, gs)
        for r in range(world):
            env["capi"].check(_nvl_call(env["lib"], R, r, opt, 0 if dev else t, wd, ad), what)
        W, m, v = cu(W0), cu(m0), cu(v0)
        _dense_flat(env, V, D, W, m, v, cu(gsum), opt, 0 if dev else t, ad, wd)
        for p in range(world):
            assert bits(R.w[p]) == bits(W), what + " weights of rank %d" % p
            assert int((R.g[p] != 0).sum()) == 0, what
            if opt == ADAM:
                assert bits(R.m[p][own[p]]) == bits(m[own[p]]) and bits(R.v[p][own[p]]) == bits(v[own[p]]), what
        if wd == 0.0:                                             # and the counterpart's bits at λ = 0
            R.load(W0, m0, v0, gs)
            for r in range(world):
                env["capi"].check(_nvl_call(env["lib"], R, r, opt, 0 if dev else t, None, ad), what)
            for p in range(world):
                assert bits(R.w[p]) == bits(W), what + " (counterpart)"


# ------------------------------------------------------------------------------------------------------ 4. rank-1
def _r1_call(lib, d, V, D, opt, t, wd=None):
    p = lambda k: d[k].data_ptr() if opt == ADAM else None
    args = [d["W"].data_ptr(), d["Wo"].data_ptr(), p("m"), p("v"), p("mo"), p("vo"), d["c"].data_ptr(),
            d["scratch"].data_ptr(), d["s"].data_ptr(), V, D, opt, 0.5 if opt == SGD else LR, B1, B2, EPS]
    tail = [t, None, stream()]
    if wd is None:
        return lib.g2v_cbow_r1_update(*args, *tail)
    return lib.g2v_cbow_r1_update_wd(*args, wd, *tail)


def _r1_problem(lib, V, D, seed, dyadic=False):
    rs = np.random.RandomState(seed)
    if dyadic:   # every product W_ih[g, d] * c[g] and every sum of them exact in float32 (< 2^24 quanta)
        W = (rs.randint(-63, 64, (V, D)) * 2.0 ** -6).astype(F32)
        Wo = (rs.randint(-63, 64, D) * 2.0 ** -6).astype(F32)
        c = (rs.randint(-63, 64, V) * 2.0 ** -12).astype(F32)
    else:
        W, Wo, c = rs.randn(V, D).astype(F32), rs.randn(D).astype(F32), (rs.randn(V) * 1e-2).astype(F32)
    c[::5] = 0
    h = {"W": W, "Wo": Wo, "c": c, "m": np.zeros((V, D), F32), "v": np.zeros((V, D), F32), "mo": np.zeros(D, F32),
         "vo": np.zeros(D, F32), "s": np.zeros(V, F32),
         "scratch": np.zeros(int(lib.g2v_cbow_r1_scratch_bytes(D)) // 4, F32)}
    return h


@pytest.mark.parametrize("D", [128, 100, 512])
def test_rank1_update_wd(env, D):
    import torch
    lib, V = env["lib"], 1001
    h = _r1_problem(lib, V, D, D)
    new = lambda: {k: cu(v.copy()) for k, v in h.items()}
    for opt in (ADAM, SGD):
        a, b = new(), new()
        na = launches(env, lambda: _r1_call(lib, a, V, D, opt, 1))
        nb = launches(env, lambda: _r1_call(lib, b, V, D, opt, 1, wd=0.0))
        assert na == nb == 3
        assert all(bits(a[k]) == bits(b[k]) for k in a if k != "scratch"), opt
        # λ > 0: W_ih as "decay W_ih, then the λ = 0 call" and W_ho as "decay W_ho, then the λ = 0 call" -- each
        # composition keeps the other matrix at its pre-step value, as the fused step reads it for the gradients
        f = new()
        assert launches(env, lambda: _r1_call(lib, f, V, D, opt, 1, wd=LAM)) == 3
        ci, co = new(), new()
        torch_decay(ci["W"], LAM)
        torch_decay(co["Wo"], LAM)
        launches(env, lambda: _r1_call(lib, ci, V, D, opt, 1))
        launches(env, lambda: _r1_call(lib, co, V, D, opt, 1))
        for k in ("W", "m", "v"):
            assert bits(f[k]) == bits(ci[k]), (opt, k)
        for k in ("Wo", "mo", "vo"):
            assert bits(f[k]) == bits(co[k]), (opt, k)
        assert float(f["c"].abs().max()) == 0.0
        # rows with c[g] = 0 (and zero moments) end at the decay, under SGD too
        zero = np.arange(V)[::5]
        assert f["W"].cpu().numpy()[zero].tobytes() == wdo.decay32(h["W"][zero], LAM).tobytes(), opt
        # s refreshed for the new weights
        s2 = torch.zeros(V, device="cuda")
        env["capi"].check(lib.g2v_cbow_r1_prepare(f["W"].data_ptr(), f["Wo"].data_ptr(), s2.data_ptr(), V, D,
                                                  stream()), "g2v_cbow_r1_prepare")
        assert bits(f["s"]) == bits(s2)


@pytest.mark.parametrize("D", [128, 100])
def test_rank1_g_ho_is_taken_from_the_pre_decay_w_ih(env, D):
    """Dyadic W_ih and c: g_ho = W_ih^T c is exact, lr = 0.5 and λ = 0.25 keep every product exact, so SGD's W_ho is
    fl(0.75 W_ho - 0.5 g_ho) with g_ho from the weights before the step -- and not from the decayed ones."""
    lib, V, lam = env["lib"], 1001, 0.25
    h = _r1_problem(lib, V, D, D + 1, dyadic=True)
    d = {k: cu(v.copy()) for k, v in h.items()}
    launches(env, lambda: _r1_call(lib, d, V, D, SGD, 1, wd=lam))
    W64, c64 = h["W"].astype(np.float64), h["c"].astype(np.float64)
    g_pre, g_post = W64.T @ c64, (W64 * (1 - lam)).T @ c64
    assert (g_pre.astype(F32) == g_pre).all()
    wo = wdo.decay32(h["Wo"], lam).astype(np.float64)
    got = d["Wo"].cpu().numpy()
    assert got.tobytes() == (wo - 0.5 * g_pre).astype(F32).tobytes()
    assert got.tobytes() != (wo - 0.5 * g_post).astype(F32).tobytes()


# ------------------------------------------------------------------------------------ 5. graphs and bad arguments
def test_a_captured_wd_step_replays_the_eager_bits(env):
    import torch
    V, D, t = 999, 129, 3
    P = Dense(V, D, 11, t)
    hyper = hyper_at(t)
    eager, graphed = P.device(), P.device()
    launches(env, lambda: P.call(env["lib"], eager, ADAM, t, hyper, wd=LAM))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            env["capi"].check(P.call(env["lib"], graphed, ADAM, t, hyper, wd=LAM), "capture")
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert bits(graphed["W"]) == P.h["W"].tobytes()          # capture records, it does not execute
    g.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert bits(eager[k]) == bits(graphed[k]), k


@pytest.mark.parametrize("bad", [-1.0, -1e-6, 1.0, 1.5, float("nan"), float("inf"), -float("inf")])
def test_bad_weight_decay_is_refused_with_nothing_launched(env, bad):
    import torch
    lib = env["lib"]
    V, D = 101, 128
    P = Dense(V, D, 1, 1)
    d = P.device()
    rows, segptr, pos, dO, h = _lazy_problem(V, D, 2)
    plan = tuple(cu(x) for x in (rows, segptr, pos, dO))
    ld = {k: cu(v.copy()) for k, v in h.items()}
    R = Ranks(2, (V + 1) * D)
    r1 = {k: cu(v.copy()) for k, v in _r1_problem(lib, V, D, 3).items()}
    before = [bits(x) for x in list(d.values()) + list(ld.values()) + R.w + list(r1.values())]
    calls = {"g2v_cbow_update_wd": lambda: P.call(lib, d, ADAM, 1, None, wd=bad),
             "g2v_cbow_lazy_adam_wd": lambda: _lazy_call(lib, plan, ld, V, D, 1, wd=bad),
             "g2v_cbow_update_nvl_wd": lambda: _nvl_call(lib, R, 0, ADAM, 1, bad),
             "g2v_cbow_r1_update_wd": lambda: _r1_call(lib, r1, V, D, ADAM, 1, wd=bad)}
    for name, fn in calls.items():
        l0 = env["capi"].launch_count()
        assert fn() != 0, name
        assert env["capi"].launch_count() == l0, name
        msg = lib.g2v_last_error().decode()
        assert name in msg and "weight_decay" in msg, msg
    torch.cuda.synchronize()
    assert before == [bits(x) for x in list(d.values()) + list(ld.values()) + R.w + list(r1.values())]


# ------------------------------------------------------------------------------------------ 6. off by default
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


# (golden, keyword arguments, bit-reproducible); the gene-slab table is cbow_ex with 3 slabs forced.  Early stopping is
# off, or (keep-best) on with a patience longer than the run, so that runs with float atomics make the same calls.
OFF_CONFIGS = [
    ("cbow_ex.npz", dict(), False),
    ("cbow_ex.npz", dict(use_graph=False), False),
    ("cbow_ex.npz", dict(early_stop=True, patience=13), False),
    ("cbow_ex.npz", dict(deterministic=True), True),
    ("cbow_ex.npz", dict(deterministic=True, use_graph=False, early_stop=True, patience=13), True),
    ("cbow_ex.npz", dict(slabs=True), False),
    ("cbow_ex.npz", dict(algo="rank1"), True),
    ("cbow_ex.npz", dict(algo="rank1", optimizer="sgd", use_graph=False), True),
    ("cbow_small.npz", dict(batch=64), False),
    ("cbow_small.npz", dict(batch=64, reshuffle=True, optimizer="sgd"), False),
    ("cbow_small.npz", dict(batch=64, optimizer="lazy_adam"), False),
    ("cbow_small.npz", dict(batch=64, reshuffle=True, optimizer="lazy_adam", deterministic=True), True),
    ("cbow_small.npz", dict(batch=64, reshuffle=True, deterministic=True), True),
    ("cbow_small.npz", dict(batch=64, optimizer="sgd", deterministic=True), True),
]


@pytest.mark.parametrize("golden,kw,exact", OFF_CONFIGS)
def test_zero_weight_decay_changes_nothing(g2v, monkeypatch, golden, kw, exact):
    from g2vec_b200 import _capi
    kw = dict(kw)
    slabs = kw.pop("slabs", False)
    if slabs:
        monkeypatch.setenv("G2V_CBOW_SLABS", "3")
    kw.setdefault("early_stop", False)
    g = helpers.cbow_golden(golden)
    seen = _record_calls(monkeypatch)
    runs = []
    for extra in ({}, {"weight_decay": 0.0}, {"weight_decay": 0}):
        del seen[:]
        l0 = _capi.launch_count()
        W, info = g2v.train_cbow(*_args(g), max_epoch=12, seed=g["seed"], log=None, return_info=True, **kw, **extra)
        runs.append((W, info, _capi.launch_count() - l0, list(seen)))
    if slabs:
        assert runs[0][1]["model"]._n_slabs == 3
    W0, i0, n0, s0 = runs[0]
    assert not any(name.endswith("_wd") for name in s0)
    for W, info, n, s in runs[1:]:
        assert n == n0 and s == s0 and info["stop_step"] is None
        assert info["model"].wd == 0.0
        if exact:
            assert W.tobytes() == W0.tobytes() and info["history"] == i0["history"]
            assert info["best_step"] == i0["best_step"]
        else:                                                     # float atomics: the same calls, near-equal weights
            assert rel_max(W, W0) < 1e-5


# ---------------------------------------------------------------------------------- 7. against the float64 trainer
def _check64(g2v, g, lists_of, epochs=12, batch=0, optimizer="adam", rates=None, **kw):
    W, info = g2v.train_cbow(*_args(g), max_epoch=epochs, seed=g["seed"], W_ih0=g["W0"], W_ho0=g["Wo0"], log=None,
                             return_info=True, batch=batch, optimizer=optimizer, weight_decay=LAM, **kw)
    n = info["best_step"] + 1 if info["best_step"] is not None else epochs
    used = rates if rates is not None else [g["lr"]] * n
    want, want_o = wdo.train64(g["rowptr"], g["gene"], g["label"], lists_of(n), g["W0"], g["Wo0"], used[:n],
                               weight_decay=LAM, batch=batch, optimizer=optimizer)
    err = rel_max(W, want)
    nodecay, _ = wdo.train64(g["rowptr"], g["gene"], g["label"], lists_of(n), g["W0"], g["Wo0"], used[:n],
                             weight_decay=0.0, batch=batch, optimizer=optimizer)
    print("steps", len(info["history"]), "returned", n, "rel", err, "decay effect", rel_max(nodecay, want))
    assert err < RTOL_VEC
    assert rel_max(nodecay, want) > 10 * RTOL_VEC                  # the decay is visible at this bar
    if n == epochs:
        assert rel_max(info["model"].W_ho.cpu().numpy(), want_o) < RTOL_VEC
    return info


@pytest.mark.parametrize("kw", [dict(), dict(use_graph=False), dict(early_stop=True, patience=13),
                                dict(deterministic=True), dict(slabs=True), dict(algo="rank1"),
                                dict(algo="rank1", use_graph=False)],
                         ids=["carried-graph", "carried-eager", "keep-best", "deterministic", "slabs", "rank1",
                              "rank1-eager"])
def test_full_batch_against_float64(g2v, monkeypatch, kw):
    kw = dict(kw)
    slabs = kw.pop("slabs", False)
    if slabs:
        monkeypatch.setenv("G2V_CBOW_SLABS", "3")
    kw.setdefault("early_stop", False)
    g = helpers.cbow_golden("cbow_ex.npz")
    info = _check64(g2v, g, lambda n: [g["tr"]] * n, **kw)
    assert len(info["history"]) == 12 and info["stop_step"] is None
    assert info["graph"] == kw.get("use_graph", True)
    if slabs:
        assert info["model"]._n_slabs == 3 and info["model"].prepared(info["windows"][0]).slabs


@pytest.mark.parametrize("reshuffle", [False, True])
@pytest.mark.parametrize("optimizer", ["adam", "sgd", "lazy_adam"])
def test_minibatch_against_float64(g2v, optimizer, reshuffle):
    g = helpers.cbow_golden("cbow_small.npz")
    lists = (lambda n: reshuffle_oracle.epoch_orders(g["tr"], g["seed"], n)) if reshuffle else (lambda n: [g["tr"]] * n)
    _check64(g2v, g, lists, batch=64, optimizer=optimizer, reshuffle=reshuffle, early_stop=False)


# ------------------------------------------------------------------------------- 8. full-batch lazy_adam vs adam
def test_full_batch_lazy_adam_against_adam(g2v):
    g = helpers.cbow_golden("cbow_ex.npz")
    kw = dict(seed=g["seed"], W_ih0=g["W0"], W_ho0=g["Wo0"], log=None, early_stop=False, weight_decay=LAM)
    rp, ge = np.asarray(g["rowptr"], np.int64), np.asarray(g["gene"])
    in_list = np.zeros(g["V"], bool)
    for w in g["tr"]:
        in_list[ge[rp[w]:rp[w + 1]]] = True
    out = ~in_list
    assert out.any() and in_list.any()
    # one step from zero moments: the rows in the list are the same bits (DESIGN.md §4.11)
    a1 = g2v.train_cbow(*_args(g), max_epoch=1, optimizer="adam", **kw)
    l1 = g2v.train_cbow(*_args(g), max_epoch=1, optimizer="lazy_adam", **kw)
    assert a1[in_list].tobytes() == l1[in_list].tobytes()
    # a run: rows in the list within the float64 bar; rows outside: the iterated decay under adam, untouched under lazy
    steps = 12
    a = g2v.train_cbow(*_args(g), max_epoch=steps, optimizer="adam", **kw)
    lz = g2v.train_cbow(*_args(g), max_epoch=steps, optimizer="lazy_adam", **kw)
    want, _ = wdo.train64(g["rowptr"], g["gene"], g["label"], [g["tr"]] * steps, g["W0"], g["Wo0"], [g["lr"]] * steps,
                          weight_decay=LAM)
    assert rel_max(a[in_list], want[in_list]) < RTOL_VEC and rel_max(lz[in_list], want[in_list]) < RTOL_VEC
    assert a[out].tobytes() == wdo.decay32(g["W0"][out], LAM, steps).tobytes()
    assert lz[out].tobytes() == g["W0"][out].tobytes()


# ------------------------------------------------------------------------------------------ 9. reproducibility
def test_deterministic_runs_repeat_bit_for_bit_on_any_grid(g2v, monkeypatch):
    from g2vec_b200 import cbow
    g = helpers.cbow_golden("cbow_small.npz")
    real = cbow.CbowModel._launch
    grid = {"max_ctas": 0}

    def launch(self, name, *a):                 # the fixed-order kernels take max_ctas as their last argument
        if name.endswith("_det") or name == "g2v_cbow_batch_expand":
            a = a[:-1] + (grid["max_ctas"],)
        return real(self, name, *a)
    monkeypatch.setattr(cbow.CbowModel, "_launch", launch)
    for kw in (dict(), dict(batch=64, reshuffle=True), dict(batch=64, optimizer="lazy_adam", reshuffle=True)):
        outs = []
        for max_ctas in (0, 0, 3):
            grid["max_ctas"] = max_ctas
            W, info = g2v.train_cbow(*_args(g), max_epoch=8, seed=g["seed"], log=None, return_info=True,
                                     deterministic=True, early_stop=False, weight_decay=LAM, **kw)
            outs.append((W.tobytes(), bits(info["model"].W_ho), info["history"]))
        assert outs[0] == outs[1] == outs[2], kw


# ------------------------------------------------------------------------------------------ 10. with lr_patience
@pytest.mark.parametrize("batch,optimizer", [(0, "adam"), (64, "lazy_adam")])
def test_with_the_plateau_schedule(g2v, batch, optimizer):
    g = helpers.cbow_golden("cbow_ex.npz" if batch == 0 else "cbow_small.npz")
    epochs = 30 if batch == 0 else 12
    W, info = g2v.train_cbow(*_args(g), max_epoch=epochs, seed=g["seed"], W_ih0=g["W0"], W_ho0=g["Wo0"], log=None,
                             return_info=True, batch=batch, optimizer=optimizer, early_stop=False, lr_patience=1,
                             lr_factor=0.5, weight_decay=LAM)
    used, cuts, _ = lro.rates(lro.val_counts(info), g["lr"], 1, 0.5)
    assert info["lr"] == [float(r) for r in used] and info["lr_reductions"] == cuts and cuts
    assert info["model"].wd == LAM                                  # λ stays what it was
    want, _ = wdo.train64(g["rowptr"], g["gene"], g["label"], [g["tr"]] * epochs, g["W0"], g["Wo0"], used,
                          weight_decay=LAM, batch=batch, optimizer=optimizer)
    assert rel_max(W, want) < RTOL_VEC


# ----------------------------------------------------------------------------------------------- 11. command line
def test_command_line(g2v, tmp_path, capsys):
    from g2vec_b200 import cli
    ef, cf, nf, _ = helpers.write_ex_tsv(tmp_path)
    base = [ef, cf, nf, None, "-r", "2", "-n", "20", "--seed", "3", "--deterministic"]
    files = {}
    for name, extra in (("off", []), ("zero", ["--weight-decay", "0"]), ("decay", ["--weight-decay", "0.01"])):
        prefix = str(tmp_path / name)
        cli.main([prefix if a is None else a for a in base] + extra)
        capsys.readouterr()
        files[name] = [open(prefix + s, "rb").read() for s in ("_vectors.txt", "_lgroups.txt", "_biomarkers.txt")]
    assert files["zero"] == files["off"]
    assert all(len(f) > 0 for f in files["decay"]) and files["decay"][0] != files["off"][0]
    for bad in ("-1", "1", "nan", "inf"):
        with pytest.raises(SystemExit) as e:
            cli.main([str(tmp_path / "bad") if a is None else a for a in base] + ["--weight-decay", bad])
        assert e.value.code == 2 and "--weight-decay" in capsys.readouterr().err
