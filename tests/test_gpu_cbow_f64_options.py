"""Class weights (DESIGN.md §4.20) and decoupled weight decay (§4.18) at every hidden-size branch of the kernels,
against float64 and against their plain forms.

The weighted rows kernels (cbow_rows_kernel<VEC, *, true>, cbow_rows_generic_kernel<true, true>,
cbow_rows_det_kernel<VEC, true>, cbow_rows_generic_det_kernel<true>) and the decayed optimizer kernels
(cbow_update_kernel<OPT, true>, cbow_lazy_adam_rows_kernel<true>, r1_update_kernel<VEC, OPT, true>,
r1_update_ho_kernel<OPT, true>) are instantiations of their own, each with its own launch set-up: the opt-in shared
memory above 48 KB, the size check, the scalar tails, the W_ho grid.  They run here at the shapes of
tests/test_gpu_cbow_f64.py, which reach every branch (tests/test_option_shapes_host.py restates the dispatch and checks
that these lists reach it):
  class weights  every *_cw route at every CASES shape and D = 132, dyadic and realistic, sum and mean, weights
                 (0.25, 4) and (0.37, 1.9): every output within the weighted float64 bound, the count exact in
                 dyadic mode; with power-of-two weights dO is the plain dO times w_y bit for bit; (1, 1) gives the
                 plain bits; the
                 fixed-order forms give the same bits on one CTA as on the full grid, and above their shared-memory
                 limit they are refused with the sizeHiddenlayer message and launch nothing;
  loop tail      g2v_cbow_loop_tail(_det), plain and _cw, gives the dO (and, fixed-order, g_ho and loss) bits of
                 g2v_cbow_fwd_do(_det), its loss and count land in acc[4] and acc[5], and ctl[6] is set;
  largest D      the weighted generic kernels run at the largest admitted D within the bound; D + 1 is refused and
                 leaves no CUDA error behind;
  dense decay    g2v_cbow_update_wd equals a float32 torch decay followed by g2v_cbow_update bit for bit, and lies
                 within the float64 Adam / SGD bound of the decayed weights, at V*D % 4 in {0, 1, 2, 3};
  lazy decay     g2v_cbow_lazy_adam_wd on a Problem's own rows equals "decay, then the λ = 0 call" bit for bit, the
                 W_ho step over one and over several 256-thread blocks, untouched rows byte-identical;
  rank-1 decay   g2v_cbow_r1_update_wd on every VEC path and on both sides of its opt-in shared memory: the
                 composition's bits, g_ho from the pre-decay W_ih, rows with c = 0 decayed, s refreshed, and W_ih and
                 W_ho within the float64 Adam / SGD bound of the decayed weights (dyadic c: the gradient is exact)."""
import numpy as np
import pytest

from tests import class_weight_oracle as cwo, f64_reference as f64, weight_decay_oracle as wdo
from tests.test_gpu_cbow_class_weight import CW_DYADIC, CW_REAL, FIXED_ORDER, OUTPUTS, run, _check
from tests.test_gpu_cbow_exchange import hyper_at
from tests.test_gpu_cbow_f64 import (CASES, UPDATE_SHAPES, assert_within, check_forward, det_max_d, generic_max_d,
                                     make_windows, problem)
from tests.test_gpu_cbow_weight_decay import ADAM, LAM, LR, SGD, Dense, _lazy_call, _r1_call, _r1_problem, bits, \
    launches, torch_decay

pytestmark = pytest.mark.gpu
F32 = np.float32

# every class-weighted route but the gene slabs, whose ABI admits D in {128, 256, 512} only
CW_ROUTES = ["fwdbwd", "fwdbwd_csc", "fwd_do", "fwdbwd_csc_det", "fwd_do_det", "loop_tail", "loop_tail_det",
             "r1_windows", "r1_windows_csc"]
DET_ROUTES = ["fwdbwd_csc_det", "fwd_do_det", "loop_tail_det"]
MODES = [("dyadic", "sum"), ("realistic", "sum"), ("dyadic", "mean"), ("realistic", "mean")]
# the dense update: UPDATE_SHAPES plus D = 256 and D = 1537; V*D % 4 takes 0, 1, 2 and 3
DENSE_WD_SHAPES = UPDATE_SHAPES + [(256, 1001), (1537, 1001)]
DENSE_T = [1, 2, 1000]
DENSE_LAMS = [LAM, float(F32(0.3))]
# rank-1: VEC 0 at D % 4 != 0 and == 0, VEC 1, 2, 4, and VEC 0 on both sides of D = 1536 (48 KB of shared memory)
R1_DS = [1, 3, 33, 128, 129, 256, 512, 513, 1000, 1536, 1537, "max"]
R1_V = 1001
R1_OPTS = [ADAM, SGD]
DENSE_VARIANTS = [("adam_host", ADAM), ("adam_dev", ADAM), ("sgd", SGD)]
# CASES, plus a D % 4 == 0 that is not a VEC size and needs no opt-in shared memory
CW_CASES = CASES + [(132, 1001, 700)]


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available()
    from g2vec_b200 import _capi
    p = torch.cuda.get_device_properties(0)
    return {"lib": _capi.load(), "capi": _capi, "sm": p.multi_processor_count,
            "optin": p.shared_memory_per_block_optin}


def _memo(r):
    """Compute a reference's g_ih and its bound once (each is a [V, D] float64 array)."""
    g, e = r.g_ih(), r.g_ih_err()
    r.g_ih, r.g_ih_err = (lambda: g), (lambda: e)
    return r


def weighted_ref(env, P, cw):
    """The WeightedStep of the whole list of P, kept on P (tests/test_gpu_cbow_f64 keeps one Problem at a time)."""
    refs = P.__dict__.setdefault("weighted_refs", {})
    if cw not in refs:
        chain = f64.atomic_chain(P.n, env["sm"]) + f64.det_chain(P.n) + 64
        refs[cw] = _memo(cwo.WeightedStep(P.rowptr, P.gene, P.label, P.win, P.N, P.W, P.Who, cw, reduce=P.reduce,
                                          chain=chain))
    return refs[cw]


def plain_ref(P):
    if not P.__dict__.get("plain_memo"):
        _memo(P.ref)
        P.plain_memo = True
    return P.ref


def det_refused(env, D):
    return D > det_max_d(env["optin"]) and D not in (128, 256, 512)


def assert_refused(env, P, route, cw):
    """The fixed-order route is refused before anything is launched, and leaves no CUDA error behind."""
    import torch
    l0 = env["capi"].launch_count()
    with pytest.raises(RuntimeError, match="sizeHiddenlayer"):
        run(env, P, route, cw)
    assert env["capi"].launch_count() == l0, route
    torch.cuda.synchronize()
    assert torch.cuda.current_stream().query()


def same_bits(a, b, keys, what):
    for k in keys:
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), (what, k)


def check_loop_tail(tail, fwd, det, what):
    """A tail pass is its forward: dO bit for bit (and g_ho, loss for the fixed-order one), the same count; its loss
    and count in acc[4] and acc[5], acc[3] carrying the count, acc[0..2] untouched."""
    same_bits(tail, fwd, ("dO", "g_ho", "loss") if det else ("dO",), what)
    assert tail["correct"] == fwd["correct"], what
    a = tail["acc"]
    assert a[0] == a[1] == a[2] == 0 and a[3] == a[5] == fwd["correct"], (what, a)


# --------------------------------------------------------------------------- 1. class weights and the loop tail
@pytest.mark.parametrize("cw", [CW_DYADIC, CW_REAL], ids=["dyadic-w", "real-w"])
@pytest.mark.parametrize("mode,reduce", MODES)
@pytest.mark.parametrize("D,V,n_list", CW_CASES)
def test_class_weighted_routes_at_every_shape(env, D, V, n_list, mode, reduce, cw):
    P = problem(env, D, V, n_list, mode, reduce)
    D = P.D
    r = weighted_ref(env, P, cw)
    what = "D=%d V=%d n=%d %s %s cw=%s" % (D, V, P.n, mode, reduce, cw)
    refused = det_refused(env, D)
    got = {}
    for route in CW_ROUTES:
        if refused and route in DET_ROUTES:
            assert_refused(env, P, route, cw)
            continue
        got[route] = g = run(env, P, route, cw)
        _check(route, g, r, "%s %s" % (route, what))
        if mode == "dyadic":
            assert g["correct"] == r.correct, (route, what, g["correct"], r.correct)
        if route in DET_ROUTES:                                  # one CTA: the same bits
            one = run(env, P, route, cw, max_ctas=1)
            same_bits(one, g, ("dO", "g_ih", "g_ho", "loss", "correct"), route + " 1 CTA " + what)
    check_loop_tail(got["loop_tail"], got["fwd_do"], False, "loop_tail " + what)
    if not refused:
        check_loop_tail(got["loop_tail_det"], got["fwd_do_det"], True, "loop_tail_det " + what)
    if mode == "realistic":
        print("%s: %d window(s) with |o64| within the logit bound" % (what, r.count_band()[2]))
    if cw != CW_DYADIC:
        return
    # the plain forms: a power-of-two weight scales dO exactly, (1, 1) is the plain bits, the plain tail is its forward
    w = np.where(P.label[P.win] != 0, F32(cw[1]), F32(cw[0]))
    plain = {}
    for route in got:
        plain[route] = p = run(env, P, route, None)
        if "dO" in OUTPUTS[route]:
            assert np.array_equal(got[route]["dO"], p["dO"] * w), route + " dO * w " + what
        unit = run(env, P, route, (1.0, 1.0))
        exact = {"dO", "correct"} | ({"c", "g_ih", "g_ho", "loss"} if route in FIXED_ORDER else set())
        if route in ("fwdbwd_csc", "fwdbwd_csc_det"):
            exact.add("g_ih")                                    # written once per row from the same dO
        same_bits(unit, p, sorted(exact & (set(OUTPUTS[route]) | {"correct"})), "(1, 1) " + route + " " + what)
    check_loop_tail(plain["loop_tail"], plain["fwd_do"], False, "plain loop_tail " + what)
    lt = plain["loop_tail"]
    check_forward(P, lt["loss"], lt["correct"], "plain loop_tail " + what, dO=lt["dO"], g_ho=lt["g_ho"])
    if not refused:
        check_loop_tail(plain["loop_tail_det"], plain["fwd_do_det"], True, "plain loop_tail_det " + what)
        ltd = plain["loop_tail_det"]
        check_forward(P, ltd["loss"], ltd["correct"], "plain loop_tail_det " + what, dO=ltd["dO"], g_ho=ltd["g_ho"])
    else:                                                        # the plain forms are refused as well
        for route in DET_ROUTES:
            assert_refused(env, P, route, None)
    plain_ref(P)
    for route in ("fwdbwd", "fwdbwd_csc"):                       # the plain atomic routes against the plain reference
        p = plain[route]
        check_forward(P, p["loss"], p["correct"], "plain " + route + " " + what, g_ho=p["g_ho"], g_ih=p["g_ih"])


# --------------------------------------------------------------------------------------- 2. largest D, weighted
def test_largest_hidden_size_runs_weighted_and_the_next_is_refused(env):
    """The weighted generic kernel (fwdbwd_cw) at the largest D its shared memory admits, the weighted deterministic
    one (fwd_do_det_cw) at its own: within the weighted bound; D + 1 refused, no error left behind."""
    import torch
    from tests import helpers
    lib, capi = env["lib"], env["capi"]
    V, n = 101, 65
    rowptr, gene, label, win = make_windows(V, n, 5, "sum")
    cu = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).astype(dt)).cuda()
    rp, ge, la, wi = cu(rowptr, np.int32), cu(gene, np.int32), cu(label, np.uint8), cu(win, np.int32)
    N = len(rowptr) - 1
    st = torch.cuda.current_stream().cuda_stream
    z = lambda *s, dtype=torch.float32: torch.zeros(*s, dtype=dtype, device="cuda")
    for D, det in ((generic_max_d(env["optin"]), False), (det_max_d(env["optin"]), True)):
        for dd, ok in ((D, True), (D + 1, False)):
            W, Wo = helpers.init_weights(V, dd, 1)
            Wd, Wod = cu(W, np.float32), cu(Wo, np.float32)
            g_ho, acc, dO, g_ih = z(dd), z(2, dtype=torch.int64), z(n), z(V, dd)
            l0 = capi.launch_count()
            if det:
                ws = torch.empty(int(lib.g2v_cbow_det_workspace_bytes(n, dd)), dtype=torch.uint8, device="cuda")
                rc = lib.g2v_cbow_fwd_do_det_cw(rp.data_ptr(), ge.data_ptr(), la.data_ptr(), wi.data_ptr(), n, 1.0 / N,
                                                Wd.data_ptr(), Wod.data_ptr(), dO.data_ptr(), g_ho.data_ptr(),
                                                acc.data_ptr(), acc.data_ptr() + 8, V, dd, 0, ws.data_ptr(), 0,
                                                CW_REAL[0], CW_REAL[1], st)
            else:
                rc = lib.g2v_cbow_fwdbwd_cw(rp.data_ptr(), ge.data_ptr(), la.data_ptr(), wi.data_ptr(), 0, n, 1.0 / N,
                                            Wd.data_ptr(), Wod.data_ptr(), g_ih.data_ptr(), g_ho.data_ptr(),
                                            acc.data_ptr(), acc.data_ptr() + 8, V, dd, 0, CW_REAL[0], CW_REAL[1], st)
            what = "D=%d det=%s" % (dd, det)
            if ok:
                capi.check(rc, what)
                torch.cuda.synchronize()
                r = cwo.WeightedStep(rowptr, gene, label, win, N, W, Wo, CW_REAL)
                lo, hi, _ = r.count_band()
                a = acc.cpu().numpy()
                assert lo <= int(a[1]) <= hi, what
                assert abs(float(a[:1].view(np.float64)[0]) - r.loss_terms.sum()) <= r.loss_err, what
                assert_within(g_ho.cpu().numpy(), r.g_ho, r.g_ho_err, "g_ho " + what)
                if det:
                    assert_within(dO.cpu().numpy(), r.dO * r.s, r.dO_err * r.s + f64.U * np.abs(r.dO * r.s),
                                  "dO " + what)
                else:
                    assert_within(g_ih.cpu().numpy(), r.g_ih(), r.g_ih_err(), "g_ih " + what)
            else:
                assert rc == 2, (what, rc)
                assert "sizeHiddenlayer" in lib.g2v_last_error().decode()
                assert capi.launch_count() == l0, what
                torch.cuda.synchronize()
                assert torch.cuda.current_stream().query()
                # no sticky or pending error: a following weighted launch succeeds
                W1, Wo1 = (cu(x, np.float32) for x in helpers.init_weights(V, 100, 1))
                acc.zero_()
                capi.check(lib.g2v_cbow_fwdbwd_cw(rp.data_ptr(), ge.data_ptr(), la.data_ptr(), wi.data_ptr(), 0, n,
                                                  1.0 / N, W1.data_ptr(), Wo1.data_ptr(), z(V, 100).data_ptr(),
                                                  z(100).data_ptr(), acc.data_ptr(), acc.data_ptr() + 8, V, 100, 0,
                                                  CW_REAL[0], CW_REAL[1], st), "fwdbwd_cw after refusal " + what)
                torch.cuda.synchronize()
                assert int(acc.cpu()[1]) > 0


# ------------------------------------------------------------------------------------------- 3. dense decay
@pytest.mark.parametrize("lam", DENSE_LAMS)
@pytest.mark.parametrize("t", DENSE_T)
@pytest.mark.parametrize("D,V", DENSE_WD_SHAPES)
def test_dense_decay_at_every_tail(env, D, V, t, lam):
    lib = env["lib"]
    P = Dense(V, D, 5 * D + V + t, t)
    for name, opt in DENSE_VARIANTS:
        what = "%s D=%d V=%d t=%d lam=%g" % (name, D, V, t, lam)
        hyper = hyper_at(t) if name == "adam_dev" else None
        fused, comp = P.device(), P.device()
        assert launches(env, lambda: P.call(lib, fused, opt, t, hyper, wd=lam)) == 1
        torch_decay(comp["W"], lam)
        torch_decay(comp["Wo"], lam)
        Wdec, Wodec = wdo.decay32(P.h["W"], lam), wdo.decay32(P.h["Wo"], lam)
        assert bits(comp["W"]) == Wdec.tobytes() and bits(comp["Wo"]) == Wodec.tobytes()
        launches(env, lambda: P.call(lib, comp, opt, t, hyper))
        for k in fused:
            assert bits(fused[k]) == bits(comp[k]), (what, k)
        assert float(fused["g"].abs().max()) == 0.0 and float(fused["go"].abs().max()) == 0.0, what
        W, Wo = fused["W"].cpu().numpy(), fused["Wo"].cpu().numpy()
        # g = m = v = 0: the element ends at fl(w - fl(λ w))
        assert W[P.zero_rows].tobytes() == Wdec[P.zero_rows].tobytes(), what
        # the step on the decayed weights, against float64 (the last element is the scalar tail of W_ih)
        if opt == ADAM:
            (W1, m1, v1), (eW, em, ev) = f64.adam64(Wdec, P.h["m"], P.h["v"], P.h["g"], LR, t)
            (Wo1, _, _), (eWo, _, _) = f64.adam64(Wodec, P.h["mo"], P.h["vo"], P.h["go"], LR, t)
            assert_within(fused["m"].cpu().numpy(), m1, em, what + " m")
            assert_within(fused["v"].cpu().numpy(), v1, ev, what + " v")
        else:
            W1, eW = f64.sgd64(Wdec, P.h["g"], LR)
            Wo1, eWo = f64.sgd64(Wodec, P.h["go"], LR)
        assert_within(W, W1, eW, what + " W_ih")
        assert_within(Wo, Wo1, eWo, what + " W_ho")
        # λ = 0: the plain update's bits and launch count
        a, b = P.device(), P.device()
        na = launches(env, lambda: P.call(lib, a, opt, t, hyper))
        nb = launches(env, lambda: P.call(lib, b, opt, t, hyper, wd=0.0))
        assert na == nb == 1, what
        for k in a:
            assert bits(a[k]) == bits(b[k]), (what, "λ = 0", k)


# -------------------------------------------------------------------------------------------- 4. lazy decay
@pytest.mark.parametrize("D,V,n_list", CW_CASES)
def test_lazy_decay_on_the_problem_rows(env, D, V, n_list):
    """g2v_cbow_lazy_adam_wd on the touched rows and CSC segments of a CASES Problem: D % 4 != 0 (scalar rows), D > 256
    (a W_ho step over several 256-thread blocks) and the largest D."""
    import torch
    P = problem(env, D, V, n_list, "dyadic", "sum")
    D, V, lib = P.D, P.V, env["lib"]
    rs = np.random.RandomState(D + 3)
    dO = torch.from_numpy((rs.randn(max(P.n, 1)) * 1e-2).astype(F32)).cuda()
    plan = (P.d["rows"], P.d["segptr"], P.d["pos"], dO)
    h = {"W": P.W, "m": (rs.randn(V, D) * 1e-3).astype(F32), "v": (rs.rand(V, D) * 1e-6).astype(F32),
         "Wo": P.Who, "mo": (rs.randn(D) * 1e-3).astype(F32), "vo": (rs.rand(D) * 1e-6).astype(F32),
         "go": (rs.randn(D) * 1e-2).astype(F32)}
    new = lambda: {k: torch.from_numpy(np.ascontiguousarray(v).copy()).cuda() for k, v in h.items()}
    t = 2
    n_launch = 2 if len(P.rows) else 1
    # λ = 0: the plain call's bits and launches
    a, b = new(), new()
    na = launches(env, lambda: _lazy_call(lib, plan, a, V, D, t))
    nb = launches(env, lambda: _lazy_call(lib, plan, b, V, D, t, wd=0.0))
    assert na == nb == n_launch
    for k in a:
        assert bits(a[k]) == bits(b[k]), k
    # λ > 0: the listed rows as "decay them, then the λ = 0 call"; W_ho as "decay W_ho, then the λ = 0 call"
    fused, comp, comp_o = new(), new(), new()
    assert launches(env, lambda: _lazy_call(lib, plan, fused, V, D, t, wd=LAM)) == n_launch
    ri = P.d["rows"].long()
    comp["W"][ri] = comp["W"][ri] - (LAM * comp["W"][ri])
    torch_decay(comp_o["Wo"], LAM)
    launches(env, lambda: _lazy_call(lib, plan, comp, V, D, t))
    launches(env, lambda: _lazy_call(lib, plan, comp_o, V, D, t))
    for k in ("W", "m", "v"):
        assert bits(fused[k]) == bits(comp[k]), k
    for k in ("Wo", "mo", "vo", "go"):
        assert bits(fused[k]) == bits(comp_o[k]), k
    # every element of W_ho took its step (non-zero gradient) and had its gradient zeroed
    assert float(fused["go"].abs().max()) == 0.0
    assert (fused["Wo"].cpu().numpy() != wdo.decay32(P.Who, LAM)).all()
    untouched = np.setdiff1d(np.arange(V), P.rows)
    for k in ("W", "m", "v"):
        assert fused[k].cpu().numpy()[untouched].tobytes() == np.ascontiguousarray(h[k][untouched]).tobytes(), k


# ------------------------------------------------------------------------------------------- 5. rank-1 decay
@pytest.mark.parametrize("D", R1_DS)
def test_rank1_decay_at_every_path(env, D):
    import torch
    lib, capi, V = env["lib"], env["capi"], R1_V
    D = generic_max_d(env["optin"]) if D == "max" else D
    h = _r1_problem(lib, V, D, D + 7, dyadic=True)
    new = lambda: {k: torch.from_numpy(v.copy()).cuda() for k, v in h.items()}
    W64, Wo64, c64 = (h[k].astype(np.float64) for k in ("W", "Wo", "c"))
    gih = np.outer(c64, Wo64)                                    # exact: 6-bit integers times powers of two
    gho = W64.T @ c64
    assert (gih.astype(F32) == gih).all() and (gho.astype(F32) == gho).all()
    zero = np.arange(V)[::5]
    Wdec, Wodec = wdo.decay32(h["W"], LAM), wdo.decay32(h["Wo"], LAM)
    for opt in R1_OPTS:
        what = "D=%d opt=%d" % (D, opt)
        a, b = new(), new()
        na = launches(env, lambda: _r1_call(lib, a, V, D, opt, 1))
        nb = launches(env, lambda: _r1_call(lib, b, V, D, opt, 1, wd=0.0))
        assert na == nb == 3, what
        for k in a:
            if k != "scratch":
                assert bits(a[k]) == bits(b[k]), (what, "λ = 0", k)
        # λ > 0: W_ih as "decay W_ih, then the λ = 0 call", W_ho as "decay W_ho, then the λ = 0 call"
        f, ci, co = new(), new(), new()
        assert launches(env, lambda: _r1_call(lib, f, V, D, opt, 1, wd=LAM)) == 3
        torch_decay(ci["W"], LAM)
        torch_decay(co["Wo"], LAM)
        launches(env, lambda: _r1_call(lib, ci, V, D, opt, 1))
        launches(env, lambda: _r1_call(lib, co, V, D, opt, 1))
        for k in ("W", "m", "v"):
            assert bits(f[k]) == bits(ci[k]), (what, k)
        for k in ("Wo", "mo", "vo"):
            assert bits(f[k]) == bits(co[k]), (what, k)
        assert float(f["c"].abs().max()) == 0.0, what
        W, Wo = f["W"].cpu().numpy(), f["Wo"].cpu().numpy()
        # rows with c[g] = 0 (and zero moments) end at the decay, under SGD too
        assert W[zero].tobytes() == Wdec[zero].tobytes(), what
        # within the float64 step on the decayed weights, g_ho from the pre-decay W_ih
        z = lambda s: np.zeros(s, F32)
        if opt == ADAM:
            (W1, _, _), (eW, _, _) = f64.adam64(Wdec, z((V, D)), z((V, D)), gih.astype(F32), LR, 1)
            (Wo1, _, _), (eWo, _, _) = f64.adam64(Wodec, z(D), z(D), gho.astype(F32), LR, 1)
        else:
            W1, eW = f64.sgd64(Wdec, gih.astype(F32), 0.5)
            Wo1, eWo = f64.sgd64(Wodec, gho.astype(F32), 0.5)
        assert_within(W, W1, eW, what + " W_ih")
        assert_within(Wo, Wo1, eWo, what + " W_ho")
        # s refreshed for the new weights
        s2 = torch.zeros(V, device="cuda")
        capi.check(lib.g2v_cbow_r1_prepare(f["W"].data_ptr(), f["Wo"].data_ptr(), s2.data_ptr(), V, D,
                                           torch.cuda.current_stream().cuda_stream), "g2v_cbow_r1_prepare")
        assert bits(f["s"]) == bits(s2), what
    # SGD with lr = 0.5 and λ = 0.25 keeps every product exact: W_ho is fl(0.75 W_ho - 0.5 g_ho) with g_ho from the
    # weights before the step, and not from the decayed ones
    d = new()
    launches(env, lambda: _r1_call(lib, d, V, D, SGD, 1, wd=0.25))
    wo = wdo.decay32(h["Wo"], 0.25).astype(np.float64)
    got = d["Wo"].cpu().numpy()
    g_post = (W64 * 0.75).T @ c64
    assert got.tobytes() == (wo - 0.5 * gho).astype(F32).tobytes()
    differs = (wo - 0.5 * gho).astype(F32) != (wo - 0.5 * g_post).astype(F32)
    assert differs.any() and (got[differs] != (wo - 0.5 * g_post).astype(F32)[differs]).all()
