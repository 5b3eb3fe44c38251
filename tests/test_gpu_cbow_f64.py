"""Every CBOW entry point of the C ABI against the float64 reference of tests/f64_reference.py, element by element.

Two modes per shape:
  dyadic     weights that are small integers times a power of two (every float32 sum of the forward exact in any
             order): the correct count equals the float64 count exactly -- windows with o == 0 exactly included, so
             `>` versus `>=` shows -- and, with a test-chosen dyadic dO, the expansions, s = W_ih . W_ho and the
             lazy-Adam gradients are bit-exact;
  realistic  init_weights scale: every element within its worst-case bound; the count may differ only on windows
             whose |o64| is within the logit's bound (reported, normally 0).
The hidden sizes reach every branch of the kernels: D % 4 != 0 (scalar paths), V*D % 4 in {1, 2, 3} (scalar tails of
the dense update and the snapshot), D > 768 (generic rows kernels with opt-in shared memory), D > 1536 (rank-1 update
with opt-in shared memory) up to the largest D the generic kernel admits; 128, 256 and 512 are controls."""
import numpy as np
import pytest

from tests import helpers
from tests import f64_reference as f64

pytestmark = pytest.mark.gpu
F32 = np.float32
POOL = [0, 1, 2, 7, 8, 9, 81]
POOL_MEAN = [0, 1, 2, 8, 64]

# D ("max" = the largest hidden size the generic rows kernel admits), V (odd: V*D % 4 takes 1, 2 and 3), list length
CASES = [(1, 4097, 7), (3, 1001, 8), (31, 1001, 63), (33, 999, 64), (127, 1003, 65), (129, 4097, 20000),
         (130, 1001, 1), (513, 999, 2000), (769, 1001, 777), (1000, 1001, 1000), (1537, 1001, 500),
         ("max", 4097, 20000), (128, 1001, 3000), (256, 1001, 3000), (512, 1001, 3000)]


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available()
    from g2vec_b200 import _capi
    p = torch.cuda.get_device_properties(0)
    return {"lib": _capi.load(), "capi": _capi, "sm": p.multi_processor_count,
            "optin": p.shared_memory_per_block_optin}


def generic_max_d(optin):
    """The largest D whose generic rows kernel fits: 8 warps x 2 rows of D floats, plus its 16-byte static CtaAcc."""
    return (optin - 16) // 64


def det_max_d(optin):
    return (optin - 1024) // 64


def make_windows(V, n_list, seed, reduce):
    """A list of n_list positions over n_list + 3 windows: lengths from the pool, a few of 1000 and one of 4096 when V
    allows, and gene-pair windows {2j, 2j + 1} (o == 0 exactly with the dyadic weights)."""
    rs = np.random.RandomState(seed)
    pool = POOL_MEAN if reduce == "mean" else POOL
    N = n_list + 3
    lens = rs.choice(pool, size=N)
    big = [1024 if reduce == "mean" else 1000] * 3 + ([4096] if V >= 4097 else [])
    for l in big:
        if V > l and N > 8:
            lens[rs.randint(N)] = l
    if N > 8:                                               # the list's first window is the longest
        lens[0] = max([l for l in big if V > l] or [pool[-1]])
    rows = []
    for i, l in enumerate(lens):
        if l == 2 and i % 3 == 0:
            j = 2 * rs.randint(0, 8)
            rows.append(np.array([j, j + 1]))
        else:
            rows.append(np.sort(rs.choice(V, size=l, replace=False)))
    rowptr = np.zeros(N + 1, np.int32); rowptr[1:] = np.cumsum(lens)
    gene = np.concatenate(rows).astype(np.int32)
    label = (rs.rand(N) < 0.5).astype(np.uint8)
    win = rs.permutation(N)[:n_list].astype(np.int64)
    if n_list > 1:
        win[0] = 0                                          # the longest window is in the list
    return rowptr, gene, label, win


class Problem:
    def __init__(self, D, V, n_list, mode, reduce, seed, sm):
        import torch
        self.D, self.V, self.mode, self.reduce = D, V, mode, reduce
        rowptr, gene, label, win = make_windows(V, n_list, seed, reduce)
        self.rowptr, self.gene, self.label, self.win = rowptr, gene, label, win
        self.N = len(rowptr) - 1
        self.n = len(win)
        if mode == "dyadic":
            self.W, self.Who, self.a = f64.dyadic_problem(rowptr, gene, V, D, seed=seed, reduce=reduce)
        else:
            self.W, self.Who = helpers.init_weights(V, D, seed)
        chain = f64.atomic_chain(self.n, sm) + f64.det_chain(self.n) + 64
        self.ref = f64.Step(rowptr, gene, label, win, self.N, self.W, self.Who, reduce=reduce, chain=chain)
        self.cscptr, self.pos = f64.csc_of(rowptr, gene, win, V)
        k = np.diff(self.cscptr)
        self.rows = np.nonzero(k)[0].astype(np.int32)
        self.segptr = np.append(self.cscptr[self.rows], self.cscptr[-1]).astype(np.int32)
        cu = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).astype(dt)).cuda()
        self.d = {"rowptr": cu(rowptr, np.int32), "gene": cu(gene if len(gene) else np.zeros(1), np.int32),
                  "label": cu(label, np.uint8), "win": cu(win, np.int32), "W": cu(self.W, np.float32),
                  "Who": cu(self.Who, np.float32), "cscptr": cu(self.cscptr, np.int32), "pos": cu(self.pos, np.int32),
                  "rows": cu(self.rows, np.int32), "segptr": cu(self.segptr, np.int32)}
        self.k_max = int(k.max()) if len(k) else 1


_problems = {}


def problem(env, D, V, n_list, mode, reduce):
    if D == "max":
        D = generic_max_d(env["optin"])
    key = (D, V, n_list, mode, reduce)
    if key not in _problems:
        _problems.clear()                                     # one large reference at a time
        _problems[key] = Problem(D, V, n_list, mode, reduce, seed=(D * 7 + n_list) % 10007, sm=env["sm"])
    return _problems[key]


def zeros(*shape, dtype=None):
    import torch
    return torch.zeros(*shape, dtype=dtype or torch.float32, device="cuda")


def stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def loss_count(acc):
    a = acc.cpu().numpy()
    return float(a[:1].view(np.float64)[0]), int(a[1])


def assert_within(got, want, err, what):
    got = np.asarray(got, np.float64)
    bad = np.abs(got - want) > err
    assert not bad.any(), "%s: %d elements outside the bound, first at %s: got %r want %r bound %r" % (
        what, int(bad.sum()), np.argwhere(bad)[0], got[bad][0], np.asarray(want)[bad][0], np.asarray(err)[bad][0])


def check_forward(P, loss, nc, what, dO=None, g_ho=None, g_ih=None, report=None):
    r = P.ref
    if P.mode == "dyadic":
        assert nc == r.correct, (what, nc, r.correct)
    else:
        lo, hi, amb = r.count_band()
        assert lo <= nc <= hi, (what, nc, lo, hi)
        if report is not None:
            report.append(amb)
    if loss is not None:
        assert abs(loss - r.loss_terms.sum()) <= r.loss_err, (what, loss, r.loss_terms.sum(), r.loss_err)
    if dO is not None:
        assert_within(dO, r.dO * r.s, r.dO_err * r.s + f64.U * np.abs(r.dO * r.s), what + " dO")
    if g_ho is not None:
        assert_within(g_ho, r.g_ho, r.g_ho_err, what + " g_ho")
    if g_ih is not None:
        assert_within(g_ih, r.g_ih(), r.g_ih_err(), what + " g_ih")


def refused(env, rc, what):
    assert rc == 2, (what, rc)
    assert "sizeHiddenlayer" in env["lib"].g2v_last_error().decode()


@pytest.mark.parametrize("mode,reduce", [("dyadic", "sum"), ("realistic", "sum"), ("dyadic", "mean"),
                                         ("realistic", "mean")])
@pytest.mark.parametrize("D,V,n_list", CASES)
def test_rows_forward_and_backward_entry_points(env, D, V, n_list, mode, reduce):
    import torch
    lib, capi = env["lib"], env["capi"]
    P = problem(env, D, V, n_list, mode, reduce)
    D, V, n, d = P.D, P.V, P.n, P.d
    red = {"sum": 0, "mean": 1}[reduce]
    inv_n = 1.0 / P.N
    st = stream()
    args = (d["rowptr"].data_ptr(), d["gene"].data_ptr(), d["label"].data_ptr())
    amb = []
    # scatter
    g_ih, g_ho, acc = zeros(V, D), zeros(D), zeros(2, dtype=torch.int64)
    capi.check(lib.g2v_cbow_fwdbwd(*args, d["win"].data_ptr(), 0, n, inv_n, d["W"].data_ptr(), d["Who"].data_ptr(),
                                   g_ih.data_ptr(), g_ho.data_ptr(), acc.data_ptr(), acc.data_ptr() + 8, V, D, red, st),
               "g2v_cbow_fwdbwd")
    check_forward(P, *loss_count(acc), "scatter", g_ho=g_ho.cpu().numpy(), g_ih=g_ih.cpu().numpy(), report=amb)
    # CSC backward
    g_ih.zero_(); g_ho.zero_(); acc.zero_()
    dO = torch.full((n,), float("nan"), device="cuda")
    capi.check(lib.g2v_cbow_fwdbwd_csc(*args, d["win"].data_ptr(), n, inv_n, d["W"].data_ptr(), d["Who"].data_ptr(),
                                       d["cscptr"].data_ptr(), d["pos"].data_ptr(), dO.data_ptr(), g_ih.data_ptr(),
                                       g_ho.data_ptr(), acc.data_ptr(), acc.data_ptr() + 8, V, D, red, st),
               "g2v_cbow_fwdbwd_csc")
    dO_csc = dO.cpu().numpy()
    check_forward(P, *loss_count(acc), "csc", dO=dO_csc, g_ho=g_ho.cpu().numpy(), g_ih=g_ih.cpu().numpy())
    # the expansion of the kernel's own dO: any float32 order of its per-gene sums
    c64 = f64.grad_c_exact(P.cscptr, P.pos, dO_csc)
    want = np.outer(c64, P.Who.astype(np.float64))
    err = np.outer(f64.c_bound(P.cscptr, P.pos, dO_csc), np.abs(P.Who)) + 2 * f64.U * np.abs(want)
    assert_within(g_ih.cpu().numpy(), want, err, "csc expansion of its dO")
    # forward to dO only
    g_ho.zero_(); acc.zero_(); dO.fill_(float("nan"))
    capi.check(lib.g2v_cbow_fwd_do(*args, d["win"].data_ptr(), n, inv_n, d["W"].data_ptr(), d["Who"].data_ptr(),
                                   dO.data_ptr(), g_ho.data_ptr(), acc.data_ptr(), acc.data_ptr() + 8, V, D, red, st),
               "g2v_cbow_fwd_do")
    check_forward(P, *loss_count(acc), "fwd_do", dO=dO.cpu().numpy(), g_ho=g_ho.cpu().numpy())
    # accuracy pass, on the list and on a sub-range of the windows without a list
    acc.zero_()
    capi.check(lib.g2v_cbow_eval(*args, d["win"].data_ptr(), 0, n, d["W"].data_ptr(), d["Who"].data_ptr(),
                                 acc.data_ptr() + 8, V, D, red, st), "g2v_cbow_eval")
    check_forward(P, None, loss_count(acc)[1], "eval")
    # deterministic forms: max_ctas 1 and 0 give the same bits, each within the bounds
    dmax = det_max_d(env["optin"])
    ws = torch.empty(max(1, int(lib.g2v_cbow_det_workspace_bytes(n, D))), dtype=torch.uint8, device="cuda")
    outs = []
    for max_ctas in (1, 0):
        g_ih.zero_(); g_ho.zero_(); acc.zero_(); dO.fill_(float("nan"))
        rc = lib.g2v_cbow_fwdbwd_csc_det(*args, d["win"].data_ptr(), n, inv_n, d["W"].data_ptr(), d["Who"].data_ptr(),
                                         d["cscptr"].data_ptr(), d["pos"].data_ptr(), dO.data_ptr(), g_ih.data_ptr(),
                                         g_ho.data_ptr(), acc.data_ptr(), acc.data_ptr() + 8, V, D, red, ws.data_ptr(),
                                         max_ctas, st)
        if D > dmax and D not in (128, 256, 512):
            refused(env, rc, "fwdbwd_csc_det")
            break
        capi.check(rc, "g2v_cbow_fwdbwd_csc_det")
        r = [x.cpu().numpy().copy() for x in (dO, g_ih, g_ho, acc)]
        check_forward(P, *loss_count(acc), "csc_det", dO=r[0], g_ho=r[2], g_ih=r[1])
        g_ho2, acc2, dO2 = zeros(D), zeros(2, dtype=torch.int64), torch.full((n,), float("nan"), device="cuda")
        capi.check(lib.g2v_cbow_fwd_do_det(*args, d["win"].data_ptr(), n, inv_n, d["W"].data_ptr(),
                                           d["Who"].data_ptr(), dO2.data_ptr(), g_ho2.data_ptr(), acc2.data_ptr(),
                                           acc2.data_ptr() + 8, V, D, red, ws.data_ptr(), max_ctas, st),
                   "g2v_cbow_fwd_do_det")
        r += [x.cpu().numpy().copy() for x in (dO2, g_ho2, acc2)]
        outs.append(b"".join(x.tobytes() for x in r))
        assert r[4].tobytes() == r[0].tobytes() and r[5].tobytes() == r[2].tobytes()
    if len(outs) == 2:
        assert outs[0] == outs[1]
    torch.cuda.synchronize()
    if amb:
        print("D=%d %s %s: %d window(s) with |o64| within the logit bound" % (D, mode, reduce, max(amb)))


@pytest.mark.parametrize("D,V,n_list", CASES)
def test_expansions_lazy_adam_and_rank1(env, D, V, n_list):
    """Test-chosen dyadic dO: the batch expansion, the CSC expansion inside the rank-1 reduce and the lazy-Adam gradient
    are exact, so g_ih equals c (x) W_ho bit for bit; lazy Adam equals the dense update of that gradient bit for bit and
    both are within the float64 Adam bound; s = W_ih . W_ho is exact; the rank-1 windows pass is within its bounds."""
    import torch
    lib, capi = env["lib"], env["capi"]
    P = problem(env, D, V, n_list, "dyadic", "sum")
    D, V, n, d = P.D, P.V, P.n, P.d
    st = stream()
    B = int(np.abs(P.Who.astype(np.float64) * 2 ** 6).max())
    dO_np = f64.dyadic_dO(n, P.k_max, B, seed=D)
    dO = torch.from_numpy(dO_np).cuda()
    c = f64.grad_c_exact(P.cscptr, P.pos, dO_np)
    g_want = np.outer(c, P.Who.astype(np.float64))
    n_rows = len(P.rows)
    for max_ctas in (1, 0):
        g_ih = zeros(V, D)
        capi.check(lib.g2v_cbow_batch_expand(d["rows"].data_ptr(), d["segptr"].data_ptr(), d["pos"].data_ptr(),
                                             dO.data_ptr(), n_rows, d["Who"].data_ptr(), g_ih.data_ptr(), V, D,
                                             max_ctas, st), "g2v_cbow_batch_expand")
        assert (g_ih.cpu().numpy().astype(np.float64) == g_want).all(), max_ctas
    # lazy Adam (device alpha, t = 2 from a zero state) against the dense update of the same gradient
    t = 2
    alpha = f64.adam_tf1_alpha(0.005, t)
    b1p, b2p = F32(0.9) * F32(0.9), F32(0.999) * F32(0.999)
    hyper = torch.tensor([b1p, b2p, alpha, 0.0], dtype=torch.float32, device="cuda")
    Wl, Wol = d["W"].clone(), d["Who"].clone()
    ml, vl, mol, vol = zeros(V, D), zeros(V, D), zeros(D), zeros(D)
    g_ho_np = (np.random.RandomState(D).randn(D) * 1e-3).astype(F32)
    g_hol = torch.from_numpy(g_ho_np).cuda()
    capi.check(lib.g2v_cbow_lazy_adam(d["rows"].data_ptr(), d["segptr"].data_ptr(), d["pos"].data_ptr(), dO.data_ptr(),
                                      n_rows, Wl.data_ptr(), ml.data_ptr(), vl.data_ptr(), Wol.data_ptr(),
                                      mol.data_ptr(), vol.data_ptr(), g_hol.data_ptr(), V, D, 0.005, 0.9, 0.999, 1e-8,
                                      0, hyper.data_ptr(), st), "g2v_cbow_lazy_adam")
    Wd, Wod = d["W"].clone(), d["Who"].clone()
    md, vd, mod, vod = zeros(V, D), zeros(V, D), zeros(D), zeros(D)
    g_hod = torch.from_numpy(g_ho_np).cuda()
    capi.check(lib.g2v_cbow_update(Wd.data_ptr(), Wod.data_ptr(), md.data_ptr(), vd.data_ptr(), mod.data_ptr(),
                                   vod.data_ptr(), g_ih.data_ptr(), g_hod.data_ptr(), V, D, 0, 0.005, 0.9, 0.999, 1e-8, t,
                                   None, st), "g2v_cbow_update")
    for a, b in ((Wl, Wd), (ml, md), (vl, vd), (Wol, Wod), (mol, mod), (vol, vod)):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
    assert float(g_hol.abs().max()) == 0.0
    (W1, m1, v1), (dW, dm, dv) = f64.adam64(P.W, np.zeros_like(P.W), np.zeros_like(P.W), g_want.astype(F32), 0.005, t)
    assert (g_want.astype(F32).astype(np.float64) == g_want).all()
    assert_within(Wl.cpu().numpy(), W1, dW, "lazy adam W")
    assert_within(ml.cpu().numpy(), m1, dm, "lazy adam m")
    assert_within(vl.cpu().numpy(), v1, dv, "lazy adam v")
    untouched = np.diff(P.cscptr) == 0
    assert Wl.cpu().numpy()[untouched].tobytes() == P.W[untouched].tobytes()

    # rank-1: s exact, the windows pass (atomic and CSC) within the bounds, count exact
    s = zeros(V)
    capi.check(lib.g2v_cbow_r1_prepare(d["W"].data_ptr(), d["Who"].data_ptr(), s.data_ptr(), V, D, st),
               "g2v_cbow_r1_prepare")
    assert (s.cpu().numpy().astype(np.float64) == P.ref.s64).all()
    args = (d["rowptr"].data_ptr(), d["gene"].data_ptr(), d["label"].data_ptr())
    r = P.ref
    for csc in (False, True):
        cc, acc = zeros(V), zeros(2, dtype=torch.int64)
        if csc:
            dOr = torch.full((n,), float("nan"), device="cuda")
            capi.check(lib.g2v_cbow_r1_windows_csc(*args, d["win"].data_ptr(), n, 1.0 / P.N, s.data_ptr(),
                                                   d["cscptr"].data_ptr(), d["pos"].data_ptr(), dOr.data_ptr(),
                                                   cc.data_ptr(), acc.data_ptr(), acc.data_ptr() + 8, V, 0, st),
                       "g2v_cbow_r1_windows_csc")
            check_forward(P, *loss_count(acc), "r1 csc", dO=dOr.cpu().numpy())
        else:
            capi.check(lib.g2v_cbow_r1_windows(*args, d["win"].data_ptr(), 0, n, 1.0 / P.N, s.data_ptr(),
                                               cc.data_ptr(), acc.data_ptr(), acc.data_ptr() + 8, V, 0, st),
                       "g2v_cbow_r1_windows")
            check_forward(P, *loss_count(acc), "r1 atomic")
        assert_within(cc.cpu().numpy(), r.c, r.c_err, "r1 c")
    # rank-1 update on a dyadic c whose g_ih = c (x) W_ho and g_ho = W_ih^T c are exact: Adam (host alpha, t = 1) and SGD
    Cc = max(1, min(255, (2 ** 24 - 1) // (V * P.a), (2 ** 24 - 1) // max(B, 1)))
    c1 = (np.random.RandomState(D + 1).randint(-Cc, Cc + 1, V) * 2.0 ** -20).astype(F32)
    c1[::5] = 0
    gih = np.outer(c1.astype(np.float64), P.Who.astype(np.float64))
    gho = P.W.astype(np.float64).T @ c1.astype(np.float64)
    assert (gho.astype(F32) == gho).all()
    for opt in (0, 1):
        W, Wo, cd = d["W"].clone(), d["Who"].clone(), torch.from_numpy(c1).cuda()
        m_, v_, mo, vo = zeros(V, D), zeros(V, D), zeros(D), zeros(D)
        scratch = zeros(int(lib.g2v_cbow_r1_scratch_bytes(D)) // 4)
        capi.check(lib.g2v_cbow_r1_update(W.data_ptr(), Wo.data_ptr(), m_.data_ptr(), v_.data_ptr(), mo.data_ptr(),
                                          vo.data_ptr(), cd.data_ptr(), scratch.data_ptr(), s.data_ptr(), V, D, opt,
                                          0.005, 0.9, 0.999, 1e-8, 1, None, st), "g2v_cbow_r1_update")
        if opt == 0:
            (W1, _, _), (dW, _, _) = f64.adam64(P.W, np.zeros_like(P.W), np.zeros_like(P.W), gih.astype(F32), 0.005, 1)
            (Wo1, _, _), (dWo, _, _) = f64.adam64(P.Who, np.zeros(D, F32), np.zeros(D, F32), gho.astype(F32), 0.005, 1)
        else:
            W1, dW = f64.sgd64(P.W, gih.astype(F32), 0.005)
            Wo1, dWo = f64.sgd64(P.Who, gho.astype(F32), 0.005)
        assert_within(W.cpu().numpy(), W1, dW, "r1 update W_ih opt %d" % opt)
        assert_within(Wo.cpu().numpy(), Wo1, dWo, "r1 update W_ho opt %d" % opt)
        assert float(cd.abs().max()) == 0.0
        Wn = W.cpu().numpy().astype(np.float64); Won = Wo.cpu().numpy().astype(np.float64)
        assert_within(s.cpu().numpy(), Wn @ Won, f64.gamma(D + 1) * (np.abs(Wn) @ np.abs(Won)), "r1 s after update")


UPDATE_SHAPES = [(1, 4097), (3, 1001), (33, 999), (130, 1001), (769, 1001), (128, 1001)]


@pytest.mark.parametrize("t", [1, 2, 1000])
@pytest.mark.parametrize("D,V", UPDATE_SHAPES)
def test_dense_update_against_float64_adam_and_sgd(env, D, V, t):
    """g2v_cbow_update on a test-chosen gradient (exact zeros, values near eps, a wide range of magnitudes) and a
    non-zero optimizer state: TF1 Adam with host and device alpha, and SGD; every element within the float64 bound,
    and the gradient zeroed, the scalar tail of W_ih (V*D % 4 != 0) and W_ho included."""
    import torch
    lib, capi = env["lib"], env["capi"]
    rs = np.random.RandomState(D * 3 + t)
    n = V * D
    W = rs.randn(n).astype(F32); Wo = rs.randn(D).astype(F32)
    def grad(k):
        g = (rs.randn(k) * 10.0 ** rs.randint(-12, 1, k)).astype(F32)
        g[::7] = 0; g[1::11] = F32(1e-8); g[2::13] = -F32(3e-9)
        g[-1] = F32(0.25)                                          # the last element (scalar tail) is not zero
        return g
    g, go = grad(n), grad(D)
    m = (rs.randn(n) * 1e-3).astype(F32) if t > 1 else np.zeros(n, F32)
    v = (rs.rand(n) * 1e-6).astype(F32) if t > 1 else np.zeros(n, F32)
    mo = (rs.randn(D) * 1e-3).astype(F32) if t > 1 else np.zeros(D, F32)
    vo = (rs.rand(D) * 1e-6).astype(F32) if t > 1 else np.zeros(D, F32)
    cu = lambda a: torch.from_numpy(a.copy()).cuda()
    b1p, b2p = F32(1), F32(1)
    for _ in range(t):
        b1p = F32(b1p * F32(0.9)); b2p = F32(b2p * F32(0.999))
    hyper = torch.tensor([b1p, b2p, f64.adam_tf1_alpha(0.005, t), 0.0], dtype=torch.float32, device="cuda")
    for variant in ("adam_host", "adam_dev", "sgd"):
        dW, dWo, dm, dv, dmo, dvo, dg, dgo = (cu(x) for x in (W, Wo, m, v, mo, vo, g, go))
        opt = 1 if variant == "sgd" else 0
        capi.check(lib.g2v_cbow_update(dW.data_ptr(), dWo.data_ptr(), dm.data_ptr(), dv.data_ptr(), dmo.data_ptr(),
                                       dvo.data_ptr(), dg.data_ptr(), dgo.data_ptr(), V, D, opt, 0.005, 0.9, 0.999,
                                       1e-8, t if variant != "adam_dev" else 0,
                                       hyper.data_ptr() if variant == "adam_dev" else None, stream()),
                   "g2v_cbow_update")
        if opt == 0:
            (W1, m1, v1), (eW, em, ev) = f64.adam64(W, m, v, g, 0.005, t)
            (Wo1, mo1, vo1), (eWo, emo, evo) = f64.adam64(Wo, mo, vo, go, 0.005, t)
            assert_within(dm.cpu().numpy(), m1, em, variant + " m")
            assert_within(dv.cpu().numpy(), v1, ev, variant + " v")
            assert_within(dmo.cpu().numpy(), mo1, emo, variant + " m_ho")
            assert_within(dvo.cpu().numpy(), vo1, evo, variant + " v_ho")
        else:
            W1, eW = f64.sgd64(W, g, 0.005)
            Wo1, eWo = f64.sgd64(Wo, go, 0.005)
        assert_within(dW.cpu().numpy(), W1, eW, variant + " W_ih")
        assert_within(dWo.cpu().numpy(), Wo1, eWo, variant + " W_ho")
        assert float(dg.abs().max()) == 0.0 and float(dgo.abs().max()) == 0.0, variant


@pytest.mark.parametrize("D,V", [(1, 4097), (3, 1001), (130, 1001), (33, 999)])
def test_loop_begin_snapshot_copies_every_element(env, D, V):
    import torch
    lib, capi = env["lib"], env["capi"]
    W = torch.from_numpy(np.random.RandomState(D).randn(V * D).astype(F32)).cuda()
    snap = torch.full((V * D,), float("nan"), device="cuda")
    ctl = torch.zeros(8, dtype=torch.int64, device="cuda")
    acc = torch.full((6,), 7, dtype=torch.int64, device="cuda")
    capi.check(lib.g2v_cbow_loop_begin(ctl.data_ptr(), acc.data_ptr(), W.data_ptr(), snap.data_ptr(), V * D, stream()),
               "g2v_cbow_loop_begin")
    assert snap.cpu().numpy().tobytes() == W.cpu().numpy().tobytes()
    assert acc.cpu().tolist() == [0, 0, 0, 0, 7, 7]


@pytest.mark.parametrize("mode", ["dyadic", "realistic"])
@pytest.mark.parametrize("D,V", [(3, 1001), (130, 1001), (128, 1001)])
def test_step_host_entry_point(env, D, V, mode):
    import g2vec_b200 as g2v
    P = problem(env, D, V, 1000, mode, "sum")
    W, Wo = P.W.copy(), P.Who.copy()
    rowptr, gene, label = P.rowptr, P.gene, P.label
    # the host step runs every window of the CSR: restate the reference over all of them
    ref = f64.Step(rowptr, gene, label, np.arange(P.N), P.N, P.W, P.Who, chain=f64.atomic_chain(P.N, env["sm"]) + 64)
    state, loss, nc = g2v.cbow_step_host(rowptr, gene, label, W, Wo, lr=0.005, t=1)
    if mode == "dyadic":
        assert nc == ref.correct
    else:
        lo, hi, _ = ref.count_band()
        assert lo <= nc <= hi
    assert abs(loss - ref.loss_terms.sum()) <= ref.loss_err + 1e-12
    # element by element, with the gradient known to within its bound: Adam's first step on W_ih and W_ho, and its first
    # moment m = (1 - beta1) g, which carries the gradient itself (the step is close to alpha * sign(g))
    omb1 = float(F32(1) - F32(0.9))
    for got, m, g, g_err, W0, what in ((W, state[0], ref.g_ih(), ref.g_ih_err(), P.W, "W_ih"),
                                       (Wo, state[2], ref.g_ho, ref.g_ho_err, P.Who, "W_ho")):
        W1, dW = f64.adam64_first_step(W0, g, g_err, 0.005)
        assert_within(got, W1, dW, "step_host adam " + what)
        assert_within(m, omb1 * g, omb1 * g_err * (1 + 2 * f64.U) + 2 * f64.U * np.abs(omb1 * g), "step_host m " + what)
    # SGD: W' = W - lr g is linear in the gradient
    W, Wo = P.W.copy(), P.Who.copy()
    _, loss, nc = g2v.cbow_step_host(rowptr, gene, label, W, Wo, lr=0.5, optimizer="sgd")
    for got, g, g_err, W0, what in ((W, ref.g_ih(), ref.g_ih_err(), P.W, "W_ih"),
                                    (Wo, ref.g_ho, ref.g_ho_err, P.Who, "W_ho")):
        W1, dW = f64.sgd64(W0, g.astype(F32), 0.5)
        assert_within(got, W1, dW + 0.5 * (g_err + f64.U * np.abs(g)), "step_host sgd " + what)


@pytest.mark.parametrize("D,slabs", [(128, 7), (256, 3), (512, 5)])
def test_slab_passes_with_windows_longer_than_a_slab(env, monkeypatch, D, slabs):
    import torch
    import g2vec_b200 as g2v
    monkeypatch.setenv("G2V_CBOW_SLABS", str(slabs))
    V = 1001
    for mode in ("dyadic", "realistic"):
        P = problem(env, D, V, 3000, mode, "sum")
        assert P.ref.lmax >= 1000 > V // slabs
        m = g2v.CbowModel(P.rowptr, P.gene, P.label, V, D, P.W, P.Who)
        wd = P.d["win"]
        assert m.prepare_slabs(wd) and m._n_slabs == slabs
        m.fwdbwd(wd, P.N)
        m.evaluate(wd, 2)
        torch.cuda.synchronize()
        acc = m.acc.cpu()
        check_forward(P, m.loss_sum(acc), int(acc[1]), "slabs " + mode, g_ho=m.g_ho.cpu().numpy(),
                      g_ih=m.g_ih.cpu().numpy())
        check_forward(P, None, int(acc[2]), "slab eval " + mode)


def test_largest_hidden_size_runs_and_the_next_is_refused(env):
    """The generic rows kernel's shared memory (8 warps x 2 rows of D floats) plus its static accumulators must fit the
    opt-in limit: the largest admitted D runs, D + 1 is refused with the sizeHiddenlayer message and leaves no CUDA
    error behind.  The same for the deterministic forward, which reserves 1 KB."""
    import torch
    lib, capi = env["lib"], env["capi"]
    V, n = 101, 65
    rowptr, gene, label, win = make_windows(V, n, 5, "sum")
    cu = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).astype(dt)).cuda()
    rp, ge, la, wi = cu(rowptr, np.int32), cu(gene, np.int32), cu(label, np.uint8), cu(win, np.int32)
    N = len(rowptr) - 1
    for D, det in ((generic_max_d(env["optin"]), False), (det_max_d(env["optin"]), True)):
        for dd, ok in ((D, True), (D + 1, False)):
            W, Wo = helpers.init_weights(V, dd, 1)
            Wd, Wod = cu(W, np.float32), cu(Wo, np.float32)
            g_ho, acc, dO = zeros(dd), zeros(2, dtype=torch.int64), zeros(n)
            if det:
                ws = torch.empty(int(lib.g2v_cbow_det_workspace_bytes(n, dd)), dtype=torch.uint8, device="cuda")
                rc = lib.g2v_cbow_fwd_do_det(rp.data_ptr(), ge.data_ptr(), la.data_ptr(), wi.data_ptr(), n, 1.0 / N,
                                             Wd.data_ptr(), Wod.data_ptr(), dO.data_ptr(), g_ho.data_ptr(),
                                             acc.data_ptr(), acc.data_ptr() + 8, V, dd, 0, ws.data_ptr(), 0, stream())
            else:
                g_ih = zeros(V, dd)
                rc = lib.g2v_cbow_fwdbwd(rp.data_ptr(), ge.data_ptr(), la.data_ptr(), wi.data_ptr(), 0, n, 1.0 / N,
                                         Wd.data_ptr(), Wod.data_ptr(), g_ih.data_ptr(), g_ho.data_ptr(),
                                         acc.data_ptr(), acc.data_ptr() + 8, V, dd, 0, stream())
            if ok:
                capi.check(rc, "D=%d" % dd)
                torch.cuda.synchronize()
                ref = f64.Step(rowptr, gene, label, win, N, W, Wo)
                lo, hi, _ = ref.count_band()
                assert lo <= int(acc.cpu()[1]) <= hi
                assert_within(g_ho.cpu().numpy(), ref.g_ho, ref.g_ho_err, "g_ho at D=%d" % dd)
            else:
                refused(env, rc, "D=%d" % dd)
                torch.cuda.synchronize()
                assert torch.cuda.current_stream().query()
                # no sticky or pending error: a following launch succeeds
                acc.zero_()
                capi.check(lib.g2v_cbow_eval(rp.data_ptr(), ge.data_ptr(), la.data_ptr(), wi.data_ptr(), 0, n,
                                             cu(helpers.init_weights(V, 128, 1)[0], np.float32).data_ptr(),
                                             cu(helpers.init_weights(V, 128, 1)[1], np.float32).data_ptr(),
                                             acc.data_ptr() + 8, V, 128, 0, stream()), "eval after refusal")
                torch.cuda.synchronize()
