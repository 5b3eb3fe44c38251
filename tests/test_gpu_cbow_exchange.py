"""The multi-GPU exchange kernels on ONE GPU, with simulated ranks, against float64 and the single-GPU update.

g2v_cbow_update_nvl and g2v_cbow_loop_counters_nvl reach their peers only through device arrays of pointers
(g_ptrs_dev, w_ptrs_dev, hist_ptrs_dev), so `world` replicas allocated on one device stand for `world` GPUs: the
tables hold the replicas' addresses and the entry point is called once per simulated rank r = 0..world-1 on one
stream.  Launches on one stream run in order, which is the cross-GPU barrier the header asks for before and after every
call.  Both multicast pointers NULL select the peer load/store form: the code a multi-GPU run executes when the buffers
have no NVLS multicast object (G2V_CBOW_NVL_MULTICAST=0).  The multicast form (multimem.*) needs one multicast object
bound to the memory of several devices; it is tested only by tests/test_gpu_multi.py on a box with two or more GPUs.

  update      one step, element by element: dyadic gradients (every float32 sum over the ranks exact in any order)
              make the weights, m and v bit-identical to g2v_cbow_update on the summed gradient; realistic gradients
              stay within the float64 Adam / SGD bound; one rank alone changes exactly its slice and nothing else;
              12 steps with the device step size, eager and replayed from a CUDA graph; the `stopped` word and the
              argument checks.
  training    one simulated N-rank step of the real kernels (shard_by_nnz, g2v_cbow_fwdbwd per shard, the exchange):
              bit-identical to g2v_cbow_update on the float32 sum the exchange forms, within the float64 bound of one
              full-list step; a second step shows that the exchange zeroed every gradient replica.
  counters    g2v_cbow_loop_counters_nvl, then g2v_cbow_loop_decide[_best] with acc == NULL: exact sums above 2^32,
              the same decisions on every rank as one loop on the summed counters, the patience rule's stop step.
  adam_tick   the device step-size state against TF1's float32 beta powers for 1000 steps.

Shapes: n = (V + 1) * D takes every residue mod 4 (the scalar tail), n / 4 < world (ranks that own nothing) and, at
world 3, a slice several times the launch's thread count (the grid-stride loop); test_cases_reach_every_partition_branch
checks that the list does."""
import numpy as np
import pytest

from tests import helpers
from tests import f64_reference as f64
from tests import patience_oracle

pytestmark = pytest.mark.gpu
F32 = np.float32
LR, B1, B2, EPS = 0.005, 0.9, 0.999, 1e-8
ADAM, SGD = 0, 1

WORLDS = [1, 2, 3, 4, 5, 7, 8]
SHAPES = [(1, 1), (2, 1), (4, 1), (6, 1), (1000, 3), (1001, 3), (1000, 33), (999, 33), (7523, 128)]
GRID_STRIDE = (3, 2 ** 23 + 2, 1)                  # n = 2^23 + 3
CASES = [(w, V, D) for w in WORLDS for V, D in SHAPES] + [GRID_STRIDE]


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available()
    from g2vec_b200 import _capi
    return {"lib": _capi.load(), "capi": _capi, "sm": torch.cuda.get_device_properties(0).multi_processor_count}


def stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------ the partition
def float4_range(n, world, rank):
    """Elements [lo, hi) of rank's float4 slice: float4s [r*c, min(n/4, (r+1)*c)) with c = ceil((n/4) / world)."""
    n4 = n // 4
    c = -(-n4 // world)
    return 4 * min(n4, rank * c), 4 * min(n4, (rank + 1) * c)


def owned(n, world, rank):
    """Every element rank owns: its float4 slice, and for the last rank the scalar tail [4*floor(n/4), n)."""
    lo, hi = float4_range(n, world, rank)
    idx = np.arange(lo, hi)
    if rank == world - 1:
        idx = np.concatenate([idx, np.arange(4 * (n // 4), n)])
    return idx


def exchange_sum(gs, world):
    """The float32 sum g2v_cbow_update_nvl forms on the peer path: on its float4 slice rank r adds the replicas to 0 in
    the order r, r+1, ..., r-1 (mod world); the scalar tail adds them in the order 0, 1, ..., world-1."""
    n = len(gs[0])
    out = np.empty(n, F32)
    for r in range(world):
        lo, hi = float4_range(n, world, r)
        a = np.zeros(hi - lo, F32)
        for p in range(world):
            a = a + gs[(r + p) % world][lo:hi]
        out[lo:hi] = a
    t0 = 4 * (n // 4)
    a = np.zeros(n - t0, F32)
    for p in range(world):
        a = a + gs[p][t0:]
    out[t0:] = a
    return out


def test_cases_reach_every_partition_branch(env):
    """The shape list itself covers what the kernel's partition can do, and the partition is one of [0, n)."""
    threads = 4 * env["sm"] * 256                  # the launch's grid is capped at 4 CTAs of 256 threads per SM
    ns = [(w, (V + 1) * D) for w, V, D in CASES]
    assert {n % 4 for _, n in ns} == {0, 1, 2, 3}
    assert any(n % 4 and w > 1 for w, n in ns)                          # a tail owned by a rank other than rank 0
    empty = [(w, n) for w, n in ns if any(len(owned(n, w, r)) == 0 for r in range(w))]
    assert any(n // 4 < w for w, n in empty)                            # n/4 < world: some ranks own nothing
    assert any(n // 4 == 0 for _, n in empty)                           # no float4 at all: the tail is everything
    assert any(w == 3 and -(-(n // 4) // w) >= 4 * threads for w, n in ns)   # several grid strides per slice
    for w, n in ns:
        if n < 10 ** 6:
            assert (np.sort(np.concatenate([owned(n, w, r) for r in range(w)])) == np.arange(n)).all(), (w, n)


# ------------------------------------------------------------------------------------------------ simulated ranks
class Ranks:
    """`world` simulated ranks of a flat [W_ih | W_ho] vector of n floats: gradient, weight, m and v replicas, each its
    own allocation (16-byte aligned, as a symmetric-memory buffer is), and the device pointer tables of the gradient
    and the weight replicas."""

    def __init__(self, world, n):
        import torch
        self.world, self.n = world, n
        self.g, self.w, self.m, self.v = ([torch.zeros(n, device="cuda") for _ in range(world)] for _ in range(4))
        table = lambda ts: torch.tensor([t.data_ptr() for t in ts], dtype=torch.int64, device="cuda")
        self.g_tab, self.w_tab = table(self.g), table(self.w)

    def load(self, W=None, m=None, v=None, gs=None):
        import torch
        for name, x in (("w", W), ("m", m), ("v", v)):
            if x is not None:
                for t in getattr(self, name):
                    t.copy_(torch.from_numpy(x))
        if gs is not None:
            for t, g in zip(self.g, gs):
                t.copy_(torch.from_numpy(g))

    def call(self, lib, rank, opt, t, alpha_dev=None, world=None, n=None, g_mc=None, w_mc=None, mv=True):
        adam = opt == ADAM and mv
        mine = rank if 0 <= rank < self.world else 0     # the argument checks pass ranks outside [0, world)
        return lib.g2v_cbow_update_nvl(self.g_tab.data_ptr(), self.w_tab.data_ptr(), g_mc, w_mc,
                                       self.m[mine].data_ptr() if adam else None,
                                       self.v[mine].data_ptr() if adam else None, self.n if n is None else n, rank,
                                       self.world if world is None else world, opt, LR, B1, B2, EPS, t, alpha_dev,
                                       stream())

    def step(self, env, opt, t, alpha_dev=None):
        for r in range(self.world):
            env["capi"].check(self.call(env["lib"], r, opt, t, alpha_dev), "g2v_cbow_update_nvl rank %d" % r)

    def state(self):
        return b"".join(x.cpu().numpy().tobytes() for x in self.g + self.w + self.m + self.v)


def dense_update(env, V, D, W, m, v, g, opt, t, alpha_dev=None):
    """g2v_cbow_update on flat [W_ih | W_ho] tensors (W_ih = the first V*D elements, W_ho the last D), in place."""
    k = 4 * V * D
    p = lambda x, off=0: x.data_ptr() + off if (opt == ADAM) else None
    env["capi"].check(env["lib"].g2v_cbow_update(W.data_ptr(), W.data_ptr() + k, p(m), p(v), p(m, k), p(v, k),
                                                 g.data_ptr(), g.data_ptr() + k, V, D, opt, LR, B1, B2, EPS, t,
                                                 alpha_dev, stream()), "g2v_cbow_update")


def beta_powers(t):
    b1p, b2p = F32(1), F32(1)
    for _ in range(t):
        b1p = F32(b1p * F32(B1)); b2p = F32(b2p * F32(B2))
    return b1p, b2p


def hyper_at(t):
    """The device step-size state {beta1^t, beta2^t, alpha_t, 0} g2v_cbow_adam_tick leaves after t ticks."""
    import torch
    b1p, b2p = beta_powers(t)
    return torch.tensor([b1p, b2p, f64.adam_tf1_alpha(LR, t), 0.0], dtype=torch.float32, device="cuda")


def cu(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def assert_same(got, want, what):
    """Bit equality of two float32 tensors, reporting the first differing element."""
    import torch
    a, b = got.reshape(-1).view(torch.int32), want.reshape(-1).view(torch.int32)
    if torch.equal(a, b):
        return
    bad = (a != b).nonzero().flatten().cpu().numpy()
    i = int(bad[0])
    raise AssertionError("%s: %d element(s) differ, first at %d of %d: got %r want %r" % (
        what, len(bad), i, a.numel(), float(got.reshape(-1)[i]), float(want.reshape(-1)[i])))


def assert_zero(ts, what):
    for p, t in enumerate(ts):
        assert int((t != 0).sum()) == 0, "%s: gradient replica %d not zeroed" % (what, p)


def assert_within(got, want, err, what):
    got = np.asarray(got, np.float64)
    bad = np.abs(got - want) > err
    assert not bad.any(), "%s: %d elements outside the bound, first at %s: got %r want %r bound %r" % (
        what, int(bad.sum()), np.argwhere(bad)[0], got[bad][0], np.asarray(want)[bad][0], np.asarray(err)[bad][0])


def dyadic_grads(world, n, rs):
    """Per rank: integers in [-1023, 1023] times 2^-(10 + e), e in 0..8 per element (the same for every rank), so every
    float32 sum of <= 8 ranks stays below 2^13 quanta of its element and is exact in any order.  Every 17th element is
    zero on every rank; the last element is not zero."""
    q = 2.0 ** -(10 + rs.randint(0, 9, n))
    gs = []
    for r in range(world):
        g = (rs.randint(-1023, 1024, n) * q).astype(F32)
        g[::17] = 0
        g[-1] = F32((r + 1) * 2.0 ** -10)
        gs.append(g)
    total = np.sum([g.astype(np.float64) for g in gs], axis=0)
    assert (total.astype(F32) == total).all()
    return gs, total.astype(F32)


def adam_state(n, t, rs):
    if t == 1:
        return np.zeros(n, F32), np.zeros(n, F32)
    return (rs.randn(n) * 1e-3).astype(F32), (rs.rand(n) * 1e-6).astype(F32)


# ------------------------------------------------------------------------------------------------ 1. the update
UPDATE_VARIANTS = [("adam", 1, False), ("adam", 2, False), ("adam", 1000, False), ("adam", 7, True), ("sgd", 1, False)]


@pytest.mark.parametrize("world,V,D", CASES)
def test_update_nvl_dyadic_is_the_dense_update_bit_for_bit(env, world, V, D):
    """Exact gradient sums: every weight replica equals g2v_cbow_update on the summed gradient bit for bit, every
    rank's owned slice of m and v equals that run's m and v (the rest of its m and v is untouched), and every gradient
    replica is zero.  Adam with host alpha at t = 1, 2, 1000 (non-zero m, v for t > 1), with device alpha, and SGD."""
    import torch
    n = (V + 1) * D
    R = Ranks(world, n)
    rs = np.random.RandomState(n % 100003 * 8 + world)
    W0 = rs.randn(n).astype(F32)
    own = [torch.from_numpy(owned(n, world, r)).cuda() for r in range(world)]
    for kind, t, dev in UPDATE_VARIANTS:
        what = "%s t=%d%s world=%d n=%d" % (kind, t, " alpha_dev" if dev else "", world, n)
        opt = ADAM if kind == "adam" else SGD
        gs, gsum = dyadic_grads(world, n, rs)
        m0, v0 = adam_state(n, t, rs)
        R.load(W0, m0, v0, gs)
        hyper = hyper_at(t) if dev else None
        R.step(env, opt, 0 if dev else t, hyper.data_ptr() if dev else None)
        W, m, v = cu(W0), cu(m0), cu(v0)
        dense_update(env, V, D, W, m, v, cu(gsum), opt, 0 if dev else t, hyper.data_ptr() if dev else None)
        for p in range(world):
            assert_same(R.w[p], W, what + " weights of rank %d" % p)
        assert_zero(R.g, what)
        m0d, v0d = cu(m0), cu(v0)
        for r in range(world):
            rest = torch.ones(n, dtype=torch.bool, device="cuda")
            rest[own[r]] = False
            if opt == ADAM:
                assert_same(R.m[r][own[r]], m[own[r]], what + " m slice of rank %d" % r)
                assert_same(R.v[r][own[r]], v[own[r]], what + " v slice of rank %d" % r)
            assert_same(R.m[r][rest], m0d[rest], what + " m outside the slice of rank %d" % r)
            assert_same(R.v[r][rest], v0d[rest], what + " v outside the slice of rank %d" % r)


@pytest.mark.parametrize("world,V,D", CASES)
def test_update_nvl_realistic_within_float64_bound(env, world, V, D):
    """Gradients of magnitudes 1e-12..1 with exact zeros: every element within the adam64 / sgd64 bound evaluated on
    the float64 sum of the rank gradients, widened by the float32 error of a sum of `world` terms, gamma(world-1) *
    sum_r |g_r|.  Adam at t = 1 (host and device alpha; m = (1 - beta1) g carries the gradient itself) and SGD."""
    n = (V + 1) * D
    R = Ranks(world, n)
    rs = np.random.RandomState(n % 100003 * 8 + world + 1)
    W0 = rs.randn(n).astype(F32)
    gs = []
    for r in range(world):
        g = (rs.randn(n) * 10.0 ** rs.randint(-12, 1, n)).astype(F32)
        g[::7] = 0                                   # zero on every rank
        g[r + 1::11] = 0                             # zero on this rank only
        g[-1] = F32(0.25 * (r + 1))
        gs.append(g)
    g64 = np.sum([g.astype(np.float64) for g in gs], axis=0)
    err = f64.gamma(world - 1) * np.sum([np.abs(g.astype(np.float64)) for g in gs], axis=0)
    omb1 = float(F32(1) - F32(B1))
    z = np.zeros(n, F32)
    for kind, dev in (("adam", False), ("adam", True), ("sgd", False)):
        what = "%s%s world=%d n=%d" % (kind, " alpha_dev" if dev else "", world, n)
        opt = ADAM if kind == "adam" else SGD
        R.load(W0, z, z, gs)
        hyper = hyper_at(1)
        R.step(env, opt, 0 if dev else 1, hyper.data_ptr() if dev else None)
        for p in range(1, world):
            assert_same(R.w[p], R.w[0], what + " weights of rank %d" % p)
        assert_zero(R.g, what)
        got = R.w[0].cpu().numpy()
        if opt == ADAM:
            W1, dW = f64.adam64_first_step(W0, g64, err, LR)
            assert_within(got, W1, dW, what + " weights")
            m = np.empty(n, F32)
            for r in range(world):
                idx = owned(n, world, r)
                m[idx] = R.m[r].cpu().numpy()[idx]
            assert_within(m, omb1 * g64, omb1 * err * (1 + 2 * f64.U) + 2 * f64.U * np.abs(omb1 * g64), what + " m")
        else:
            W1, dW = f64.sgd64(W0, g64.astype(F32), LR)
            assert_within(got, W1, dW + float(F32(LR)) * (err + f64.U * np.abs(g64)), what + " weights")


@pytest.mark.parametrize("world,V,D", CASES)
def test_update_nvl_each_rank_changes_exactly_its_slice(env, world, V, D):
    """One rank alone, every replica filled with distinct non-zero values: g_p of every rank p becomes zero on the
    caller's slice, w_p of every rank takes the new weights there (computed from the caller's own w, m, v and the sum of
    every g_p on that slice), the caller's m and v change only there, and nothing else changes by a bit."""
    import torch
    n = (V + 1) * D
    R = Ranks(world, n)
    rs = np.random.RandomState(n % 100003 * 8 + world + 2)
    q = 2.0 ** -(10 + rs.randint(0, 9, n))
    mk = lambda f: [cu(f()) for _ in range(world)]
    g0 = mk(lambda: (rs.randint(1, 1024, n) * rs.choice([-1, 1], n) * q).astype(F32))
    w0 = mk(lambda: rs.randn(n).astype(F32))
    m0 = mk(lambda: (rs.randn(n) * 1e-3).astype(F32))
    v0 = mk(lambda: (rs.rand(n) * 1e-6 + 1e-9).astype(F32))
    gsum = torch.stack(g0).double().sum(0)
    assert torch.equal(gsum.float().double(), gsum)
    gsum = gsum.float()
    t = 3
    for r in range(world):
        for dst, src in zip((R.g, R.w, R.m, R.v), (g0, w0, m0, v0)):
            for a, b in zip(dst, src):
                a.copy_(b)
        env["capi"].check(R.call(env["lib"], r, ADAM, t), "g2v_cbow_update_nvl rank %d alone" % r)
        W, m, v = w0[r].clone(), m0[r].clone(), v0[r].clone()
        dense_update(env, V, D, W, m, v, gsum.clone(), ADAM, t)
        own = torch.from_numpy(owned(n, world, r)).cuda()
        rest = torch.ones(n, dtype=torch.bool, device="cuda")
        rest[own] = False
        what = "rank %d of %d alone, n=%d" % (r, world, n)
        for p in range(world):
            assert int((R.g[p][own] != 0).sum()) == 0, what + ": g of rank %d not zeroed on the slice" % p
            assert_same(R.g[p][rest], g0[p][rest], what + ": g of rank %d outside the slice" % p)
            assert_same(R.w[p][own], W[own], what + ": w of rank %d on the slice" % p)
            assert_same(R.w[p][rest], w0[p][rest], what + ": w of rank %d outside the slice" % p)
            if p == r:
                assert_same(R.m[p][own], m[own], what + ": m on the slice")
                assert_same(R.v[p][own], v[own], what + ": v on the slice")
                assert_same(R.m[p][rest], m0[p][rest], what + ": m outside the slice")
                assert_same(R.v[p][rest], v0[p][rest], what + ": v outside the slice")
            else:
                assert_same(R.m[p], m0[p], what + ": m of rank %d" % p)
                assert_same(R.v[p], v0[p], what + ": v of rank %d" % p)


@pytest.mark.parametrize("world,V,D", [(3, 1000, 3), (4, 6, 1), (5, 1001, 3), (7, 999, 33), (8, 7523, 128)])
def test_update_nvl_twelve_steps_eager_and_graph_replay(env, world, V, D):
    """12 steps of fresh dyadic gradients, each g2v_cbow_adam_tick then the `world` rank calls with alpha_dev: after every
    step the weights, the owned m / v slices and the step-size state equal the g2v_cbow_update trajectory bit for bit.
    A second set of replicas runs steps 2.. from ONE captured step (tick + rank calls) replayed as a CUDA graph, as the
    device loop replays this kernel: the same bits as the eager steps."""
    import torch
    n = (V + 1) * D
    T, CAPTURE_AT = 12, 2
    rs = np.random.RandomState(world * 31 + D)
    W0 = rs.randn(n).astype(F32)
    z = np.zeros(n, F32)
    A, B = Ranks(world, n), Ranks(world, n)
    A.load(W0, z, z); B.load(W0, z, z)
    W, m, v, g = cu(W0), cu(z), cu(z), cu(z)
    init = lambda: torch.tensor([1.0, 1.0, 0.0, 0.0], device="cuda")
    hA, hB, hR = init(), init(), init()
    tick = lambda h: env["capi"].check(env["lib"].g2v_cbow_adam_tick(h.data_ptr(), LR, B1, B2, stream()),
                                       "g2v_cbow_adam_tick")
    own = [torch.from_numpy(owned(n, world, r)).cuda() for r in range(world)]
    graph = None
    for s in range(T):
        gs, gsum = dyadic_grads(world, n, rs)
        A.load(gs=gs)
        tick(hA)
        A.step(env, ADAM, 0, hA.data_ptr())
        g.copy_(torch.from_numpy(gsum))
        tick(hR)
        dense_update(env, V, D, W, m, v, g, ADAM, 0, hR.data_ptr())
        B.load(gs=gs)
        if s < CAPTURE_AT:
            tick(hB)
            B.step(env, ADAM, 0, hB.data_ptr())
        else:
            if graph is None:
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    tick(hB)
                    B.step(env, ADAM, 0, hB.data_ptr())
            graph.replay()
        what = "step %d world=%d n=%d" % (s, world, n)
        assert_same(hA, hR, what + " step-size state")
        assert_same(hB, hR, what + " step-size state (graph)")
        for p in range(world):
            assert_same(A.w[p], W, what + " weights of rank %d" % p)
            assert_same(B.w[p], W, what + " weights of rank %d (graph)" % p)
            assert_same(A.m[p][own[p]], m[own[p]], what + " m slice of rank %d" % p)
            assert_same(A.v[p][own[p]], v[own[p]], what + " v slice of rank %d" % p)
            assert_same(B.m[p][own[p]], m[own[p]], what + " m slice of rank %d (graph)" % p)
            assert_same(B.v[p][own[p]], v[own[p]], what + " v slice of rank %d (graph)" % p)
        assert_zero(A.g, what)
        assert_zero(B.g, what + " (graph)")
    torch.cuda.synchronize()


def test_update_nvl_stopped_word_and_refused_arguments(env):
    """With a loop attached whose ctl.stopped is set the rank calls change no byte of any buffer.  Bad arguments are
    refused with a non-zero return code and a message, and launch nothing."""
    import torch
    lib, capi = env["lib"], env["capi"]
    world, V, D = 3, 1000, 3
    n = (V + 1) * D
    R = Ranks(world, n)
    rs = np.random.RandomState(4)
    gs, _ = dyadic_grads(world, n, rs)
    m0, v0 = adam_state(n, 2, rs)
    R.load(rs.randn(n).astype(F32), m0, v0, gs)
    hyper = hyper_at(2)
    torch.cuda.synchronize()
    before = R.state()
    ctl = torch.zeros(8, dtype=torch.int64, device="cuda")
    ctl[0] = 1
    capi.check(lib.g2v_cbow_loop_attach(ctl.data_ptr()), "g2v_cbow_loop_attach")
    try:
        for opt, t, adev in ((ADAM, 2, None), (ADAM, 0, hyper.data_ptr()), (SGD, 1, None)):
            R.step(env, opt, t, adev)
        torch.cuda.synchronize()
    finally:
        capi.check(lib.g2v_cbow_loop_attach(None), "g2v_cbow_loop_attach")
    assert R.state() == before, "a stopped loop's update changed a buffer"
    other = R.g[0].data_ptr()
    bad = [("rank < 0", dict(rank=-1)), ("rank >= world", dict(rank=world)), ("world < 1", dict(rank=0, world=0)),
           ("n < 1", dict(n=0)), ("g_multicast only", dict(g_mc=other)), ("w_multicast only", dict(w_mc=other)),
           ("Adam without m/v", dict(mv=False)), ("t < 1 without alpha_dev", dict(t=0))]
    for what, kw in bad:
        args = dict(rank=1, opt=ADAM, t=2)
        args.update(kw)
        l0 = capi.launch_count()
        rc = R.call(lib, **args)
        assert rc != 0, what
        assert "g2v_cbow_update_nvl" in lib.g2v_last_error().decode(), what
        assert capi.launch_count() == l0, what
    torch.cuda.synchronize()
    assert R.state() == before, "a refused call changed a buffer"
    R.step(env, ADAM, 2)                           # detached: the same calls now run
    torch.cuda.synchronize()
    assert_zero(R.g, "after detach")


# ------------------------------------------------------------------------------------------------ 2. a training step
@pytest.mark.parametrize("mode", ["dyadic", "realistic"])
@pytest.mark.parametrize("world", [2, 3, 5])
@pytest.mark.parametrize("V,D", [(999, 33), (1001, 128)])
def test_simulated_training_step_with_the_real_kernels(env, V, D, world, mode):
    """The training list dealt by shard_by_nnz; each simulated rank accumulates g2v_cbow_fwdbwd over its shard into its
    own [g_ih | g_ho] replica with inv_n = 1/len(list), from its own weight replica; then the `world` exchange calls.
    Two steps, nothing zeroed by hand.  Each step: every rank's gradient within its shard's float64 bound (so the
    exchange left no stale gradient behind), weights bit-identical to g2v_cbow_update on the float32 sum the exchange
    forms from those gradients, m / v slices likewise, every replica zeroed; after the first step the weights lie within
    the float64 bound of one full-list Step, whose gradient bound is the sum of the shard bounds plus the rounding of
    the world-term sum."""
    import torch
    from g2vec_b200.cbow import shard_by_nnz
    capi, lib = env["capi"], env["lib"]
    N = 1500
    rowptr, gene, label = helpers.random_windows(N, V, 0, 40, seed=world * 100 + D)
    lens = np.diff(rowptr).astype(np.int64)
    tr = np.random.RandomState(D + world).permutation(N)[:1200].astype(np.int64)
    if mode == "dyadic":
        Wi, Wo, _ = f64.dyadic_problem(rowptr, gene, V, D, seed=world)
    else:
        Wi, Wo = helpers.init_weights(V, D, world)
    k = V * D
    n = k + D
    W0 = np.concatenate([Wi.ravel(), Wo]).astype(F32)
    shards = [shard_by_nnz(tr, lens, world, r) for r in range(world)]
    assert sorted(np.concatenate(shards).tolist()) == sorted(tr.tolist())
    rp, ge, la = cu(rowptr), cu(gene), cu(label)
    sh = [cu(s.astype(np.int32)) for s in shards]
    inv_n = 1.0 / len(tr)
    R = Ranks(world, n)
    z = np.zeros(n, F32)
    R.load(W0, z, z)
    W, m, v = cu(W0), cu(z), cu(z)
    own = [torch.from_numpy(owned(n, world, r)).cuda() for r in range(world)]
    for t in (1, 2):
        what = "%s world=%d D=%d step %d" % (mode, world, D, t)
        Wt = R.w[0].cpu().numpy()
        Wt_ih, Wt_ho = Wt[:k].reshape(V, D), Wt[k:]
        assert_zero(R.g, what + " before the forward")
        count = 0
        for r in range(world):
            acc = torch.zeros(2, dtype=torch.int64, device="cuda")
            wr, gr = R.w[r].data_ptr(), R.g[r].data_ptr()
            capi.check(lib.g2v_cbow_fwdbwd(rp.data_ptr(), ge.data_ptr(), la.data_ptr(), sh[r].data_ptr(), 0,
                                           len(shards[r]), inv_n, wr, wr + 4 * k, gr, gr + 4 * k, acc.data_ptr(),
                                           acc.data_ptr() + 8, V, D, 0, stream()), "g2v_cbow_fwdbwd rank %d" % r)
            count += int(acc.cpu()[1])
        gs = [x.cpu().numpy().copy() for x in R.g]
        steps = [f64.Step(rowptr, gene, label, s, len(tr), Wt_ih, Wt_ho,
                          chain=f64.atomic_chain(len(s), env["sm"]) + 64) for s in shards]
        g64s, errs = [], []
        for r, S in enumerate(steps):
            g64s.append(np.concatenate([S.g_ih().ravel(), S.g_ho]))
            errs.append(np.concatenate([S.g_ih_err().ravel(), S.g_ho_err]))
            assert_within(gs[r], g64s[r], errs[r], what + " gradient of rank %d" % r)
        full = f64.Step(rowptr, gene, label, tr, len(tr), Wt_ih, Wt_ho)
        if mode == "dyadic" and t == 1:                 # the update leaves the weights no longer dyadic
            assert count == full.correct, (what, count, full.correct)
        else:
            lo, hi, _ = full.count_band()
            assert lo <= count <= hi, (what, count, lo, hi)
        R.step(env, ADAM, t)
        dense_update(env, V, D, W, m, v, cu(exchange_sum(gs, world)), ADAM, t)
        for p in range(world):
            assert_same(R.w[p], W, what + " weights of rank %d" % p)
            assert_same(R.m[p][own[p]], m[own[p]], what + " m slice of rank %d" % p)
            assert_same(R.v[p][own[p]], v[own[p]], what + " v slice of rank %d" % p)
        assert_zero(R.g, what + " after the exchange")
        if t == 1:
            g64 = np.concatenate([full.g_ih().ravel(), full.g_ho])
            err = (np.sum(errs, axis=0) + f64.gamma(world - 1) * np.sum([np.abs(a) + e for a, e in zip(g64s, errs)], 0)
                   + np.abs(g64 - np.sum(g64s, axis=0)))
            W1, dW = f64.adam64_first_step(W0, g64, err, LR)
            assert_within(R.w[0].cpu().numpy(), W1, dW, what + " weights vs the full-list float64 step")


# ------------------------------------------------------------------------------------------------ 3. the counters
VAL = [10, 12, 12, 11, 13, 9, 9, 9, 20, 20]     # validation offsets: rise, tie, drop, new best, 3 bad steps, more
BIG = 3 * 2 ** 32 + 5


def split_counts(total, world, rs):
    """`world` non-negative parts of `total` (parts above 2^32 when the total allows)."""
    cuts = np.sort(rs.randint(0, total + 1, size=world - 1, dtype=np.int64))
    return np.diff(np.concatenate([[0], cuts, [total]])).astype(np.int64)


@pytest.mark.parametrize("rule", ["decide", "best1", "best3"])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_counter_exchange_and_decision_on_the_summed_counters(env, world, rule):
    """Each step every rank sets acc[1..3] and calls g2v_cbow_loop_counters_nvl, then every rank decides with acc ==
    NULL.  Every rank's hist row holds the exact sums in slots 1..3 (above 2^32) and its own slot 0 untouched; every
    rank's ctl (and best) equals a single-rank loop driven by the summed acc; the stop step is the patience rule's.
    Once stopped, further counter and decide calls add and change nothing."""
    import torch
    lib, capi = env["lib"], env["capi"]
    K = 3 if rule == "best3" else 1
    T = len(VAL)
    rs = np.random.RandomState(world * 7 + K)
    totals = [[2 ** 33 + int(rs.randint(1000)), BIG + v, 2 ** 34 + int(rs.randint(1000))] for v in VAL]
    totals += [totals[-1], totals[-1]]                          # two more steps after max_steps
    parts = [[split_counts(x, world, rs) for x in row] for row in totals]
    i64 = lambda *shape: torch.zeros(*shape, dtype=torch.int64, device="cuda")
    ctl, acc, hist = [i64(8) for _ in range(world + 1)], [i64(6) for _ in range(world + 1)], []
    for r in range(world + 1):                                  # index `world`: the single-rank loop
        h = np.zeros((T + 2, 4), np.int64)
        h[:, 0] = -(1000 * r + np.arange(T + 2)) - 1            # slot 0 sentinels
        hist.append(cu(h))
        capi.check(lib.g2v_cbow_loop_init(ctl[r].data_ptr(), T, 1, stream()), "g2v_cbow_loop_init")
    best = [torch.tensor([K, -1, 0, 0], dtype=torch.int64, device="cuda") for _ in range(world + 1)]
    tab = torch.tensor([h.data_ptr() for h in hist[:world]], dtype=torch.int64, device="cuda")

    def decide(r, a):
        if rule == "decide":
            capi.check(lib.g2v_cbow_loop_decide(ctl[r].data_ptr(), a, hist[r].data_ptr(), stream()), "decide")
        else:
            capi.check(lib.g2v_cbow_loop_decide_best(ctl[r].data_ptr(), best[r].data_ptr(), a, hist[r].data_ptr(),
                                                     stream()), "decide_best")

    for s in range(T + 2):
        prev = [(c.cpu().numpy().copy(), b.cpu().numpy().copy(), h.cpu().numpy().copy())
                for c, b, h in zip(ctl, best, hist)]
        stopped = bool(prev[world][0][0])
        for r in range(world):
            acc[r].copy_(torch.tensor([-7] + [int(parts[s][j][r]) for j in range(3)] + [0, 0], dtype=torch.int64))
            capi.check(lib.g2v_cbow_loop_counters_nvl(ctl[r].data_ptr(), acc[r].data_ptr(), tab.data_ptr(), None,
                                                      world, stream()), "g2v_cbow_loop_counters_nvl")
        for r in range(world):
            decide(r, None)
        acc[world].copy_(torch.tensor([0] + totals[s] + [0, 0], dtype=torch.int64))
        decide(world, acc[world].data_ptr())
        c = [x.cpu().numpy() for x in ctl]
        b = [x.cpu().numpy() for x in best]
        h = [x.cpu().numpy() for x in hist]
        what = "world=%d %s step %d" % (world, rule, s)
        for r in range(world):
            assert (c[r] == c[world]).all(), (what, r, c[r], c[world])
            assert (b[r] == b[world]).all(), (what, r, b[r], b[world])
            if stopped:
                assert (h[r] == prev[r][2]).all(), (what, "a stopped loop's counters changed hist", r)
                assert (c[r] == prev[r][0]).all(), (what, r)
            else:
                assert h[r][s, 1:].tolist() == totals[s], (what, r, h[r][s], totals[s])
                assert h[r][s, 0] == prev[r][2][s, 0], (what, "slot 0 changed", r)
                assert (np.delete(h[r], s, axis=0) == np.delete(prev[r][2], s, axis=0)).all(), (what, r)
        if stopped and rule != "decide":
            assert b[world][3] == 0 and (b[world][:3] == prev[world][1][:3]).all(), what
    stop, best_step = patience_oracle.apply_rule([BIG + v for v in VAL], K, T)
    c = ctl[0].cpu().numpy()
    assert c[0] == 1 and c[2] == (-1 if stop is None else stop), (rule, c, stop)
    assert c[1] == (T if stop is None else stop + 1), (rule, c)
    if rule != "decide":
        assert best[0].cpu().numpy()[1] == best_step, (rule, best[0], best_step)
    assert stop is not None and any(VAL[i] == VAL[i - 1] for i in range(1, stop + 1))   # a tie before the stop
    assert K == 1 or stop >= K and all(VAL[i] < max(VAL[:stop - K + 1]) for i in range(stop - K + 1, stop + 1))


@pytest.mark.parametrize("world", [2, 3, 5])
def test_exchanged_validation_count_equals_one_pass_over_the_whole_list(env, world):
    """Each simulated rank adds g2v_cbow_eval over its validation shard into acc[2]; after the exchange and the decide
    every rank's history holds exactly the count of one g2v_cbow_eval over the whole list (each window is evaluated by
    the same code either way)."""
    import torch
    from g2vec_b200.cbow import shard_by_nnz
    lib, capi = env["lib"], env["capi"]
    N, V = 3000, 1001
    rowptr, gene, label = helpers.random_windows(N, V, 0, 40, seed=world)
    lens = np.diff(rowptr).astype(np.int64)
    va = np.random.RandomState(world).permutation(N)[:2000].astype(np.int64)
    rp, ge, la = cu(rowptr), cu(gene), cu(label)
    for D in (33, 128):
        Wi, Wo = helpers.init_weights(V, D, D)
        Wd, Wod = cu(Wi), cu(Wo)
        whole = torch.zeros(1, dtype=torch.int64, device="cuda")
        capi.check(lib.g2v_cbow_eval(rp.data_ptr(), ge.data_ptr(), la.data_ptr(), cu(va.astype(np.int32)).data_ptr(),
                                     0, len(va), Wd.data_ptr(), Wod.data_ptr(), whole.data_ptr(), V, D, 0, stream()),
                   "g2v_cbow_eval")
        ctl = [torch.zeros(8, dtype=torch.int64, device="cuda") for _ in range(world)]
        acc = [torch.zeros(6, dtype=torch.int64, device="cuda") for _ in range(world)]
        hist = [torch.zeros(4, dtype=torch.int64, device="cuda") for _ in range(world)]
        tab = torch.tensor([h.data_ptr() for h in hist], dtype=torch.int64, device="cuda")
        shards = [cu(shard_by_nnz(va, lens, world, r).astype(np.int32)) for r in range(world)]
        for r in range(world):
            capi.check(lib.g2v_cbow_loop_init(ctl[r].data_ptr(), 1, 1, stream()), "g2v_cbow_loop_init")
            capi.check(lib.g2v_cbow_eval(rp.data_ptr(), ge.data_ptr(), la.data_ptr(), shards[r].data_ptr(), 0,
                                         shards[r].numel(), Wd.data_ptr(), Wod.data_ptr(), acc[r].data_ptr() + 16, V,
                                         D, 0, stream()), "g2v_cbow_eval rank %d" % r)
            capi.check(lib.g2v_cbow_loop_counters_nvl(ctl[r].data_ptr(), acc[r].data_ptr(), tab.data_ptr(), None,
                                                      world, stream()), "g2v_cbow_loop_counters_nvl")
        for r in range(world):
            capi.check(lib.g2v_cbow_loop_decide(ctl[r].data_ptr(), None, hist[r].data_ptr(), stream()), "decide")
        want = int(whole.cpu()[0])
        assert 0 < want < len(va)
        for r in range(world):
            assert hist[r].cpu().tolist() == [0, 0, want, 0], (D, r, hist[r], want)
            assert int(ctl[r].cpu()[3]) == want, (D, r)


# ------------------------------------------------------------------------------------------------ 4. adam_tick
@pytest.mark.parametrize("lr", [0.005, 0.05])
def test_adam_tick_follows_tf1_float32_beta_powers(env, lr):
    """After t ticks from {1, 1, 0, 0} the state is {beta1^t, beta2^t, alpha_t, 0} of TF1's float32 beta-power
    variables (f64.adam_tf1_alpha's sequence), bit for bit, for every t <= 1000."""
    import torch
    T = 1000
    state = torch.tensor([1.0, 1.0, 0.0, 0.0], device="cuda")
    out = torch.zeros(T, 4, device="cuda")
    for t in range(T):
        env["capi"].check(env["lib"].g2v_cbow_adam_tick(state.data_ptr(), lr, B1, B2, stream()), "g2v_cbow_adam_tick")
        out[t].copy_(state)
    got = out.cpu().numpy()
    want = np.zeros((T, 4), F32)
    b1p, b2p = F32(1), F32(1)
    for t in range(T):
        b1p = F32(b1p * F32(B1)); b2p = F32(b2p * F32(B2))
        want[t, :3] = b1p, b2p, F32(F32(F32(lr) * np.sqrt(F32(F32(1) - b2p))) / F32(F32(1) - b1p))
    for t in list(range(1, 33)) + [100, 999, 1000]:
        assert want[t - 1, 2] == f64.adam_tf1_alpha(lr, t), t
    bad = np.nonzero((got.view(np.int32) != want.view(np.int32)).any(axis=1))[0]
    assert len(bad) == 0, "t=%d: got %r want %r" % (bad[0] + 1, got[bad[0]], want[bad[0]])
