"""The error bound of the certified accuracy pass (DESIGN.md §4.16), on the CPU: tau, restated in numpy float32 the way
certified_tau computes it, covers |o32 - o64| + |o'32 - o64| -- the row-gather logit and the collapsed logit, each
evaluated in float32 in the kernels' summation orders, against the exact value -- on random, near-zero,
huge-magnitude and subnormal-product inputs, and on subnormal mean-scaled h against a large W_ho, for sum and mean.

The float32 model rounds every product before adding it.  The kernels are compiled with nvcc's default --fmad=true,
so some of their `a * b + c` are one FFMA, one rounding instead of two: the model takes at least as many roundings on
every term's path as the kernels do, and is a case that the bound must cover, not the kernels' exact bits."""
import math

import numpy as np
import pytest

F32 = np.float32
INF = F32(np.inf)


def tau(T, scale, l, D, A):
    """certified_tau of g2v_cbow.cu, in float32 (A: the float32 sum_d |W_ho[d]|)."""
    k = l + D + 16
    if not (T <= F32(2.0 ** 126)) or k > (1 << 22):
        return INF
    with np.errstate(over="ignore", under="ignore"):
        rel = F32(F32(F32(k) * F32(2.0 ** -21)) * scale)
        abs_ = F32(F32(F32((l + 3) * D) + A) * F32(2.0 ** -145))
        return F32(F32(rel * T) + abs_)


def warp_tree(parts, width):
    """Butterfly (xor-shuffle) sum over `width` lanes, as warp_sum / the 8-lane reduction: every lane ends with the
    same value; lane 0's is returned."""
    p = [F32(x) for x in parts]
    o = width // 2
    while o:
        p = [F32(p[i] + p[i ^ o]) for i in range(width)]
        o //= 2
    return p[0]


def lane_dot(a, b, absval=False):
    """<a, b> with lane L summing d = L, L + 32, ... in order, then warp_sum (the summation order of
    r1_prepare_kernel and of the generic rows kernel; each product rounded on its own, see the module docstring)."""
    parts = []
    for L in range(32):
        s = F32(0)
        for d in range(L, len(a), 32):
            p = F32(a[d] * b[d])
            s = F32(s + (abs(p) if absval else p))
        parts.append(s)
    return warp_tree(parts, 32)


def logits(W, Who, genes, mean):
    """(o32, o'32, tau, o64) of one window."""
    l, D = len(genes), W.shape[1]
    scale = F32(F32(1) / F32(l)) if (mean and l) else F32(1)
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        h = np.zeros(D, F32)
        for g in genes:                                     # rows gather: genes in order
            h = (h + W[g]).astype(F32)
        if mean:
            h = (h * scale).astype(F32)
        o32 = lane_dot(h, Who)
        s = {g: lane_dot(W[g], Who) for g in set(genes)}
        t = {g: lane_dot(W[g], Who, absval=True) for g in set(genes)}
        ps, pt = [], []
        for sub in range(8):                                # 8 lanes per window
            a, b = F32(0), F32(0)
            for j in range(sub, l, 8):
                a = F32(a + s[genes[j]]); b = F32(b + t[genes[j]])
            ps.append(a); pt.append(b)
        o1 = F32(warp_tree(ps, 8) * scale)
        T = warp_tree(pt, 8)
        A = lane_dot(np.ones(D, F32), Who, absval=True)
    exact = math.fsum(float(W[g, d]) * float(Who[d]) for g in genes for d in range(D)) * float(scale)
    return o32, o1, tau(T, scale, l, D, A), exact


def case(kind, D, seed):
    rs = np.random.RandomState(seed)
    V = 40
    W = (rs.randn(V, D) / np.sqrt(D)).astype(F32)
    Who = (rs.randn(D) / np.sqrt(D)).astype(F32)
    windows = [list(rs.choice(V, size=rs.randint(1, 30), replace=False)) for _ in range(12)]
    if kind == "near_zero":                                 # last gene's row = minus the float32 running sum
        for w in windows:
            if len(w) > 1:
                run = np.zeros(D, F32)
                for g in w[:-1]:
                    run = (run + W[g]).astype(F32)
                W[w[-1]] = -run
    elif kind == "huge":
        W = (W * F32(1e14)).astype(F32); Who = (Who * F32(1e14)).astype(F32)
    elif kind == "subnormal":                               # products around 2^-140 .. 2^-150
        W = (W * F32(2.0 ** -70)).astype(F32); Who = (Who * F32(2.0 ** -72)).astype(F32)
    elif kind == "subnormal_h":                             # subnormal h (and scale * h) against a large W_ho
        W = (W * F32(2.0 ** -146)).astype(F32); Who = (Who * F32(2.0 ** 100)).astype(F32)
    return W, Who, windows + [[rs.randint(V)] * 3]          # plus a window listing one gene three times


@pytest.mark.parametrize("mean", [False, True])
@pytest.mark.parametrize("D", [1, 7, 33, 128])
@pytest.mark.parametrize("kind", ["random", "near_zero", "huge", "subnormal", "subnormal_h"])
def test_tau_covers_both_float32_logits(kind, D, mean):
    W, Who, windows = case(kind, D, seed=D * 3 + len(kind))
    finite = 0
    for genes in windows:
        o32, o1, t, exact = logits(W, Who, genes, mean)
        assert np.isfinite(o32) and np.isfinite(o1)
        if not np.isfinite(t):
            continue
        finite += 1
        err = abs(float(o32) - exact) + abs(float(o1) - exact)
        assert float(t) >= err, (kind, D, mean, genes, float(t), err)
        if float(abs(o1)) > float(t):                       # a decided window: o has o' 's sign
            assert (o32 > 0) == (o1 > 0) and o32 != 0
    assert finite == len(windows)


def underflow_window(D):
    """A mean window {0, 1} whose scale * h[0] = 1.5 * 2^-149 rounds to 2^-148 and is then multiplied by W_ho[0] =
    2^100: the row gather's o is +2^-51 while the exact logit (and o') is -2^-51.  Columns beyond 2 are zero."""
    W = np.zeros((2, D), F32)
    W[0, :2] = [2.0 ** -149, -3.5 * 2.0 ** -49]
    W[1, 0] = 2.0 ** -148
    Who = np.zeros(D, F32)
    Who[:2] = [2.0 ** 100, 1.0]
    return W, Who


@pytest.mark.parametrize("D", [2, 128])
def test_an_underflowing_mean_scale_times_a_large_w_ho_is_not_decided(D):
    W, Who = underflow_window(D)
    o32, o1, t, exact = logits(W, Who, [0, 1], mean=True)
    assert o32 == F32(2.0 ** -51) and o1 == F32(-2.0 ** -51) and exact == -2.0 ** -51
    assert float(t) >= abs(float(o32) - exact) + abs(float(o1) - exact)
    assert not abs(o1) > t                                  # the window is gathered


def test_empty_and_non_finite_inputs_are_never_decided():
    assert float(tau(F32(0), F32(1), 0, 128, F32(0))) > 0   # an empty window: o' = 0 is not > tau
    assert tau(F32(np.inf), F32(1), 5, 128, F32(1)) == INF
    assert tau(F32(2.0 ** 127), F32(1), 5, 128, F32(1)) == INF      # too close to overflow
    assert tau(F32(1), F32(1), (1 << 22), 128, F32(1)) == INF      # too many roundings for the gamma bound
    assert tau(F32(1), F32(1), 5, 128, INF) == INF          # sum |W_ho| overflowed
    for t in (tau(F32(np.nan), F32(1), 5, 128, F32(1)), tau(F32(1), F32(1), 5, 128, F32(np.nan))):
        assert not (F32(1e30) > t)                          # NaN: the comparison fails, the window is gathered
