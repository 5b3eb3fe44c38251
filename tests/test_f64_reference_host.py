"""The float64 CBOW reference and its per-element bounds (tests/f64_reference.py), checked on the CPU before the GPU tests
hold the kernels to them: the float32 oracle and a float32 numpy restatement satisfy every bound; the bounds are not
vacuous (one window or one gene less breaks them); dyadic inputs sum to the same float32 bits in any order."""
import numpy as np
import pytest

import oracle
from tests import f64_reference as f64

F32 = np.float32


def windows(V, lens, seed, pairs=True):
    """Windows of the given lengths over distinct random genes; with `pairs`, every 5th window of length 2 is a
    gene pair {2j, 2j + 1} (opposite rows in the dyadic weights: o == 0 exactly)."""
    rs = np.random.RandomState(seed)
    rows = []
    for i, l in enumerate(lens):
        if pairs and l == 2 and i % 5 == 0:
            j = 2 * rs.randint(0, min(V, 16) // 2)
            rows.append(np.array([j, j + 1]))
        else:
            rows.append(np.sort(rs.choice(V, size=l, replace=False)))
    rowptr = np.zeros(len(lens) + 1, np.int32); rowptr[1:] = np.cumsum(lens)
    gene = np.concatenate(rows).astype(np.int32) if len(rows) else np.zeros(0, np.int32)
    label = (rs.rand(len(lens)) < 0.5).astype(np.uint8)
    return rowptr, gene, label


def f32_forward(rowptr, gene, label, win, n_total, W, Who, reduce="sum"):
    """A float32 restatement (numpy's own summation order): per-position dO * scale, g_ih, g_ho, loss, count."""
    inv_n = F32(1) / F32(n_total)
    V, D = W.shape
    dOs = np.zeros(len(win), F32)
    g_ih = np.zeros((V, D), F32); g_ho = np.zeros(D, F32)
    loss, nc = 0.0, 0
    for i, n in enumerate(win):
        g = gene[rowptr[n]:rowptr[n + 1]]
        h = W[g].sum(0, dtype=F32) if len(g) else np.zeros(D, F32)
        sc = F32(1) / F32(len(g)) if (reduce == "mean" and len(g)) else F32(1)
        h = (h * sc).astype(F32)
        o = F32(np.dot(h, Who))
        y = F32(label[n])
        sig = F32(1) / (F32(1) + np.exp(-o, dtype=F32)) if o >= 0 else np.exp(o, dtype=F32) / (F32(1) + np.exp(o, dtype=F32))
        dO = F32(F32(sig - y) * inv_n)
        loss += float(F32(max(o, F32(0)) - o * y + np.log1p(np.exp(-abs(o), dtype=F32), dtype=F32)))
        nc += int((o > 0) == (y != 0))
        g_ho += (h * dO).astype(F32)
        s = F32(dO * sc)
        np.add.at(g_ih, g, (Who * s).astype(F32))
        dOs[i] = s
    return dOs, g_ih, g_ho, loss, nc


def check_step(ref, dOs, g_ih, g_ho, loss=None, nc=None, exact_count=False):
    assert (np.abs(dOs - ref.dO * ref.s) <= ref.dO_err * ref.s + f64.U * np.abs(ref.dO * ref.s)).all()
    assert (np.abs(g_ih - ref.g_ih()) <= ref.g_ih_err()).all()
    assert (np.abs(g_ho - ref.g_ho) <= ref.g_ho_err).all()
    if loss is not None:
        assert abs(loss - ref.loss_terms.sum()) <= ref.loss_err
    if nc is not None:
        lo, hi, _ = ref.count_band()
        assert (nc == ref.correct) if exact_count else (lo <= nc <= hi)


CASES = [(1, 4099, [0, 1, 2, 7, 8, 9, 81, 4096, 2, 2]), (3, 301, [0, 1, 2, 7, 8, 9, 81, 2, 2, 300]),
         (33, 1001, [1, 2, 7, 8, 9, 81, 1000, 0, 2]), (130, 257, [2, 0, 1, 81, 9, 8, 7, 2, 256])]


@pytest.mark.parametrize("D,V,lens", CASES)
def test_float32_oracle_satisfies_every_bound(D, V, lens):
    rs = np.random.RandomState(D)
    lens = list(lens) * 3
    rowptr, gene, label = windows(V, lens, seed=D)
    W = (np.clip(rs.randn(V, D), -2, 2) / np.sqrt(D)).astype(F32)
    Who = (np.clip(rs.randn(D), -2, 2) / np.sqrt(D)).astype(F32)
    N = len(lens)
    win = rs.permutation(N)
    g_ih, g_ho, loss, nc = oracle.cbow_grad(rowptr, gene, label, win, N + 5, W, Who)
    ref = f64.Step(rowptr, gene, label, win, N + 5, W, Who)
    assert (np.abs(g_ih - ref.g_ih()) <= ref.g_ih_err()).all()
    assert (np.abs(g_ho - ref.g_ho) <= ref.g_ho_err).all()
    assert abs(loss * (N + 5) - ref.loss_terms.sum()) <= ref.loss_err
    lo, hi, _ = ref.count_band()
    assert lo <= nc <= hi
    # per-position dO and the mean reduction through the float32 restatement
    for reduce in ("sum", "mean"):
        ref = f64.Step(rowptr, gene, label, win, N + 5, W, Who, reduce=reduce)
        check_step(ref, *f32_forward(rowptr, gene, label, win, N + 5, W, Who, reduce))


def test_bounds_are_not_vacuous():
    """One window less, or one gene less in one window, must break the per-element g_ih bound or the per-position dO
    bound: the bounds are far tighter than the effect of the smallest structural mistake."""
    D, V = 33, 501
    lens = [0, 1, 2, 7, 8, 9, 81] * 6
    rowptr, gene, label = windows(V, lens, seed=3)
    rs = np.random.RandomState(3)
    W = (np.clip(rs.randn(V, D), -2, 2) / np.sqrt(D)).astype(F32)
    Who = (np.clip(rs.randn(D), -2, 2) / np.sqrt(D)).astype(F32)
    N = len(lens)
    win = np.arange(N)
    ref = f64.Step(rowptr, gene, label, win, N, W, Who)
    for drop in (1, 5, 13, N - 1):                                    # one window less
        keep = np.delete(win, drop)
        g_ih, _, _, _ = oracle.cbow_grad(rowptr, gene, label, keep, N, W, Who)
        assert (np.abs(g_ih - ref.g_ih()) > ref.g_ih_err()).any(), drop
    for n in (1, 4, 6, 20):                                           # one gene less in window n
        b, e = rowptr[n], rowptr[n + 1]
        assert e > b
        gene2 = np.delete(gene, e - 1)
        rowptr2 = rowptr.copy(); rowptr2[n + 1:] -= 1
        dOs, g_ih, _, _, _ = f32_forward(rowptr2, gene2, label, win, N, W, Who)
        bad_dO = np.abs(dOs - ref.dO * ref.s) > ref.dO_err * ref.s + f64.U * np.abs(ref.dO * ref.s)
        bad_g = np.abs(g_ih - ref.g_ih()) > ref.g_ih_err()
        assert bad_dO[n] or bad_g.any(), n


@pytest.mark.parametrize("D,lmax", [(3631, 80), (3631, 4096), (1, 4096), (130, 1000), (1537, 9)])
def test_dyadic_sums_are_order_independent(D, lmax):
    rs = np.random.RandomState(D + lmax)
    V = max(lmax + 1, 64) | 1
    rowptr = np.array([0, lmax], np.int32)
    gene = np.sort(rs.choice(V, size=lmax, replace=False)).astype(np.int32)
    W, Who, a = f64.dyadic_problem(rowptr, gene, V, D, seed=1)
    rows = W[gene]
    want_h = rows.astype(np.float64).sum(0)
    want_o = float(want_h @ Who.astype(np.float64))
    for k in range(3):
        p = rs.permutation(lmax)
        h = np.zeros(D, F32)
        for j in p:                                                   # sequential float32 sum in a random order
            h += rows[j]
        assert (h.astype(np.float64) == want_h).all()
        terms = (h * Who).astype(F32)
        q = rs.permutation(D)
        o = F32(0)
        for j in q:
            o = F32(o + terms[j])
        assert float(o) == want_o
        assert float(terms.sum(dtype=F32)) == want_o                  # numpy's pairwise order too
    s = (W.astype(np.float64) @ Who.astype(np.float64))
    assert (s.astype(F32).astype(np.float64) == s).all()


def test_opposite_gene_pairs_give_exact_zero_logits():
    V, D = 257, 130
    rowptr = np.array([0, 2, 4, 4], np.int32); gene = np.array([0, 1, 6, 7], np.int32)
    W, Who, _ = f64.dyadic_problem(rowptr, gene, V, D, seed=2)
    ref = f64.Step(rowptr, gene, np.array([0, 1, 0], np.uint8), np.arange(3), 3, W, Who)
    assert (ref.o == 0).all() and ref.correct == 2                     # o > 0 is false: label 0 correct, label 1 not


@pytest.mark.parametrize("t", [1, 2, 1000])
def test_float32_adam_satisfies_the_adam_bound(t):
    rs = np.random.RandomState(t)
    n = 4099
    W = rs.randn(n).astype(F32)
    g = (rs.randn(n) * 10.0 ** rs.randint(-12, 1, n)).astype(F32)
    g[::7] = 0; g[1::11] = F32(1e-8); g[2::11] = -F32(3e-9)            # exact zeros, values near eps
    m = (rs.randn(n) * 1e-3).astype(F32) if t > 1 else np.zeros(n, F32)
    v = (rs.rand(n) * 1e-6).astype(F32) if t > 1 else np.zeros(n, F32)
    (W1, m1, v1), (dW, dm, dv) = f64.adam64(W, m, v, g, 0.005, t)
    Wc, mc, vc = W.copy(), m.copy(), v.copy()
    oracle.adam_(Wc, mc, vc, g.copy(), 0.005, t)
    assert (np.abs(Wc - W1) <= dW).all() and (np.abs(mc - m1) <= dm).all() and (np.abs(vc - v1) <= dv).all()
    # not vacuous: a step with the other t, or m updated with 1 - beta2, breaks it
    (W2, _, _), _ = f64.adam64(W, m, v, g, 0.005, t + 1)
    assert (np.abs(Wc - W2) > dW).any()
    mb = m + (g.astype(np.float64) - m) * float(F32(1) - F32(0.999))
    assert (np.abs(mb - m1) > dm).any()
    W3, dW3 = f64.sgd64(W, g, 0.5)
    Ws = W.copy(); oracle.sgd_(Ws, g, 0.5)
    assert (np.abs(Ws - W3) <= dW3).all()


def test_alpha_matches_the_kernels_float32_formula():
    b1p, b2p = F32(1), F32(1)
    for _ in range(1000):
        b1p *= F32(0.9); b2p *= F32(0.999)
    want = F32(0.005) * np.sqrt(F32(1) - b2p) / (F32(1) - b1p)
    assert f64.adam_tf1_alpha(0.005, 1000) == want


def test_dyadic_expansion_inputs_are_exact():
    rs = np.random.RandomState(0)
    V, n = 301, 2000
    rowptr, gene, label = windows(V, list(rs.randint(0, 40, n)), seed=0, pairs=False)
    cscptr, pos = f64.csc_of(rowptr, gene, np.arange(n), V)
    k_max = int(np.diff(cscptr).max())
    dO = f64.dyadic_dO(n, k_max, 64, seed=1)
    c = f64.grad_c_exact(cscptr, pos, dO)
    vals = dO[pos]
    for k in range(2):
        p = rs.permutation(len(pos))
        acc = np.zeros(V, F32)
        seg = np.repeat(np.arange(V), np.diff(cscptr))
        for j in p:
            acc[seg[j]] = F32(acc[seg[j]] + vals[j])
        assert (acc.astype(np.float64) == c).all()
