"""Float64 restatement of one CBOW step, with a worst-case float32 error bound for every output element.

The float32 oracle (oracle/g2v_oracle.c) rounds the way the kernels do, so comparing against it needs aggregate
tolerances.  This module states the same operations in float64 (numpy + scipy.sparse, so that D = 3631 with 20k
windows takes seconds) and bounds, per element, how far ANY float32 evaluation order of the kernels may lie from it:

    u = 2^-24,  gamma_k = k u / (1 - k u)                    (a sum of k + 1 float32 terms, in any order, is within
                                                              gamma_k * (sum of their magnitudes) of the exact sum)
    o_n      |d o_n|    <= gamma_{l_n + D + 4} * s_n * sum_d |W_ho[d]| sum_{g in n} |W_ih[g, d]|
    dO_n     |d dO_n|   <= inv_n (|d o_n| / 4 + 4u) + 2u |dO_n|        (sigma' <= 1/4; a few ulps of sigma, not of
                                                                         dO: sigma - y cancels when y = 1, o >> 0)
    c_g      |d c_g|    <= sum_{n ni g} s_n (|d dO_n| + u |dO_n|) + gamma_{k_g + 2} sum_{n ni g} s_n |dO_n|
    g_ih     |d g[g,d]| <= |W_ho[d]| |d c_g| + u |g64[g, d]|
    g_ho, loss: the same with the number of float32 terms one accumulator chain adds (`chain`).

s_n is the window's scale (1, or 1/l_n for the mean), inv_n the float32 1/N the kernels receive, and the float64
values are computed from the same float32 inputs.  Dyadic inputs (``dyadic_problem``) make every float32 sum of the
forward exact in every order, so the correct count must equal the float64 count exactly."""
import numpy as np
import scipy.sparse as sp

U = 2.0 ** -24
F32 = np.float32


def gamma(k):
    k = np.asarray(k, dtype=np.float64)
    return k * U / (1.0 - k * U)


def incidence(rowptr, gene, win, V):
    """X [len(win), V] float64 CSR: X[i, g] = how often gene g occurs in window win[i] (a repeated gene counts twice,
    as the gather adds its row twice)."""
    rowptr = np.asarray(rowptr, np.int64); gene = np.asarray(gene, np.int64); win = np.asarray(win, np.int64)
    lens = rowptr[win + 1] - rowptr[win]
    ptr = np.zeros(len(win) + 1, np.int64); ptr[1:] = np.cumsum(lens)
    first = np.repeat(rowptr[win], lens) + (np.arange(ptr[-1]) - np.repeat(ptr[:-1], lens))
    X = sp.csr_matrix((np.ones(ptr[-1]), gene[first], ptr), shape=(len(win), V))
    X.sum_duplicates()
    return X, lens


def csc_of(rowptr, gene, win, V):
    """The transposed incidence the CSC backward reads: cscptr [V + 1], pos (list positions, ascending per gene)."""
    rowptr = np.asarray(rowptr, np.int64); win = np.asarray(win, np.int64)
    lens = rowptr[win + 1] - rowptr[win]
    ptr = np.zeros(len(win) + 1, np.int64); ptr[1:] = np.cumsum(lens)
    first = np.repeat(rowptr[win], lens) + (np.arange(ptr[-1]) - np.repeat(ptr[:-1], lens))
    g = np.asarray(gene, np.int64)[first]
    pos = np.repeat(np.arange(len(win)), lens)
    order = np.argsort(g, kind="stable")
    cscptr = np.zeros(V + 1, np.int64); cscptr[1:] = np.cumsum(np.bincount(g, minlength=V))
    return cscptr.astype(np.int32), pos[order].astype(np.int32)


def sigmoid64(o):
    o = np.asarray(o, np.float64)
    z = np.exp(-np.abs(o))
    return np.where(o >= 0, 1.0 / (1.0 + z), z / (1.0 + z))


def adam_tf1_alpha(lr, t, beta1=0.9, beta2=0.999):
    """alpha_t with beta^t by repeated float32 multiplication, as TF1's beta*_power variables (and the kernels)."""
    b1p, b2p = F32(1), F32(1)
    for _ in range(t):
        b1p = F32(b1p * F32(beta1)); b2p = F32(b2p * F32(beta2))
    return F32(F32(F32(lr) * np.sqrt(F32(F32(1) - b2p))) / F32(F32(1) - b1p))


class Step:
    """Float64 forward/backward of the windows win (list positions 0..n-1) and the per-element bounds.

    chain: the number of float32 terms one accumulator chain of the g_ho / loss reduction adds (per-warp partial,
    CTA sum, global sum); ``atomic_chain`` / ``det_chain`` give the kernels' values."""

    def __init__(self, rowptr, gene, label, win, n_total, W_ih, W_ho, reduce="sum", chain=None):
        W = np.asarray(W_ih, np.float32).astype(np.float64)
        Who = np.asarray(W_ho, np.float32).reshape(-1).astype(np.float64)
        V, D = W.shape
        self.V, self.D = V, D
        win = np.asarray(win, np.int64)
        X, lens = incidence(rowptr, gene, win, V)
        self.X, self.lens = X, lens
        y = np.asarray(label, np.float64)[win]
        self.y = y
        mean = reduce == "mean"
        self.s = np.where(mean & (lens > 0), 1.0 / np.maximum(lens, 1), 1.0)
        self.inv_n = float(F32(1.0) / F32(n_total))
        self.s64 = W @ Who                                        # rank-1 s = W_ih . W_ho
        self.o = (X @ self.s64) * self.s
        sig = sigmoid64(self.o)
        self.dO = (sig - y) * self.inv_n
        self.loss_terms = np.maximum(self.o, 0) - self.o * y + np.log1p(np.exp(-np.abs(self.o)))
        self.correct = int(((self.o > 0) == (y != 0)).sum())
        self.c = X.T @ (self.dO * self.s)                          # per-gene sum of dO * scale
        self.g_ho = W.T @ self.c                                   # = sum_n h_n dO_n
        # ---- bounds
        absW, absWho = np.abs(W), np.abs(Who)
        self.s_abs = absW @ absWho
        lmax = int(lens.max()) if len(lens) else 0
        self.o_err = gamma(lens + D + 4) * self.s * (X @ self.s_abs)
        self.dO_err = self.inv_n * (self.o_err / 4 + 4 * U) + 2 * U * np.abs(self.dO)
        k_g = np.asarray(X.sum(axis=0)).ravel()
        self.k_g = k_g
        self.c_err = X.T @ (self.s * (self.dO_err + U * np.abs(self.dO))) + gamma(k_g + 2) * (X.T @ (self.s * np.abs(self.dO)))
        chain = len(win) + 8 if chain is None else chain
        self.chain = chain
        self.g_ho_err = absW.T @ (X.T @ (self.s * (self.dO_err + (gamma(lens + 4) + gamma(chain + 1) + 2 * U)
                                                   * np.abs(self.dO)))) + U * np.abs(self.g_ho)
        self.loss_err = float((self.o_err + 6 * U * (np.abs(self.o) + 1)).sum()
                              + gamma(chain + 1) * self.loss_terms.sum()) + 1e-300
        self.s_err = gamma(D + 1) * self.s_abs
        self.lmax = lmax
        self.Who = Who

    def g_ih(self):
        return np.outer(self.c, self.Who)

    def g_ih_err(self):
        return np.outer(self.c_err, np.abs(self.Who)) + U * np.abs(self.g_ih())

    def ambiguous(self):
        """Windows whose predicate o > 0 a float32 evaluation may decide either way (an empty window's o is 0 in any
        arithmetic)."""
        return (np.abs(self.o) <= self.o_err) & (self.o_err > 0)

    def count_band(self):
        amb = self.ambiguous()
        ok = (self.o > 0) == (self.y != 0)
        return int((ok & ~amb).sum()), int((ok | amb).sum()), int(amb.sum())


def atomic_chain(n_win, sm_count, occupancy=8, warps=8):
    """Terms of the longest accumulator chain of an atomic forward: a warp's windows, its CTA's warps, the CTAs."""
    return -(-n_win // (warps * sm_count)) + warps + sm_count * occupancy


def det_chain(n_win, tile=64, warps=8, sum_warps=32):
    """The deterministic forward: 8 windows per warp and tile, 8 warps, the tiles (32 interleaved slices + 32)."""
    n_tiles = -(-n_win // tile)
    return tile // warps + warps + -(-n_tiles // sum_warps) + sum_warps


def _segment_sums(cscptr, vals):
    """Per-segment float64 sums, each segment summed on its own (a running sum over all segments would lose the low
    bits of a small segment that follows large ones)."""
    cscptr = np.asarray(cscptr, np.int64)
    out = np.zeros(len(cscptr) - 1)
    nonempty = np.diff(cscptr) > 0
    if nonempty.any():
        out[nonempty] = np.add.reduceat(vals, cscptr[:-1][nonempty])
    return out


def grad_c_exact(cscptr, pos, dO):
    """c[g] = sum of dO over the gene's CSC segment in float64 (exact for dyadic dO, within a float64 rounding of the
    exact sum otherwise: ``c_bound`` includes it)."""
    vals = np.asarray(dO, np.float32).astype(np.float64)[np.asarray(pos, np.int64)]
    return _segment_sums(cscptr, vals)


def c_bound(cscptr, pos, dO):
    """Any float32 order of the segment sums: |c32 - c64| <= gamma_k * sum |dO| (plus the float64 sum's own rounding)."""
    k = np.diff(np.asarray(cscptr, np.int64))
    vals = np.abs(np.asarray(dO, np.float32).astype(np.float64))[np.asarray(pos, np.int64)]
    return (gamma(k + 1) + 2.0 ** -53 * (k + 1)) * _segment_sums(cscptr, vals)


# ------------------------------------------------------------------------------------------------ optimizers
def adam64(W, m, v, g, lr, t, beta1=0.9, beta2=0.999, eps=1e-8):
    """TF1 ApplyAdam in float64 on float32 inputs (alpha, 1 - beta and eps as the float32 values the kernels use).
    Returns (W', m', v') in float64 and their per-element bounds (dW, dm, dv)."""
    f = lambda a: np.asarray(a, np.float32).astype(np.float64)
    W, m, v, g = f(W), f(m), f(v), f(g)
    alpha = float(adam_tf1_alpha(lr, t, beta1, beta2))
    omb1, omb2 = float(F32(1) - F32(beta1)), float(F32(1) - F32(beta2))
    e = float(F32(eps))
    m1 = m + (g - m) * omb1
    v1 = v + (g * g - v) * omb2
    den = np.sqrt(v1) + e
    step = m1 * alpha / den
    W1 = W - step
    dm = 3 * U * (np.abs(m) + np.abs((g - m) * omb1))           # m' may cancel: absolute, from its two terms
    dv = 4 * U * v1                                              # v' = v (1 - omb2) + g^2 omb2: both terms >= 0
    dW = U * np.abs(W1) + 8 * U * np.abs(step) + alpha * dm / den
    return (W1, m1, v1), (dW, dm, dv)


def adam64_first_step(W, g, g_err, lr, beta1=0.9, beta2=0.999, eps=1e-8):
    """The first TF1 Adam step (t = 1, m = v = 0) when the float32 gradient is only known within g +- g_err (the
    gradient bound of a Step).  From a zero state the step alpha*omb1*g / (sqrt(omb2)|g| + eps) is odd and increasing
    in g, so its deviation over the interval is largest at an end point.  Returns (W' float64, per-element bound)."""
    g = np.asarray(g, np.float64); g_err = np.asarray(g_err, np.float64)
    z = np.zeros(np.shape(W), np.float32)
    (W1, _, _), (dW, _, _) = adam64(W, z, z, g.astype(np.float32), lr, 1, beta1, beta2, eps)
    alpha = float(adam_tf1_alpha(lr, 1, beta1, beta2))
    omb1, omb2, e = float(F32(1) - F32(beta1)), float(F32(1) - F32(beta2)), float(F32(eps))
    step = lambda x: alpha * omb1 * x / (np.sqrt(omb2) * np.abs(x) + e)
    gf = g.astype(np.float32).astype(np.float64)                  # adam64 ran on the float32 rounding of g
    s0 = step(gf)
    spread = np.maximum(np.abs(step(g + g_err) - s0), np.abs(step(g - g_err) - s0))
    return W1, dW + spread


def sgd64(W, g, lr):
    f = lambda a: np.asarray(a, np.float32).astype(np.float64)
    W, g = f(W), f(g)
    step = float(F32(lr)) * g
    W1 = W - step
    return W1, 2 * U * (np.abs(W1) + np.abs(step))


# ------------------------------------------------------------------------------------------------ dyadic inputs
def dyadic_problem(rowptr, gene, V, D, seed, reduce="sum"):
    """Weights that are small integers times a power of two, the integer range chosen from the shape so that every
    partial sum of h, of o = h . W_ho and of s = W_ih . W_ho stays below 2^24 quanta: every float32 sum of the forward
    is then exact in any order.  Gene pairs (2j, 2j + 1) of the first 16 genes have opposite rows, so a window
    {2j, 2j + 1} has o == 0 exactly.  Returns (W_ih, W_ho) float32."""
    lens = np.diff(np.asarray(rowptr, np.int64))
    lmax = max(1, int(lens.max()) if len(lens) else 1)
    budget = 2 ** 24 - 1
    a = 1
    while (2 * a + 1) ** 2 * lmax * D <= budget and a < 64:   # |h_d| <= lmax A, |o| partial <= D lmax A B (A = B = a)
        a = 2 * a + 1
    assert a * a * lmax * D <= budget, "shape (lmax=%d, D=%d) has no dyadic budget" % (lmax, D)
    rs = np.random.RandomState(seed)
    Wi = rs.randint(-a, a + 1, size=(V, D)).astype(np.float64)
    Wo = rs.randint(-a, a + 1, size=D).astype(np.float64)
    Wo[Wo == 0] = 1
    for j in range(0, min(V, 16) - 1, 2):
        Wi[j + 1] = -Wi[j]
    W_ih = (Wi * 2.0 ** -8).astype(np.float32)
    W_ho = (Wo * 2.0 ** -6).astype(np.float32)
    # the budget, checked on the actual values: largest magnitude sums in quanta
    assert np.abs(Wi).max() * lmax <= budget and np.abs(Wi).max() * np.abs(Wo).max() * lmax * D <= budget
    assert (W_ih.astype(np.float64) * 2 ** 8 == Wi).all() and (W_ho.astype(np.float64) * 2 ** 6 == Wo).all()
    if reduce == "mean":
        assert all(l == 0 or (l & (l - 1)) == 0 for l in lens), "dyadic mean needs power-of-two window lengths"
    return W_ih, W_ho, a


def dyadic_dO(n, k_max, B, seed, quantum=2.0 ** -20):
    """Test-chosen per-position dO (float32) whose per-gene sums c and products c * W_ho are exact in float32: integers
    in [-C, C] times `quantum` with k_max * C * B < 2^24 (B: the largest |W_ho| in its own quanta)."""
    C = max(1, min(4095, (2 ** 24 - 1) // max(1, k_max * B)))
    assert k_max * C * B < 2 ** 24
    rs = np.random.RandomState(seed)
    return (rs.randint(-C, C + 1, size=n) * quantum).astype(np.float32)
