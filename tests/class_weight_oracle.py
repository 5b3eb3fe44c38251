"""Class weights of the training loss (DESIGN.md §4.20) -- test infrastructure for tests/test_class_weight_host.py and
tests/test_gpu_cbow_class_weight.py.

``do32`` restates the kernels' rounding of one window's weighted dO and loss term in NumPy float32:
    dO = fl(fl(fl(sigmoid(o) - y) * inv_n) * w_y),   loss term = fl(w_y * l).
``WeightedStep`` is tests/f64_reference.Step with every window's dO and loss term multiplied by w_y in float64, and
the bounds widened by that factor plus the one extra rounding of each product.  ``train64`` is the float64 trainer of
tests/weight_decay_oracle.train64 (λ = 0) with the weighted gradient, for the loop tests.
"""
import numpy as np

from tests import f64_reference as f64

F32 = np.float32
U = f64.U


def weights_of(label, cw):
    """w_{y_n} per window (float64 of the float32 weights)."""
    w0, w1 = (float(F32(w)) for w in cw)
    return np.where(np.asarray(label) != 0, w1, w0).astype(np.float64)


def balanced(labels):
    """sklearn's compute_class_weight("balanced") on a label array, as float32 values."""
    y = np.asarray(labels).reshape(-1) != 0
    n, n1 = y.shape[0], int(y.sum())
    return float(F32(n / (2.0 * (n - n1)))), float(F32(n / (2.0 * n1)))


def sigmoid32(o):
    """sigmoid_stable of the kernels in float32 (expf and the division correctly rounded here; the kernels' expf is
    within 2 ulp, so callers compare to a few ulps, not bits)."""
    o = np.asarray(o, F32)
    z = np.exp(-np.abs(o)).astype(F32)
    one = F32(1)
    return np.where(o >= 0, one / (one + z), z / (one + z)).astype(F32)


def do32(o, y, inv_n, cw):
    """(dO, loss term) of windows with float32 logits o and labels y, rounded as the weighted kernels round them."""
    o = np.asarray(o, F32)
    y = np.asarray(y, F32)
    w = np.where(y != 0, F32(cw[1]), F32(cw[0])).astype(F32)
    d = (sigmoid32(o) - y).astype(F32)
    d = (d * F32(inv_n)).astype(F32)
    dO = (d * w).astype(F32)
    l = (np.maximum(o, F32(0)) - o * y + np.log1p(np.exp(-np.abs(o)))).astype(F32)
    return dO, (w * l).astype(F32)


class WeightedStep(f64.Step):
    """f64.Step with class weights cw = (w0, w1): dO_n and the loss terms times w_{y_n}; c, g_ho and the bounds
    recomputed from them (each weighted dO and loss term carries one more rounding, u |value|)."""

    def __init__(self, rowptr, gene, label, win, n_total, W_ih, W_ho, cw, reduce="sum", chain=None):
        super().__init__(rowptr, gene, label, win, n_total, W_ih, W_ho, reduce=reduce, chain=chain)
        w = weights_of(np.asarray(label)[np.asarray(win, np.int64)], cw)
        self.w = w
        X = self.X
        self.dO = self.dO * w
        self.loss_terms = self.loss_terms * w
        self.dO_err = self.dO_err * w + U * np.abs(self.dO)
        self.c = X.T @ (self.dO * self.s)
        Wih = np.asarray(W_ih, np.float32).astype(np.float64)
        self.g_ho = Wih.T @ self.c
        self.c_err = X.T @ (self.s * (self.dO_err + U * np.abs(self.dO))) + f64.gamma(self.k_g + 2) * (
            X.T @ (self.s * np.abs(self.dO)))
        lens, chain = self.lens, self.chain
        self.g_ho_err = np.abs(Wih).T @ (X.T @ (self.s * (self.dO_err + (f64.gamma(lens + 4) + f64.gamma(chain + 1)
                                                                         + 2 * U) * np.abs(self.dO))))
        self.g_ho_err = self.g_ho_err + U * np.abs(self.g_ho)
        self.loss_err = float((w * (self.o_err + 6 * U * (np.abs(self.o) + 1))).sum()
                              + (f64.gamma(chain + 1) + U) * self.loss_terms.sum()) + 1e-300


def train64(rowptr, gene, label, lists, W_ih0, W_ho0, step_rates, cw, batch=0, optimizer="adam", beta1=0.9,
            beta2=0.999, eps=1e-8):
    """Epoch e trains on ``lists[e]`` at ``step_rates[e]``: one full-batch step (``batch`` <= 0) or one per consecutive
    batch.  The loss of a batch of N windows is (1/N) sum w_{y_n} l_n (sum reduce).  "adam", "sgd" and "lazy_adam"
    (the batch's rows of W_ih, all of W_ho) as tests/weight_decay_oracle.train64.  Returns (W_ih, W_ho) in float64."""
    W = np.asarray(W_ih0, np.float32).astype(np.float64)
    Wo = np.asarray(W_ho0, np.float32).reshape(-1).astype(np.float64)
    V = W.shape[0]
    m, v, mo, vo = np.zeros_like(W), np.zeros_like(W), np.zeros_like(Wo), np.zeros_like(Wo)
    y_all = np.asarray(label, np.float64)
    w_all = weights_of(label, cw)
    t = 0
    for win, lr in zip(lists, step_rates):
        win = np.asarray(win, np.int64)
        B = len(win) if batch <= 0 else batch
        for lo in range(0, len(win), B):
            sub = win[lo:lo + B]
            X, _ = f64.incidence(rowptr, gene, sub, V)
            o = X @ (W @ Wo)
            dO = (f64.sigmoid64(o) - y_all[sub]) / len(sub) * w_all[sub]
            c = X.T @ dO
            g, go = np.outer(c, Wo), W.T @ c
            t += 1
            if optimizer == "sgd":
                W -= float(lr) * g
                Wo -= float(lr) * go
                continue
            rows = np.unique(X.indices) if optimizer == "lazy_adam" else slice(None)
            alpha = float(lr) * np.sqrt(1.0 - beta2 ** t) / (1.0 - beta1 ** t)
            m[rows] = beta1 * m[rows] + (1 - beta1) * g[rows]
            v[rows] = beta2 * v[rows] + (1 - beta2) * g[rows] ** 2
            W[rows] -= alpha * m[rows] / (np.sqrt(v[rows]) + eps)
            mo = beta1 * mo + (1 - beta1) * go
            vo = beta2 * vo + (1 - beta2) * go ** 2
            Wo -= alpha * mo / (np.sqrt(vo) + eps)
    return W, Wo
