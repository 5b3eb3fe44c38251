"""Float64 trainer with decoupled weight decay (DESIGN.md §4.18) -- test infrastructure for
tests/test_weight_decay_host.py and tests/test_gpu_cbow_weight_decay.py.

``train64`` is AdamW / SGDW / lazy AdamW on the CBOW model in float64, as TF1's DecoupledWeightDecayExtension applies
them: on every optimizer step the gradient is taken at the weights before the step, then every element the step
updates is decayed, w -= λ w (λ = float32(weight_decay)), then the Adam / SGD step runs on the decayed value with m and
v untouched by the decay.  The forward and gradient are those of tests/lr_plateau_oracle.adam64_train (loss sum over
a batch's windows divided by its size), so at λ = 0 the Adam trainer is adam64_train.  A rate per step, as
adam64_train takes it; λ is not scaled by it.
"""
import numpy as np

from tests import f64_reference

F32 = np.float32


def decay_factor(weight_decay, t):
    """(1 - λ)^t in float64 with λ the float32 value the kernels use: where a row with zero gradient and zero moments
    ends after t Adam steps (in float32: within t roundings of it)."""
    return (1.0 - float(F32(weight_decay))) ** t


def train64(rowptr, gene, label, lists, W_ih0, W_ho0, step_rates, weight_decay=0.0, batch=0, optimizer="adam",
            beta1=0.9, beta2=0.999, eps=1e-8):
    """Epoch e trains on the window list ``lists[e]`` at rate ``step_rates[e]``: one full-batch step (``batch`` <= 0)
    or one step per consecutive batch of ``batch`` windows.  ``optimizer``: "adam" and "sgd" decay and update all of
    W_ih and W_ho every step; "lazy_adam" decays and updates only the rows of W_ih the batch gathered (each once) and
    all of W_ho.  Returns (W_ih, W_ho) in float64."""
    lam = float(F32(weight_decay))
    W = np.asarray(W_ih0, np.float32).astype(np.float64)
    Wo = np.asarray(W_ho0, np.float32).reshape(-1).astype(np.float64)
    V = W.shape[0]
    m, v, mo, vo = np.zeros_like(W), np.zeros_like(W), np.zeros_like(Wo), np.zeros_like(Wo)
    y_all = np.asarray(label, np.float64)
    t = 0
    for win, lr in zip(lists, step_rates):
        win = np.asarray(win, np.int64)
        B = len(win) if batch <= 0 else batch
        for lo in range(0, len(win), B):
            sub = win[lo:lo + B]
            X, _ = f64_reference.incidence(rowptr, gene, sub, V)
            o = X @ (W @ Wo)
            dO = (f64_reference.sigmoid64(o) - y_all[sub]) / len(sub)
            c = X.T @ dO
            g, go = np.outer(c, Wo), W.T @ c             # at the weights before the step
            t += 1
            rows = np.unique(X.indices) if optimizer == "lazy_adam" else slice(None)
            W[rows] -= lam * W[rows]
            Wo -= lam * Wo
            if optimizer == "sgd":
                W -= float(lr) * g
                Wo -= float(lr) * go
                continue
            alpha = float(lr) * np.sqrt(1.0 - beta2 ** t) / (1.0 - beta1 ** t)
            m[rows] = beta1 * m[rows] + (1 - beta1) * g[rows]
            v[rows] = beta2 * v[rows] + (1 - beta2) * g[rows] ** 2
            W[rows] -= alpha * m[rows] / (np.sqrt(v[rows]) + eps)
            mo = beta1 * mo + (1 - beta1) * go
            vo = beta2 * vo + (1 - beta2) * go ** 2
            Wo -= alpha * mo / (np.sqrt(vo) + eps)
    return W, Wo


def decay32(w, weight_decay, steps=1):
    """The kernels' decay fl(w - fl(λ w)) in float32, iterated ``steps`` times."""
    w = np.asarray(w, np.float32).copy()
    lam = F32(weight_decay)
    for _ in range(steps):
        w = (w - (lam * w).astype(F32)).astype(F32)
    return w
