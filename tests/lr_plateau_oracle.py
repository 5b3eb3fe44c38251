"""CPU restatement of the reduce-on-plateau learning rate (DESIGN.md §4.17) and a float64 Adam trainer that takes a
per-step rate -- test infrastructure for tests/test_lr_plateau_host.py and tests/test_gpu_cbow_lr_plateau.py.

``rates`` is Keras ReduceLROnPlateau(mode="max", min_delta=0, cooldown=0) on integer validation counts, in float32 as
g2v_cbow_lr_plateau computes it.  ``adam64_train`` is TF1 Adam on the CBOW model in float64 (the forward and the
gradient of tests/f64_reference.py, kept in float64 between steps), with alpha_t = lr_s sqrt(1 - beta2^t) / (1 - beta1^t):
a rate that changes between steps leaves m and v as they are, as TF1 does when its learning rate is a variable.
"""
import numpy as np

from tests import f64_reference

F32 = np.float32


def rates(val_counts, lr, patience, factor=0.1, min_lr=0.0):
    """The rule on a sequence of correct validation counts: (the float32 rate each step trained with, the steps whose
    decision cut the rate, the rate after the last decision)."""
    lr, factor, min_lr = F32(lr), F32(factor), F32(min_lr)
    best, wait = -1, 0
    used, cuts = [], []
    for s, v in enumerate(val_counts):
        used.append(lr)
        v = int(v)
        if v > best:                             # strict: a tie is not an improvement
            best, wait = v, 0
            continue
        wait += 1
        if wait >= patience:
            if lr > min_lr:
                lr = max(F32(lr * factor), min_lr)
                cuts.append(s)
            wait = 0
    return used, cuts, lr


def val_counts(info):
    """The correct validation counts of a train_cbow run, from its history (ACC[val] = float32(count) / n_val)."""
    n_va = max(info["n_val"], 1)
    return [int(np.rint(float(h[1]) * n_va)) for h in info["history"]]


def adam64_train(rowptr, gene, label, lists, W_ih0, W_ho0, step_rates, batch=0, lazy=False, beta1=0.9, beta2=0.999,
                 eps=1e-8):
    """Epoch e trains on the window list ``lists[e]`` at rate ``step_rates[e]``: one full-batch step (``batch`` <= 0)
    or one step per consecutive batch of ``batch`` windows, loss sum over the batch's windows divided by its size.
    ``lazy``: W_ih, m and v change only on the rows of the genes the batch gathered (TF1 LazyAdam).  Returns (W_ih,
    W_ho) in float64."""
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
            g, go = np.outer(c, Wo), W.T @ c
            t += 1
            alpha = float(lr) * np.sqrt(1.0 - beta2 ** t) / (1.0 - beta1 ** t)
            rows = np.unique(X.indices) if lazy else slice(None)
            m[rows] = beta1 * m[rows] + (1 - beta1) * g[rows]
            v[rows] = beta2 * v[rows] + (1 - beta2) * g[rows] ** 2
            W[rows] -= alpha * m[rows] / (np.sqrt(v[rows]) + eps)
            mo = beta1 * mo + (1 - beta1) * go
            vo = beta2 * vo + (1 - beta2) * go ** 2
            Wo -= alpha * mo / (np.sqrt(vo) + eps)
    return W, Wo
