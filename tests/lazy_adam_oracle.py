"""CPU restatement of the lazy (touched-row) TF1 Adam step and of a mini-batch training loop with it -- test
infrastructure for tests/test_gpu_cbow_lazy.py and tests/test_lazy_adam_host.py.

``lazy_adam_`` is tf.contrib.opt.LazyAdamOptimizer's sparse apply on the rows an embedding lookup gathered: gather
those rows of var, m and v, take one TF1 ApplyAdam step on them (``oracle.adam_``, the same arithmetic as the dense
step), scatter them back; every other row is left as it is.
"""
import numpy as np

import oracle


def lazy_adam_(var, m, v, g, rows, lr, t, beta1=0.9, beta2=0.999, eps=1e-8):
    """In place on the float32 [V, D] arrays var, m, v; g = dense gradient [V, D] (only its ``rows`` are read)."""
    rows = np.unique(np.asarray(rows, dtype=np.int64))
    sub = [np.ascontiguousarray(a[rows]) for a in (var, m, v, g)]
    oracle.adam_(sub[0], sub[1], sub[2], sub[3], lr, t, beta1, beta2, eps)
    var[rows], m[rows], v[rows] = sub[0], sub[1], sub[2]


def touched(rowptr, gene, win):
    """The distinct genes of the listed windows (what an embedding lookup of the batch gathers)."""
    parts = [gene[rowptr[n]:rowptr[n + 1]] for n in win]
    return np.unique(np.concatenate(parts)) if parts else np.zeros(0, np.int64)


def mean_grad(rowptr, gene, label, win, n_total, W0, Wo0):
    """Gradient of the segmented-MEAN model over the listed windows (float64 restatement), as float32."""
    V, D = W0.shape
    g_ih, g_ho = np.zeros((V, D)), np.zeros(D)
    for n in win:
        gs = gene[rowptr[n]:rowptr[n + 1]]
        scale = 1.0 / len(gs) if len(gs) else 1.0
        h = W0[gs].astype(np.float64).sum(0) * scale
        dO = (1 / (1 + np.exp(-float(h @ Wo0))) - label[n]) / n_total
        g_ho += h * dO
        np.add.at(g_ih, gs, dO * scale * Wo0)
    return g_ih.astype(np.float32), g_ho.astype(np.float32)


def lazy_step(rowptr, gene, label, win, W, Wo, state, lr, t, reduce="sum"):
    """One lazy_adam step over the batch ``win`` (loss mean over the batch); state = [m_ih, v_ih, m_ho, v_ho]."""
    if reduce == "sum":
        g_ih, g_ho, _, _ = oracle.cbow_grad(rowptr, gene, label, win, len(win), W, Wo)
    else:
        g_ih, g_ho = mean_grad(rowptr, gene, label, win, len(win), W, Wo)
    lazy_adam_(W, state[0], state[1], g_ih, touched(rowptr, gene, win), lr, t)
    oracle.adam_(Wo, state[2], state[3], np.ascontiguousarray(g_ho, dtype=np.float32), lr, t)


def lazy_minibatch_train(rowptr, gene, label, tr, W0, Wo0, lr, batch, epochs):
    """``epochs`` passes over consecutive batches of the training list ``tr`` with lazy_step; returns (W_ih, W_ho)."""
    W, Wo = W0.copy(), Wo0.copy()
    st = [np.zeros_like(W), np.zeros_like(W), np.zeros_like(Wo), np.zeros_like(Wo)]
    t = 0
    for _ in range(epochs):
        for lo in range(0, len(tr), batch):
            t += 1
            lazy_step(rowptr, gene, label, tr[lo:lo + batch], W, Wo, st, lr, t)
    return W, Wo
