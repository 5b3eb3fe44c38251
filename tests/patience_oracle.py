"""CPU restatement of the full-batch training loop with early stopping by patience (DESIGN.md §4.15) -- test
infrastructure for tests/test_patience_host.py and tests/test_gpu_cbow_patience.py.

``cbow_train`` is ``oracle.cbow_train`` (G2Vec.py:259-286: one full-batch step, then the validation and the training
accuracy at the updated weights) with the patience rule in place of the reference's strict-drop break: a step whose
correct validation count is >= the best so far becomes the best (ties: the later step) and its W_ih is kept; the
``patience``-th step in a row below the best stops the loop.  With patience 1 it is ``oracle.cbow_train``'s rule.
"""
import numpy as np

import oracle


def cbow_train(rowptr, gene, label, tr, va, W_ih0, W_ho0, lr, max_steps=500, patience=1, optimizer="adam"):
    """Returns (W_ih of the best step, history [(step, acc_val, acc_tr)], stop step or None, best step)."""
    W_ih = np.array(W_ih0, dtype=np.float32, copy=True)
    W_ho = np.array(W_ho0, dtype=np.float32, copy=True).reshape(-1)
    m_ih = np.zeros_like(W_ih); v_ih = np.zeros_like(W_ih)
    m_ho = np.zeros_like(W_ho); v_ho = np.zeros_like(W_ho)
    f32 = np.float32
    hist, result, stop = [], W_ih.copy(), None
    best_val, best_step, bad = -1, None, 0
    for step in range(max_steps):
        g_ih, g_ho, _, _ = oracle.cbow_grad(rowptr, gene, label, tr, len(tr), W_ih, W_ho)
        if optimizer == "adam":
            oracle.adam_(W_ih, m_ih, v_ih, g_ih, lr, step + 1)
            oracle.adam_(W_ho, m_ho, v_ho, g_ho, lr, step + 1)
        else:
            oracle.sgd_(W_ih, g_ih, lr); oracle.sgd_(W_ho, g_ho, lr)
        n_val = oracle.cbow_eval(rowptr, gene, label, va, W_ih, W_ho)
        n_tr = oracle.cbow_eval(rowptr, gene, label, tr, W_ih, W_ho)
        hist.append((step, float(f32(n_val) / f32(max(len(va), 1))), float(f32(n_tr) / f32(max(len(tr), 1)))))
        if n_val >= best_val:
            best_val, best_step, bad = n_val, step, 0
            result = W_ih.copy()
        else:
            bad += 1
            if bad >= patience:
                stop = step
                break
    return result, hist, stop, best_step


def apply_rule(val_counts, patience, max_steps=None):
    """The rule on a trajectory of correct validation counts: (stop step or None, best step)."""
    best_val, best_step, bad = -1, None, 0
    for step, v in enumerate(val_counts[:max_steps]):
        if v >= best_val:
            best_val, best_step, bad = v, step, 0
        else:
            bad += 1
            if bad >= patience:
                return step, best_step
    return None, best_step
