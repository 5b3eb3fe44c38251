"""CPU restatement of the validation-loss monitor (DESIGN.md §4.19) -- test infrastructure for
tests/test_val_loss_host.py and tests/test_gpu_cbow_val_loss.py.

* ``q_terms`` / ``Q``: the fixed-point loss of every window, q_n = rint(min(l_n, 64) 2^24) with
  l_n = max(z,0) - z y + log1p(exp(-|z|)) in float64 (64 for a z that is not finite).
* ``logits64``: the collapsed logit z_n = scale_n sum_{g in n} s[g] in float64 from s = W_ih W_ho in float64.
* ``logits32``: the same logit as g2v_cbow_val_loss computes it from a given float32 s: lane k of 8 adds
  s[g_k], s[g_{k+8}], ... in float32, the 8 partials are combined by the xor tree 4, 2, 1, then scaled.
* ``apply_rule`` / ``rates``: early stopping and reduce-on-plateau on a Q trajectory, as the score 2^62 - Q.
* ``cbow_train``: the full-batch loop of oracle.cbow_train (oracle.cbow_grad + oracle.adam_) deciding on Q.
"""
import numpy as np

import oracle
from tests import lr_plateau_oracle

CAP, UNIT, TOP = 64.0, float(1 << 24), 1 << 62


def q_terms(z, y):
    """int64 q_n of float logits z (any float dtype) and 0/1 labels y."""
    z = np.asarray(z, np.float64)
    y = np.asarray(y, np.float64)
    fin = np.isfinite(z)
    zf = np.where(fin, z, 0.0)
    with np.errstate(over="ignore"):
        l = np.maximum(zf, 0.0) - zf * y + np.log1p(np.exp(-np.abs(zf)))
    l = np.where(fin, np.minimum(l, CAP), CAP)
    return np.rint(l * UNIT).astype(np.int64)


def _lists(rowptr, win):
    rowptr = np.asarray(rowptr, np.int64)
    win = np.asarray(win, np.int64)
    return rowptr[win], rowptr[win + 1]


def logits64(rowptr, gene, win, W_ih, W_ho, reduce="sum"):
    s = np.asarray(W_ih, np.float32).astype(np.float64) @ np.asarray(W_ho, np.float32).reshape(-1).astype(np.float64)
    b, e = _lists(rowptr, win)
    gene = np.asarray(gene, np.int64)
    z = np.array([s[gene[bb:ee]].sum() for bb, ee in zip(b, e)], dtype=np.float64)
    if reduce == "mean":
        z = np.where(e > b, z / np.maximum(e - b, 1), z)
    return z


def logits32(rowptr, gene, win, s, reduce="sum"):
    """The float32 logits g2v_cbow_val_loss forms from the float32 s (one value per gene)."""
    s = np.asarray(s, np.float32)
    gene = np.asarray(gene, np.int64)
    b, e = _lists(rowptr, win)
    f = np.float32
    out = np.empty(len(b), dtype=np.float32)
    for i, (bb, ee) in enumerate(zip(b, e)):
        p = [f(0)] * 8
        for k in range(8):
            for j in range(bb + k, ee, 8):
                p[k] = f(p[k] + s[gene[j]])
        a = [f(p[k] + p[k ^ 4]) for k in range(8)]
        a = [f(a[k] + a[k ^ 2]) for k in range(8)]
        z = f(a[0] + a[1])
        if reduce == "mean" and ee > bb:
            z = f(z * (f(1) / f(ee - bb)))
        out[i] = z
    return out


def Q(rowptr, gene, label, win, W_ih, W_ho, reduce="sum"):
    """Q of the list from the float64 collapsed logits (a Python int)."""
    z = logits64(rowptr, gene, win, W_ih, W_ho, reduce)
    return int(q_terms(z, np.asarray(label)[np.asarray(win, np.int64)]).sum())


def mean_loss(Qv, n_val):
    return int(Qv) / (max(int(n_val), 1) << 24)


def apply_rule(Qs, patience):
    """Early stopping on a Q trajectory: (stop step or None, best step); Q <= best is the new best (ties: later)."""
    best, best_step, bad = None, None, 0
    for step, q in enumerate(Qs):
        if best is None or q <= best:
            best, best_step, bad = q, step, 0
        else:
            bad += 1
            if bad >= patience:
                return step, best_step
    return None, best_step


def rates(Qs, lr, patience, factor=0.1, min_lr=0.0):
    """Reduce-on-plateau on a Q trajectory: lr_plateau_oracle.rates on the scores 2^62 - Q (a tie is no improvement)."""
    return lr_plateau_oracle.rates([TOP - int(q) for q in Qs], lr, patience, factor, min_lr)


def cbow_train(rowptr, gene, label, tr, va, W_ih0, W_ho0, lr, max_steps=500, patience=1):
    """Full-batch Adam (oracle.cbow_grad / oracle.adam_ in float32) stopped by the loss rule.  Returns (W_ih of the best
    step, history [(step, acc_val, acc_tr)], Q per step, stop step or None, best step)."""
    W_ih = np.array(W_ih0, dtype=np.float32, copy=True)
    W_ho = np.array(W_ho0, dtype=np.float32, copy=True).reshape(-1)
    m_ih, v_ih = np.zeros_like(W_ih), np.zeros_like(W_ih)
    m_ho, v_ho = np.zeros_like(W_ho), np.zeros_like(W_ho)
    f32 = np.float32
    hist, Qs, result, stop = [], [], W_ih.copy(), None
    best, best_step, bad = None, None, 0
    for step in range(max_steps):
        g_ih, g_ho, _, _ = oracle.cbow_grad(rowptr, gene, label, tr, len(tr), W_ih, W_ho)
        oracle.adam_(W_ih, m_ih, v_ih, g_ih, lr, step + 1)
        oracle.adam_(W_ho, m_ho, v_ho, g_ho, lr, step + 1)
        n_val = oracle.cbow_eval(rowptr, gene, label, va, W_ih, W_ho)
        n_tr = oracle.cbow_eval(rowptr, gene, label, tr, W_ih, W_ho)
        hist.append((step, float(f32(n_val) / f32(max(len(va), 1))), float(f32(n_tr) / f32(max(len(tr), 1)))))
        q = Q(rowptr, gene, label, va, W_ih, W_ho)
        Qs.append(q)
        if best is None or q <= best:
            best, best_step, bad = q, step, 0
            result = W_ih.copy()
        else:
            bad += 1
            if bad >= patience:
                stop = step
                break
    return result, hist, Qs, stop, best_step
