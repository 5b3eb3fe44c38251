"""CPU restatements for reshuffled mini-batch epochs (DESIGN.md §4.12) -- test infrastructure for
tests/test_reshuffle_host.py and tests/test_gpu_cbow_reshuffle.py:

* ``perm(seed, epoch, n)``: the epoch permutation P, vectorised NumPy (Philox4x32-10 rounds in uint64 arithmetic);
* ``epoch_list``: one rank's share of the epoch's list, tr[P(rank + i*world)];
* ``batch_plan_torch``: the torch.sort construction of the per-batch transposed incidence that CbowModel.prepare_batches
  used before g2v_cbow_batch_plan (the builder must give the same arrays, bit for bit);
* the oracle training loops of tests/lazy_adam_oracle.py and of the dense mini-batch test, fed one order per epoch.
"""
import numpy as np

import oracle
from tests import lazy_adam_oracle

DOMAIN = 0x53480000
_M = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on arrays of counters (broadcast), uint32 words out: the arithmetic of oracle.philox4x32_10."""
    c = [np.asarray(x, dtype=np.uint64) & _M for x in (c0, c1, c2, c3)]
    c = np.broadcast_arrays(*c)
    c = [x.copy() for x in c]
    k = [np.uint64(int(k0) & 0xFFFFFFFF), np.uint64(int(k1) & 0xFFFFFFFF)]
    for r in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k[0]) & _M, p1 & _M, ((p0 >> np.uint64(32)) ^ c[3] ^ k[1]) & _M, p0 & _M]
        k = [(k[0] + np.uint64(0x9E3779B9)) & _M, (k[1] + np.uint64(0xBB67AE85)) & _M]
    return [x.astype(np.uint32) for x in c]


def half_bits(n):
    b = 2
    while b < 32 and (1 << b) < n:
        b += 2
    return b // 2


def feistel(x, h, seed, epoch, n):
    mask = np.uint64((1 << h) - 1)
    x = np.asarray(x, dtype=np.uint64)
    L, R = x >> np.uint64(h), x & mask
    for r in range(4):
        w0 = philox4x32_10(R, DOMAIN | r, epoch, n, seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)[0]
        L, R = R, L ^ (w0.astype(np.uint64) & mask)
    return (L << np.uint64(h)) | R


def perm_at(i, seed, epoch, n):
    """P(seed, epoch, n) at the positions i: Feistel, cycle-walked back into [0, n)."""
    h = half_bits(n)
    y = feistel(i, h, seed, epoch, n)
    out = y >= np.uint64(n)
    while out.any():
        y[out] = feistel(y[out], h, seed, epoch, n)
        out = y >= np.uint64(n)
    return y.astype(np.int64)


def perm(seed, epoch, n):
    return perm_at(np.arange(n, dtype=np.uint64), seed, epoch, n)


def epoch_list(tr, seed, epoch, rank=0, world=1):
    n = len(tr)
    return np.asarray(tr)[perm_at(np.arange(rank, n, world, dtype=np.uint64), seed, epoch, n)]


def epoch_orders(tr, seed, epochs):
    """The lists train_cbow(reshuffle=True) trains on: the split's order, then tr[P(seed, e)] for e >= 1."""
    tr = np.asarray(tr)
    return [tr] + [epoch_list(tr, seed, e) for e in range(1, epochs)]


def batch_plan_torch(rowptr, gene, V, win, B):
    """The former CbowModel.prepare_batches: one stable sort of (batch, gene) keys.  rowptr, gene, win: int32 device
    tensors.  Returns (rows, segptr, pos, batch_rowptr) as NumPy int32."""
    import torch
    dev = win.device
    n = int(win.shape[0])
    B = min(int(B), n) if B > 0 else n
    w = win.to(torch.int64)
    starts = rowptr[w].to(torch.int64)
    lens = rowptr[w + 1].to(torch.int64) - starts
    total = int(lens.sum())
    pos = torch.repeat_interleave(torch.arange(n, device=dev), lens)
    first = torch.cumsum(lens, 0) - lens
    idx = starts[pos] + (torch.arange(total, device=dev) - first[pos])
    b = pos // B
    key, order = torch.sort(b * V + gene[idx].to(torch.int64), stable=True)
    rel = (pos - b * B)[order].to(torch.int32)
    head = torch.ones(total, dtype=torch.bool, device=dev)
    head[1:] = key[1:] != key[:-1]
    seg = torch.nonzero(head).squeeze(1)
    rows = (key[seg] % V).to(torch.int32)
    segptr = torch.cat([seg, torch.tensor([total], device=dev)]).to(torch.int32)
    n_b = -(-n // B)
    per = torch.bincount(key[seg] // V, minlength=n_b).cpu().numpy()
    brp = np.concatenate([[0], np.cumsum(per)]).astype(np.int32)
    return rows.cpu().numpy(), segptr.cpu().numpy(), rel.cpu().numpy(), brp


def lazy_minibatch_train_orders(rowptr, gene, label, orders, W0, Wo0, lr, batch):
    """lazy_adam_oracle.lazy_minibatch_train with one list per epoch (``orders[e]`` for epoch e)."""
    W, Wo = W0.copy(), Wo0.copy()
    st = [np.zeros_like(W), np.zeros_like(W), np.zeros_like(Wo), np.zeros_like(Wo)]
    t = 0
    for tr in orders:
        for lo in range(0, len(tr), batch):
            t += 1
            lazy_adam_oracle.lazy_step(rowptr, gene, label, tr[lo:lo + batch], W, Wo, st, lr, t)
    return W, Wo


def dense_minibatch_train_orders(rowptr, gene, label, orders, W0, Wo0, lr, batch, optimizer="adam"):
    """The oracle loop of the dense mini-batch test (sum-reduced batch gradient, TF1 Adam or SGD on every row), with
    one list per epoch."""
    W, Wo = W0.copy(), Wo0.copy()
    st = [np.zeros_like(W), np.zeros_like(W), np.zeros_like(Wo), np.zeros_like(Wo)]
    t = 0
    for tr in orders:
        for lo in range(0, len(tr), batch):
            sub = tr[lo:lo + batch]
            g_ih, g_ho, _, _ = oracle.cbow_grad(rowptr, gene, label, sub, len(sub), W, Wo)
            t += 1
            if optimizer == "adam":
                oracle.adam_(W, st[0], st[1], g_ih, lr, t); oracle.adam_(Wo, st[2], st[3], g_ho, lr, t)
            else:
                oracle.sgd_(W, g_ih, lr); oracle.sgd_(Wo, g_ho, lr)
    return W, Wo
