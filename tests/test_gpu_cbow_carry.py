"""The device loop's carried forward (g2v_cbow_loop_tail): on one GPU with the CSC backward, a step's
training-accuracy pass is also the next step's forward -- it stores dO, the g_ho partial, the loss and the count, and
the next step's g2v_cbow_fwdbwd_csc only expands dO into g_ih.  Checked against the same kernels run without a loop."""
import numpy as np
import pytest

from tests import helpers

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def g2v():
    import torch
    assert torch.cuda.is_available()
    import g2vec_b200
    return g2vec_b200


def rel_max(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def setup(g2v, D, seed=3, W=None):
    """A rows/Adam model over random windows with its training list CSC-prepared, as train_cbow builds it."""
    import torch
    from g2vec_b200 import cbow
    V, N = 500, 4000
    rowptr, gene, label = helpers.random_windows(N, V - 20, 1, 60, seed=seed)     # 20 genes in no window
    W0, Wo0 = helpers.init_weights(V, D, seed) if W is None else W
    tr, va = cbow.split_indices(N, seed)
    tr_d = torch.from_numpy(tr.astype(np.int32)).cuda()
    va_d = torch.from_numpy(va.astype(np.int32)).cuda()
    m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005)
    m.prepare_csc(tr_d)
    return m, tr_d, va_d


def host_step(m, tr_d, va_d):
    """One iteration of the reference loop with no loop attached: what the parent commit's DeviceLoop launched."""
    import torch
    m.acc.zero_()
    m.fwdbwd(tr_d, len(tr_d)); m.update(); m.evaluate(va_d, 2); m.evaluate(tr_d, 3)
    torch.cuda.synchronize()
    return [int(x) for x in m.acc.cpu()[1:4]]


@pytest.mark.parametrize("D", [128, 100])
def test_tail_pass_writes_the_records_dO_as_the_next_forward_bit_for_bit(g2v, D):
    import torch
    from g2vec_b200 import cbow
    m, tr_d, va_d = setup(g2v, D)
    n = len(tr_d)
    loop = cbow.DeviceLoop(m, None, tr_d, va_d, n, 10, False, snapshot=False)
    assert loop.carried
    loop.attach()
    try:
        loop.one(True)
        torch.cuda.synchronize()
    finally:
        loop.detach()
    acc = m.acc.cpu()
    dO_tail = m.prepared(tr_d).dO.clone()
    # the same weights, a fresh model, the full CSC forward + expansion with no loop attached
    r, r_tr, _ = setup(g2v, D, W=(m.W_ih.cpu().numpy(), m.W_ho.cpu().numpy()))
    assert r.route(r_tr) == "csc" and torch.equal(r_tr, tr_d)
    r.fwdbwd(r_tr, n)
    r.evaluate(r_tr, 3)
    torch.cuda.synchronize()
    racc = r.acc.cpu()
    assert torch.equal(dO_tail, r.prepared(r_tr).dO)
    assert int(acc[3]) == int(acc[5]) == int(racc[1]) == int(racc[3])
    assert abs(m.loss_sum(acc[4:]) - r.loss_sum(racc)) <= 1e-9 * abs(r.loss_sum(racc))
    assert rel_max(m.g_ho.cpu().numpy(), r.g_ho.cpu().numpy()) < 1e-5
    # the next step's fwdbwd: forward skipped on the device, expansion of the carried dO -- the same g_ih bits
    loop.attach()
    try:
        m.fwdbwd(tr_d, n)
        torch.cuda.synchronize()
    finally:
        loop.detach()
    assert torch.equal(m.g_ih, r.g_ih)


def test_pending_carry_skips_the_forward_and_feeds_the_records_expansion(g2v):
    import torch
    from g2vec_b200 import cbow
    m, tr_d, va_d = setup(g2v, 128, seed=5)
    n = len(tr_d)
    loop = cbow.DeviceLoop(m, None, tr_d, va_d, n, 10, False, snapshot=False)
    loop.attach()
    try:
        loop.one(True)
        torch.cuda.synchronize()
        dO = m.prepared(tr_d).dO
        dO[7] = 1000.0                                     # poisoned: a forward would overwrite it
        want_dO = dO.clone()
        acc0, g_ho0 = m.acc.clone(), m.g_ho.clone()
        m.fwdbwd(tr_d, n)
        torch.cuda.synchronize()
    finally:
        loop.detach()
    assert torch.equal(dO, want_dO)
    assert torch.equal(m.acc, acc0) and torch.equal(m.g_ho, g_ho0)   # no loss, count or g_ho added
    cscptr, pos = m.prepared(tr_d).cscptr.long(), m.prepared(tr_d).pos.long()
    seg = torch.repeat_interleave(torch.arange(m.V, device="cuda"), cscptr[1:] - cscptr[:-1])
    c = torch.zeros(m.V, dtype=torch.float64, device="cuda").index_add_(0, seg, want_dO[pos].double())
    want = (c[:, None] * m.W_ho.double()[None, :]).cpu().numpy()
    assert rel_max(m.g_ih.double().cpu().numpy(), want) < 1e-5
    g = int(m.gene[m.rowptr[tr_d[7].long()]])            # a gene of the poisoned window carries the poison
    assert abs(float(c[g])) > 100.0


def test_reset_drops_the_pending_carry(g2v):
    """Steps, reset(), more steps: the same counters and weights as the host-driven steps -- g_ho of the dropped
    tail is not added twice, and the first step after reset() runs the full forward."""
    import torch
    from g2vec_b200 import cbow
    m, tr_d, va_d = setup(g2v, 128, seed=7)
    h, _, _ = setup(g2v, 128, seed=7)
    n = len(tr_d)
    host = [host_step(h, tr_d, va_d) for _ in range(5)]
    loop = cbow.DeviceLoop(m, None, tr_d, va_d, n, 10, False, snapshot=False)
    loop.attach()
    try:
        for _ in range(2):
            loop.one(True)
        loop.reset()
        assert float(m.g_ho.abs().max()) == 0.0 and int(m.acc[4:].abs().max()) == 0
        for _ in range(3):
            loop.one(True)
        loop.fetch()
        torch.cuda.synchronize()
    finally:
        loop.detach()
    hist = loop.hist_pin.view(-1, 4)[:3, 1:].tolist()
    for got, want in zip(hist, host[2:]):
        assert all(abs(a - b) <= 2 for a, b in zip(got, want)), (hist, host[2:])
    # g_ho's unordered atomics stay below 1e-4 (the bound of the other vector tests); a g_ho added twice does not
    assert rel_max(m.W_ho.cpu().numpy(), h.W_ho.cpu().numpy()) < 1e-4
    assert rel_max(m.W_ih.cpu().numpy(), h.W_ih.cpu().numpy()) < 1e-5


def test_graph_captured_after_reset_equals_eager_steps(g2v):
    """bench.py's pattern: eager steps, reset(), capture one step, replay.  The first replay has no carry pending
    and must run the full forward; later replays consume the carry."""
    import torch
    from g2vec_b200 import cbow
    a, tr_d, va_d = setup(g2v, 256, seed=11)
    b, _, _ = setup(g2v, 256, seed=11)
    n = len(tr_d)
    la = cbow.DeviceLoop(a, None, tr_d, va_d, n, 20, False, snapshot=False)
    lb = cbow.DeviceLoop(b, None, tr_d, va_d, n, 20, False, snapshot=False)
    for lp in (la, lb):
        lp.attach()
        try:
            for _ in range(2):
                lp.one(True)
            lp.reset()
            if lp is la:
                g = lp.capture([True])
                for _ in range(6):
                    g.replay()
            else:
                for _ in range(6):
                    lp.one(True)
                lp.fetch()
            torch.cuda.synchronize()
        finally:
            lp.detach()
    ha, hb = la.hist_pin.view(-1, 4)[:6].tolist(), lb.hist_pin.view(-1, 4)[:6].tolist()
    assert ha[0][1] > 0                                   # the first replay counted its own full forward
    for x, y in zip(ha, hb):
        assert all(abs(p - q) <= 2 for p, q in zip(x[1:], y[1:])), (ha, hb)
    for x, y in zip(ha[1:], ha[:-1]):
        assert x[1] == y[3]                               # acc[1] of step s is ACC[tr] of step s-1, exactly
    # g_ho's atomics differ between the two runs; Adam magnifies that noise on near-zero W_ho components
    assert rel_max(a.W_ih.cpu().numpy(), b.W_ih.cpu().numpy()) < 1e-5
    assert rel_max(a.W_ho.cpu().numpy(), b.W_ho.cpu().numpy()) < 1e-4


@pytest.mark.parametrize("det", [False, True])
def test_preparing_another_list_leaves_the_loop_step_unchanged(g2v, det):
    """A loop built on tr_d, then prepare_csc of a longer list: the loop's steps still run tr_d's CSC forward, carry
    and tail, so two steps count, carry and expand what the same steps without that prepare do."""
    import torch
    from g2vec_b200 import cbow
    V, N, D = 500, 4000, 128
    rowptr, gene, label = helpers.random_windows(N, V - 20, 1, 60, seed=13)
    W0, Wo0 = helpers.init_weights(V, D, 13)
    tr, va = cbow.split_indices(N, 13)
    tr_d = torch.from_numpy(tr.astype(np.int32)).cuda()
    va_d = torch.from_numpy(va.astype(np.int32)).cuda()
    other = torch.cat([tr_d, va_d])
    n = len(tr_d)
    out = []
    for extra in (True, False):
        m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005, deterministic=det)
        m.prepare_csc(tr_d)
        loop = cbow.DeviceLoop(m, None, tr_d, va_d, n, 10, False, snapshot=False)
        assert loop.carried
        if extra:
            m.prepare_csc(other)
            assert m.route(tr_d) == ("csc_det" if det else "csc") and m.prepared(tr_d).n == n
        loop.attach()
        try:
            for _ in range(2):
                loop.one(True)
            loop.fetch()
            m.fwdbwd(tr_d, n)                              # the third step's expansion of the carried dO
            torch.cuda.synchronize()
        finally:
            loop.detach()
        out.append((loop.hist_pin.view(-1, 4)[:2, 1:].tolist(), m.g_ih.cpu().numpy(), m.W_ih.cpu().numpy()))
    (h1, g1, w1), (h2, g2, w2) = out
    if det:
        assert h1 == h2 and g1.tobytes() == g2.tobytes() and w1.tobytes() == w2.tobytes()
    else:
        for x, y in zip(h1, h2):
            assert all(abs(p - q) <= 2 for p, q in zip(x, y)), (h1, h2)
        assert rel_max(g1, g2) < 1e-5 and rel_max(w1, w2) < 1e-5
