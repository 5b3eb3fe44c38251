"""g2v_cbow_loop_tail_val (DESIGN.md §4.32): the carried step's validation pass and tail pass in one window launch.
Against g2v_cbow_loop_tail and g2v_cbow_eval_certified on the same inputs: dO and the training count acc[5] bit for
bit, the validation count exactly, g_ho and the loss acc[4] up to the order of their atomics; and a DeviceLoop that
routes to it against one that runs the two passes apart."""
import numpy as np
import pytest

from tests import helpers

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available()
    from g2vec_b200 import _capi
    return _capi.load()


def _stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def _case(V, D, N, lmin, lmax, seed):
    import torch
    rowptr, gene, label = helpers.random_windows(N, V, lmin, lmax, seed=seed)
    W, Wo = helpers.init_weights(V, D, seed)
    cu = lambda a: torch.from_numpy(a).cuda()
    return cu(rowptr), cu(gene), cu(label), cu(W), cu(Wo)


def _run(lib, case, tr, va, V, D, reduce, cw, fused):
    """One carried tail (+ validation pass) from zeroed state: (dO, g_ho, acc) after the launches."""
    import torch
    from g2vec_b200 import _capi
    rowptr, gene, label, W, Wo = case
    dO = torch.full((max(len(tr), 1),), -7.0, dtype=torch.float32, device="cuda")
    g_ho = torch.zeros(D, dtype=torch.float32, device="cuda")
    acc = torch.zeros(6, dtype=torch.int64, device="cuda")
    ctl = torch.zeros(8, dtype=torch.int64, device="cuda")
    st = torch.zeros(2 * V, dtype=torch.float32, device="cuda")
    p = lambda t: t.data_ptr()
    inv_n = 1.0 / max(len(tr), 1)
    cwa = tuple(cw) if cw else ()
    sfx = "_cw" if cw else ""
    if fused:
        name = "g2v_cbow_loop_tail_val" + sfx
        _capi.check(getattr(lib, name)(p(ctl), p(rowptr), p(gene), p(label), p(tr), len(tr), inv_n, p(va), len(va),
                                       p(W), p(Wo), p(st), p(dO), p(g_ho), p(acc), V, D, reduce, *cwa, _stream()), name)
    else:
        _capi.check(lib.g2v_cbow_eval_certified(p(rowptr), p(gene), p(label), p(va), 0, len(va), p(W), p(Wo), p(st),
                                                p(acc) + 16, None, V, D, reduce, 0, _stream()), "g2v_cbow_eval_certified")
        name = "g2v_cbow_loop_tail" + sfx
        _capi.check(getattr(lib, name)(p(ctl), p(rowptr), p(gene), p(label), p(tr), len(tr), inv_n, p(W), p(Wo),
                                       p(dO), p(g_ho), p(acc), V, D, reduce, *cwa, _stream()), name)
    torch.cuda.synchronize()
    assert int(ctl[7]) == 0                               # the work counter is left at 0 for the next launch
    return dO.cpu(), g_ho.cpu().numpy(), acc.cpu(), ctl.cpu()


def _compare(lib, case, tr, va, V, D, reduce, cw):
    import torch
    a = _run(lib, case, tr, va, V, D, reduce, cw, fused=True)
    b = _run(lib, case, tr, va, V, D, reduce, cw, fused=False)
    assert torch.equal(a[0], b[0]), "dO"
    assert int(a[2][5]) == int(b[2][5]) and int(a[2][3]) == int(b[2][3]), "training count"
    assert int(a[2][2]) == int(b[2][2]), "validation count"
    assert torch.equal(a[3], b[3]), "ctl"
    # each warp sums its windows' loss terms in float32, and the queue hands a warp other windows than the static
    # stride does: the loss and g_ho agree to float32 reassociation
    la, lb = (float(x[2][4:5].view(torch.float64)[0]) for x in (a, b))
    assert abs(la - lb) <= 1e-5 * max(abs(lb), 1e-30), "loss"
    scale = max(float(np.abs(b[1]).max()), 1e-30)
    assert float(np.abs(a[1] - b[1]).max()) <= 1e-5 * scale, "g_ho"
    return a


@pytest.mark.parametrize("D", [128, 256, 512])
@pytest.mark.parametrize("reduce", [0, 1])
@pytest.mark.parametrize("cw", [None, (0.25, 3.0)])
def test_fused_launch_equals_the_two_passes(env, D, reduce, cw):
    import torch
    from g2vec_b200 import _capi
    V, N = 700, 6000
    red = [_capi.REDUCE_SUM, _capi.REDUCE_MEAN][reduce]
    case = _case(V, D, N, 0, 90, seed=D + reduce)          # lmin 0: empty windows in both lists
    rs = np.random.RandomState(D)
    perm = rs.permutation(N).astype(np.int32)
    tr, va = torch.from_numpy(perm[:4500]).cuda(), torch.from_numpy(perm[4500:]).cuda()
    a = _compare(env, case, tr, va, V, D, red, cw)
    assert 0 < int(a[2][2]) < len(va)


@pytest.mark.parametrize("n_tr,n_va", [(0, 0), (0, 37), (53, 0), (1, 1), (1, 3), (2, 5), (3, 4)])
def test_empty_and_short_lists(env, n_tr, n_va):
    import torch
    from g2vec_b200 import _capi
    V, D, N = 300, 128, 200
    case = _case(V, D, N, 0, 12, seed=n_tr * 7 + n_va)
    perm = np.random.RandomState(1).permutation(N).astype(np.int32)
    tr = torch.from_numpy(perm[:n_tr].copy()).cuda()
    va = torch.from_numpy(perm[n_tr:n_tr + n_va].copy()).cuda()
    _compare(env, case, tr, va, V, D, _capi.REDUCE_SUM, None)
    _compare(env, case, tr, va, V, D, _capi.REDUCE_MEAN, (2.0, 0.5))


def test_rejects_what_it_has_no_kernel_for(env):
    import torch
    from g2vec_b200 import _capi
    z = torch.zeros(64, dtype=torch.int64, device="cuda")
    p = z.data_ptr()
    assert env.g2v_cbow_loop_tail_val(p, p, p, p, p, 4, 0.25, p, 4, p, p, p, p, p, p, 10, 100, 0, None) != 0
    assert env.g2v_cbow_loop_tail_val(None, p, p, p, p, 4, 0.25, p, 4, p, p, p, p, p, p, 10, 128, 0, None) != 0
    assert env.g2v_cbow_loop_tail_val_cw(p, p, p, p, p, 4, 0.25, p, 4, p, p, p, p, p, p, 10, 128, 0, 0.0, 1.0,
                                         None) != 0
    torch.cuda.synchronize()


def _loop_run(D, seed, fused, monkeypatch, capture=False):
    import torch
    from g2vec_b200 import cbow
    import g2vec_b200 as g2v
    V, N = 500, 4000
    rowptr, gene, label = helpers.random_windows(N, V - 20, 1, 60, seed=seed)
    W0, Wo0 = helpers.init_weights(V, D, seed)
    tr, va = cbow.split_indices(N, seed)
    tr_d = torch.from_numpy(tr.astype(np.int32)).cuda()
    va_d = torch.from_numpy(va.astype(np.int32)).cuda()
    m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005)
    m.prepare_csc(tr_d)
    seen = []
    real = cbow.CbowModel._launch

    def launch(self, name, *args):
        seen.append(name)
        return real(self, name, *args)
    monkeypatch.setattr(cbow.CbowModel, "_launch", launch)
    if not fused:
        monkeypatch.setattr(cbow, "TAIL_VAL_D", ())
    loop = cbow.DeviceLoop(m, None, tr_d, va_d, len(tr_d), 20, True, snapshot=True)
    loop.attach()
    try:
        if capture:
            loop.one(True)
            loop.reset()
            g = loop.capture([True] * 5)
            for _ in range(4):
                g.replay()
        else:
            for _ in range(20):
                loop.one(True)
            loop.fetch()
        torch.cuda.synchronize()
    finally:
        loop.detach()
        monkeypatch.undo()
    assert ("g2v_cbow_loop_tail_val" in seen) == fused
    assert ("g2v_cbow_eval_certified" in seen) != fused
    return loop.hist_pin.view(-1, 4).tolist(), int(loop.ctl_pin[2]), m.W_ih.cpu().numpy(), m.W_ho.cpu().numpy()


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("D,capture", [(128, False), (256, False), (128, True)])
def test_device_loop_route_equals_the_parent_launches(monkeypatch, D, capture):
    """20 steps (eager, or four replays of a 5-step graph captured right after reset()): the same history and stop
    step as the loop that runs the validation pass and the tail apart (counts up to g_ho's atomic order); weights
    within the carried-loop tolerance."""
    ha, sa, wa, oa = _loop_run(D, 17, True, monkeypatch, capture)
    hb, sb, wb, ob = _loop_run(D, 17, False, monkeypatch, capture)
    assert sa == sb
    n = sa + 1 if sa >= 0 else 20
    assert ha[0][1] > 0                                   # the first step counted its own full forward
    # g_ho's unordered atomics differ from run to run on either route: counts within 2, as test_gpu_cbow_carry.py
    for x, y in zip(ha[:n], hb[:n]):
        assert all(abs(p - q) <= 2 for p, q in zip(x[1:], y[1:])), (ha[:n], hb[:n])
    assert _rel(wa, wb) < 1e-5 and _rel(oa, ob) < 1e-4
