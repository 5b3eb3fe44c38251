"""GPU checks of the certified accuracy pass (g2v_cbow_eval_certified, DESIGN.md §4.16): its count is g2v_cbow_eval's
count exactly, with and without the forced row gather, on every kernel branch (D = 128/256/512 and the generic
kernel up to its largest D), sum and mean, listed and unlisted sub-ranges, empty windows, repeated genes, windows of up
to 4096 genes, initial and trained weights; windows whose logit is 0 or within a few ulps of 0 take the row gather;
the count agrees with the float64 reference; and training runs are bit for bit those of the row-gather pass."""
import re

import numpy as np
import pytest

from tests import helpers
from tests import f64_reference as f64
from tests.test_gpu_cbow_f64 import Problem, generic_max_d

pytestmark = pytest.mark.gpu

DS = [1, 33, 100, 128, 129, 256, 512, 1537, "max"]


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available()
    from g2vec_b200 import _capi
    p = torch.cuda.get_device_properties(0)
    return {"lib": _capi.load(), "capi": _capi, "sm": p.multi_processor_count,
            "optin": p.shared_memory_per_block_optin}


def counts(env, d, W, Who, V, D, red, win, lo, n):
    """(g2v_cbow_eval count, [(certified count, n_gathered) for force_gather 0 and 1]) for windows [lo, lo + n) of the
    list win (None: of the table)."""
    import torch
    lib, capi = env["lib"], env["capi"]
    st = torch.cuda.current_stream().cuda_stream
    acc = torch.zeros(3, dtype=torch.int64, device="cuda")
    scratch = torch.full((2 * V,), float("nan"), device="cuda")
    args = (d["rowptr"].data_ptr(), d["gene"].data_ptr(), d["label"].data_ptr(), None if win is None else win.data_ptr(),
            lo, n, W.data_ptr(), Who.data_ptr())
    capi.check(lib.g2v_cbow_eval(*args, acc.data_ptr(), V, D, red, st), "g2v_cbow_eval")
    want = int(acc[0])
    got = []
    for force in (0, 1):
        acc.zero_()
        capi.check(lib.g2v_cbow_eval_certified(*args, scratch.data_ptr(), acc.data_ptr() + 8, acc.data_ptr() + 16, V, D,
                                               red, force, st), "g2v_cbow_eval_certified")
        got.append((int(acc[1]), int(acc[2])))
    return want, got


def check(env, d, W, Who, V, D, red, win, lo, n, what):
    want, got = counts(env, d, W, Who, V, D, red, win, lo, n)
    assert got[0][0] == want and got[1][0] == want, (what, want, got)
    assert got[1][1] == n, (what, got)
    return want, got[0][1]


@pytest.mark.parametrize("reduce", ["sum", "mean"])
@pytest.mark.parametrize("mode", ["dyadic", "realistic"])
@pytest.mark.parametrize("D", DS)
def test_certified_count_equals_the_row_gather_count(env, D, mode, reduce):
    import torch
    if D == "max":
        D = generic_max_d(env["optin"])
    V, n_list = 4097, (2000 if D > 1000 else 5000)
    P = Problem(D, V, n_list, mode, reduce, seed=D + 11, sm=env["sm"])
    d, red = P.d, {"sum": 0, "mean": 1}[reduce]
    W, Who = d["W"], d["Who"]
    nc, gathered = check(env, d, W, Who, V, D, red, d["win"], 0, P.n, "list")
    # the float64 reference: exact on dyadic inputs (o == 0 windows included), within the band otherwise
    if mode == "dyadic":
        assert nc == P.ref.correct
        assert gathered >= int((P.ref.o == 0).sum())
    else:
        lo, hi, _ = P.ref.count_band()
        assert lo <= nc <= hi
    assert gathered >= int((P.ref.lens == 0).sum())         # empty windows always take the row gather
    check(env, d, W, Who, V, D, red, d["win"], 17, P.n - 40, "list sub-range")
    check(env, d, W, Who, V, D, red, None, 3, P.N - 5, "unlisted sub-range")
    if mode == "realistic":
        # weights after 20 trained steps
        from g2vec_b200 import CbowModel
        m = CbowModel(P.rowptr, P.gene, P.label, V, D, P.W, P.Who, reduce=reduce, lr=0.01)
        for _ in range(20):
            m.fwdbwd(d["win"], P.N)
            m.update()
        torch.cuda.synchronize()
        check(env, d, m.W_ih, m.W_ho, V, D, red, d["win"], 0, P.n, "trained")


def test_empty_windows_and_repeated_genes_take_or_keep_the_gather_count(env):
    import torch
    V, D = 500, 128
    rowptr, gene, label = helpers.random_windows(3000, V, 1, 40, seed=3)
    lens = np.diff(rowptr.astype(np.int64))
    lens[4] = lens[7] = 0                                   # two empty windows
    rowptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    gene = gene[:rowptr[-1]].copy()
    gene[rowptr[10] + 1] = gene[rowptr[10]]                # window 10 lists a gene twice
    W, Who = helpers.init_weights(V, D, 4)
    cu = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).astype(dt)).cuda()
    d = {"rowptr": cu(rowptr, np.int32), "gene": cu(gene, np.int32), "label": cu(label, np.uint8)}
    for red in (0, 1):
        _, gathered = check(env, d, cu(W, np.float32), cu(Who, np.float32), V, D, red, None, 0, len(lens), "table")
        assert gathered >= 2                                # the empty windows always take the row gather


@pytest.mark.parametrize("D", [128, 100, 512])
def test_windows_with_logit_near_zero_take_the_row_gather(env, D):
    """The last gene's row is minus the float32 running sum of the others (h == 0 exactly in the kernel's order),
    then nudged by a few ulps: |o| is 0 or a few ulps, far inside the band, so those windows must be gathered, and
    the counts must still equal g2v_cbow_eval's."""
    import torch
    rs = np.random.RandomState(D)
    n_adv, k = 64, 12
    V = n_adv * k + 200
    W, Who = helpers.init_weights(V, D, 7)
    W = W.copy()
    rows = []
    for w in range(n_adv):
        g = np.arange(w * k, (w + 1) * k)
        run = np.zeros(D, np.float32)
        for j in g[:-1]:
            run = (run + W[j]).astype(np.float32)
        W[g[-1]] = -run
        if w % 2:
            idx = rs.randint(D, size=3)
            W[g[-1], idx] = np.nextafter(W[g[-1], idx], np.float32(np.inf) * rs.choice([-1, 1], size=3))
        rows.append(g)
    for _ in range(3000):                                   # ordinary windows over the remaining genes
        rows.append(np.sort(rs.choice(np.arange(n_adv * k, V), size=rs.randint(1, 60), replace=False)))
    lens = np.array([len(r) for r in rows])
    rowptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    gene = np.concatenate(rows).astype(np.int32)
    label = (rs.rand(len(rows)) < 0.5).astype(np.uint8)
    cu = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).astype(dt)).cuda()
    d = {"rowptr": cu(rowptr, np.int32), "gene": cu(gene, np.int32), "label": cu(label, np.uint8)}
    perm = cu(rs.permutation(len(rows)), np.int32)
    for red in (0, 1):
        _, gathered = check(env, d, cu(W, np.float32), cu(Who, np.float32), V, D, red, perm, 0, len(rows), "adv")
        assert gathered >= n_adv, gathered
        assert gathered < len(rows) // 2, gathered         # the ordinary windows are decided without rows


@pytest.mark.parametrize("D", [2, 128, 129])
def test_an_underflowing_mean_scale_times_a_large_w_ho_takes_the_row_gather(env, D):
    """tests/test_certified_host.py's window whose row-gather logit (+2^-51) has the opposite sign of the exact and the
    collapsed logit (-2^-51), because scale * h[0] underflows and is then multiplied by W_ho[0] = 2^100: the certified
    count must still be g2v_cbow_eval's."""
    import torch
    from tests.test_certified_host import underflow_window
    W, Who = underflow_window(D)
    rowptr = np.array([0, 2, 4, 5], np.int32)               # the window twice (labels 1 and 0), and {1}
    gene = np.array([0, 1, 0, 1, 1], np.int32)
    label = np.array([1, 0, 1], np.uint8)
    cu = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).astype(dt)).cuda()
    d = {"rowptr": cu(rowptr, np.int32), "gene": cu(gene, np.int32), "label": cu(label, np.uint8)}
    want, got = counts(env, d, cu(W, np.float32), cu(Who, np.float32), 2, D, 1, None, 0, 3)
    assert got[0][0] == want and got[1] == (want, 3), (want, got)
    assert got[0][1] >= 2                                   # both copies of the window are gathered


def test_refuses_the_d_range_g2v_cbow_eval_refuses(env):
    import torch
    lib = env["lib"]
    D = generic_max_d(env["optin"]) + 1
    V = 3
    z = lambda n, dt=torch.float32: torch.zeros(n, dtype=dt, device="cuda")
    rowptr, gene, label = z(2, torch.int32), z(1, torch.int32), z(1, torch.uint8)
    W, Who, st, acc = z(V * D), z(D), z(2 * V), z(2, torch.int64)
    s = torch.cuda.current_stream().cuda_stream
    rc0 = lib.g2v_cbow_eval(rowptr.data_ptr(), gene.data_ptr(), label.data_ptr(), None, 0, 1, W.data_ptr(),
                            Who.data_ptr(), acc.data_ptr(), V, D, 0, s)
    msg0 = lib.g2v_last_error().decode()
    rc1 = lib.g2v_cbow_eval_certified(rowptr.data_ptr(), gene.data_ptr(), label.data_ptr(), None, 0, 1, W.data_ptr(),
                                      Who.data_ptr(), st.data_ptr(), acc.data_ptr(), None, V, D, 0, 0, s)
    msg1 = lib.g2v_last_error().decode()
    assert rc0 == rc1 == 2 and "sizeHiddenlayer" in msg0 and msg0 == msg1


def _train(g2v, monkeypatch, g, use_graph, row_gather):
    from g2vec_b200 import cbow
    if row_gather:                                          # CbowModel.evaluate as it was: g2v_cbow_eval
        def evaluate(self, win, slot, win_begin=0, n_win=None):
            n = int((win.shape[0] - win_begin) if n_win is None else n_win)
            self._launch("g2v_cbow_eval", self.rowptr.data_ptr(), self.gene.data_ptr(), self.label.data_ptr(),
                         self._ptr(win), int(win_begin), n, self.W_ih.data_ptr(), self.W_ho.data_ptr(),
                         self.acc.data_ptr() + 8 * slot, self.V, self.D, self.reduce)
        monkeypatch.setattr(cbow.CbowModel, "evaluate", evaluate)
    else:
        monkeypatch.undo()
    lines = []
    W, info = g2v.train_cbow(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"], max_epoch=500,
                             seed=g["seed"], log=lambda *a: lines.append(" ".join(map(str, a))), return_info=True,
                             use_graph=use_graph, deterministic=True)
    monkeypatch.undo()
    lines = [re.sub(r" \([0-9.]+ sec\)", "", s) for s in lines]   # the log's wall-clock times are not compared
    return W.tobytes(), info["model"].W_ho.cpu().numpy().tobytes(), info["history"], info["stop_step"], lines


@pytest.mark.parametrize("name", ["cbow_small.npz", "cbow_ex.npz"])
def test_training_runs_equal_the_row_gather_pass_bit_for_bit(monkeypatch, name):
    import g2vec_b200 as g2v
    g = helpers.cbow_golden(name)
    for use_graph in (True, False):
        a = _train(g2v, monkeypatch, g, use_graph, row_gather=False)
        b = _train(g2v, monkeypatch, g, use_graph, row_gather=True)
        assert a == b, (name, use_graph)
        assert a[3] == g["stop_step"]


def test_the_device_loop_launches_the_certified_pass(monkeypatch):
    import g2vec_b200 as g2v
    from g2vec_b200 import cbow
    seen = []
    g = helpers.cbow_golden("cbow_small.npz")
    real = cbow.CbowModel._launch

    def launch(self, name, *args):
        seen.append(name)
        return real(self, name, *args)
    monkeypatch.setattr(cbow.CbowModel, "_launch", launch)
    g2v.train_cbow(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"], max_epoch=3, seed=g["seed"], log=None,
                   early_stop=False, use_graph=False)
    assert "g2v_cbow_eval_certified" in seen and "g2v_cbow_eval" not in seen
