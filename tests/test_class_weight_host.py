"""Class weights of the training loss (DESIGN.md §4.20) on the host: the float32 restatement of a weighted step against
float64, the checks of ``class_weight`` in check_config / train_cbow and of ``--class-weight`` on the command line,
"balanced" from the training split, and which entry points every route calls with and without weights.  CPU."""

import numpy as np
import pytest
import torch

from g2vec_b200 import cbow, cli
from tests import class_weight_oracle as cwo, f64_reference as f64, helpers

F32 = np.float32


@pytest.mark.parametrize("cw", [(1.0, 1.0), (0.25, 4.0), (0.37, 1.9)])
def test_float32_step_against_float64(cw):
    rs = np.random.RandomState(5)
    o = (rs.randn(4000) * 6).astype(F32)
    o[:3] = [0, 40, -40]
    y = (rs.rand(4000) < 0.5).astype(F32)
    inv_n = F32(1) / F32(4000)
    dO, lt = cwo.do32(o, y, inv_n, cw)
    w = cwo.weights_of(y, cw)
    want = (f64.sigmoid64(o) - y) * float(inv_n) * w
    # sigma within a few ulps, then two roundings of the products (sigma - y may cancel: absolute term)
    err = 8 * f64.U * np.abs(want) + 4 * f64.U * float(inv_n) * w
    assert (np.abs(dO - want) <= err).all()
    l64 = (np.maximum(o, 0) - o.astype(np.float64) * y + np.log1p(np.exp(-np.abs(o.astype(np.float64))))) * w
    assert (np.abs(lt - l64) <= 8 * f64.U * (np.abs(l64) + w)).all()


def test_unit_weights_give_the_unweighted_bits():
    rs = np.random.RandomState(1)
    o = (rs.randn(1000) * 4).astype(F32)
    y = (rs.rand(1000) < 0.5).astype(F32)
    inv_n = F32(1) / F32(1000)
    dO, lt = cwo.do32(o, y, inv_n, (1, 1))
    plain = ((cwo.sigmoid32(o) - y).astype(F32) * inv_n).astype(F32)
    assert dO.view(np.int32).tolist() == plain.view(np.int32).tolist()
    # dyadic weights scale exactly (no overflow or underflow here)
    d4, _ = cwo.do32(o, y, inv_n, (0.25, 4))
    assert np.array_equal(d4, plain * np.where(y != 0, F32(4), F32(0.25)))


BAD = [0, -1, float("inf"), float("nan"), 1e40, -0.0, 1e-50, True, "1", None]


@pytest.mark.parametrize("bad", BAD)
def test_check_config_refuses_bad_weights(bad):
    for pair in ((bad, 1.0), (1.0, bad)):
        if bad is None:
            continue
        with pytest.raises(ValueError, match="class_weight"):
            cbow.check_config("rows", "adam", False, class_weight=pair)
        with pytest.raises(ValueError, match="class_weight"):
            cbow.class_weight_pair(pair)
    rowptr = np.array([0, 1, 2, 3], np.int32)
    with pytest.raises(ValueError, match="class_weight"):
        cbow.train_cbow(rowptr, np.zeros(3, np.int32), np.zeros(3, np.uint8), 4, 8, 0.01, log=None,
                        class_weight=(bad, 1.0))


@pytest.mark.parametrize("bad", ["", "Balanced", "1,2", (1,), (1, 2, 3), [], 1.0, {"a": 1}])
def test_check_config_refuses_other_shapes(bad):
    with pytest.raises(ValueError, match="class_weight"):
        cbow.check_config("rows", "adam", False, class_weight=bad)


def test_check_config_accepts():
    for cw in (None, "balanced", (1, 1), (0.25, 4), [0.37, 1.9], (np.float32(2), np.float64(3)), (1e-30, 3e38)):
        for algo, opt in (("rows", "adam"), ("rows", "sgd"), ("rows", "lazy_adam"), ("rank1", "adam")):
            cbow.check_config(algo, opt, False, class_weight=cw)
        cbow.check_config("rows", "adam", True, batch=64, reshuffle=True, class_weight=cw, weight_decay=0.01,
                          lr_patience=2, monitor="val_loss")
        cbow.check_config("rows", "sgd", False, several_gpus=True, class_weight=cw)
    assert cbow.class_weight_pair((0.37, 1.9)) == (float(F32(0.37)), float(F32(1.9)))
    assert cbow.class_weight_pair(None) is None


def test_command_line_arguments():
    base = ["E", "C", "N", "R"]
    assert cli.parse_arguments(base).class_weight is None
    assert cli.parse_arguments(base + ["--class-weight", "balanced"]).class_weight == "balanced"
    assert cli.parse_arguments(base + ["--class-weight", "1,1"]).class_weight == (1.0, 1.0)
    assert cli.parse_arguments(base + ["--class-weight", "0.37,1.9"]).class_weight == (float(F32(0.37)),
                                                                                       float(F32(1.9)))
    for bad in ("0,1", "1,0", "-1,1", "1,-1", "inf,1", "nan,1", "1e40,1", "1,", ",1", "1", "a,b", "1,2,3",
                "Balanced", ""):
        with pytest.raises(SystemExit):
            cli.parse_arguments(base + ["--class-weight=" + bad])


@pytest.mark.parametrize("n0,n1", [(300, 100), (50, 350), (7, 1), (1, 7)])
def test_balanced_is_sklearns_rule(n0, n1):
    labels = np.array([0] * n0 + [1] * n1 + [1, 0] * 10, np.uint8)      # the tail is outside the training split
    tr = np.random.RandomState(0).permutation(n0 + n1)
    w0, w1 = cbow.balanced_class_weight(labels, tr)
    n = n0 + n1
    assert (w0, w1) == (float(F32(n / (2.0 * n0))), float(F32(n / (2.0 * n1))))
    assert (w0, w1) == cwo.balanced(labels[tr])
    # each label carries half of the weighted count
    assert abs(w0 * n0 - n / 2) <= 1e-6 * n and abs(w1 * n1 - n / 2) <= 1e-6 * n
    assert cbow.balanced_class_weight(torch.from_numpy(labels), tr) == (w0, w1)
    try:
        from sklearn.utils.class_weight import compute_class_weight
    except ImportError:
        return
    sk = compute_class_weight("balanced", classes=np.array([0, 1]), y=labels[tr])
    assert (w0, w1) == (float(F32(sk[0])), float(F32(sk[1])))


@pytest.mark.parametrize("label", [0, 1])
def test_balanced_refuses_a_one_label_split(label):
    labels = np.full(40, label, np.uint8)
    labels[-5:] = 1 - label                                  # the other label only outside the split
    with pytest.raises(ValueError, match="both labels"):
        cbow.balanced_class_weight(labels, np.arange(35))
    rowptr = np.arange(41, dtype=np.int32)
    with pytest.raises(ValueError, match="both labels"):
        cbow.train_cbow(rowptr, np.zeros(40, np.int32), labels, 4, 8, 0.01, log=None, class_weight="balanced",
                        split=(np.arange(35), np.arange(35, 40)))


# ---- which entry points each route calls
class _Lib:
    """Records the name of every entry point called; each returns 0."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            return 0
        return f


def _fake_model(algo, lazy, det, cw):
    m = object.__new__(cbow.CbowModel)
    V, D, N = 30, 8, 40
    rowptr, gene, label = helpers.random_windows(N, V, 1, 5, seed=2)
    m.device, m.V, m.D, m.algo, m.lazy, m.det = torch.device("cpu"), V, D, algo, lazy, det
    m.rowptr, m.gene, m.label = (torch.from_numpy(a) for a in (rowptr, gene, label))
    m._lists, m._pending, m._dO, m._det_ws = {}, None, torch.zeros(N), torch.zeros(64, dtype=torch.uint8)
    z = torch.zeros
    m.W_ih, m.W_ho, m.g_ih, m.g_ho, m.s, m.c = z(V, D), z(D), z(V, D), z(D), z(V), z(V)
    m.acc, m.reduce, m._n_slabs = z(6, dtype=torch.int64), 0, 3
    m.cw = cbow.class_weight_pair(cw)
    m.lib = _Lib()
    m._stream = lambda: 0
    return m, N


PLAIN = {"scatter": ["g2v_cbow_fwdbwd"], "slabs": ["g2v_cbow_fwdbwd_slabs"], "csc": ["g2v_cbow_fwdbwd_csc"],
         "csc_det": ["g2v_cbow_fwdbwd_csc_det"], "batch_lazy": ["g2v_cbow_fwd_do"],
         "batch_det": ["g2v_cbow_fwd_do_det", "g2v_cbow_batch_expand"], "r1": ["g2v_cbow_r1_windows"],
         "r1_csc": ["g2v_cbow_r1_windows_csc"]}
CW_FORMS = {"g2v_cbow_fwdbwd", "g2v_cbow_fwdbwd_csc", "g2v_cbow_fwd_do", "g2v_cbow_fwdbwd_csc_det",
            "g2v_cbow_fwd_do_det", "g2v_cbow_loop_tail", "g2v_cbow_loop_tail_det", "g2v_cbow_fwdbwd_slabs",
            "g2v_cbow_r1_windows", "g2v_cbow_r1_windows_csc"}


def _prepare(m, route, N):
    win = torch.arange(N, dtype=torch.int32)
    rec = m._record(win)
    if route in ("csc", "csc_det", "r1_csc"):
        rec.cscptr, rec.pos, rec.dO = torch.zeros(m.V + 1, dtype=torch.int32), torch.zeros(1), torch.zeros(N)
    if route == "slabs":
        rec.slabs[(0, N)] = torch.zeros(1)
    if route in ("batch_lazy", "batch_det"):
        rec.plan = type("P", (), {"rows": torch.zeros(4, dtype=torch.int32), "segptr": torch.zeros(5, dtype=torch.int32),
                                  "pos": torch.zeros(4, dtype=torch.int32)})()
        rec.B, rec.brp = 16, [0, 4, 8, 12]
        return win, 0, 16
    return win, 0, N


ROUTES = [("rows", False, False, "scatter"), ("rows", False, False, "slabs"), ("rows", False, False, "csc"),
          ("rows", False, True, "csc_det"), ("rows", True, False, "batch_lazy"), ("rows", False, True, "batch_det"),
          ("rank1", False, False, "r1"), ("rank1", False, False, "r1_csc")]


@pytest.mark.parametrize("algo,lazy,det,route", ROUTES)
def test_every_route_calls_the_parent_entry_points_without_weights_and_cw_forms_with(algo, lazy, det, route):
    seen = []
    for cw in (None, (1, 1), (0.25, 4)):
        m, N = _fake_model(algo, lazy, det, cw)
        win, lo, n = _prepare(m, route, N)
        assert m.route(win, lo, n) == route
        m.fwdbwd(win, N, lo, n)
        if route in ("csc", "csc_det"):                     # the carried loop's tail pass over the same list
            m.loop_tail(torch.zeros(8, dtype=torch.int64), win, N)
        names = [c[0] for c in m.lib.calls if not c[0].endswith("_bytes")]      # sizes, not launches
        want = PLAIN[route] + (["g2v_cbow_loop_tail" + ("_det" if det else "")] if route in ("csc", "csc_det") else [])
        if cw is None:
            assert names == want
        else:
            assert names == [x + "_cw" if x in CW_FORMS else x for x in want]
            for name, args in m.lib.calls:
                if name.endswith("_cw"):
                    assert args[-3:-1] == cbow.class_weight_pair(cw)      # then the stream
        seen.append(names)
    assert seen[1] == seen[2]


def test_every_cw_form_is_bound():
    from g2vec_b200 import _capi
    for name in CW_FORMS:
        plain, cw = _capi.SIGNATURES[name], _capi.SIGNATURES[name + "_cw"]
        assert cw[1] == plain[1][:-1] + [_capi._f32, _capi._f32, plain[1][-1]]


def test_train_cbow_resolves_balanced_before_the_model(monkeypatch):
    got = {}

    class Stop(Exception):
        pass

    def fake_model(*a, **k):
        got.update(k)
        raise Stop
    monkeypatch.setattr(cbow, "CbowModel", fake_model)
    rowptr, gene, label = helpers.random_windows(200, 30, 1, 4, seed=3)
    label[:] = 0
    label[:50] = 1
    tr, va = np.arange(40, 200), np.arange(40)              # 10 label-1 windows in the training split
    with pytest.raises(Stop):
        cbow.train_cbow(rowptr, gene, label, 30, 8, 0.01, log=None, class_weight="balanced", split=(tr, va))
    assert got["class_weight"] == (float(F32(160 / 300)), float(F32(160 / 20)))
    for cw, want in ((None, None), ((0.5, 2), (0.5, 2))):
        with pytest.raises(Stop):
            cbow.train_cbow(rowptr, gene, label, 30, 8, 0.01, log=None, class_weight=cw, split=(tr, va))
        assert got["class_weight"] == want
