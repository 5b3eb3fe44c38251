"""CPU checks of the CBOW trainer's host routing (g2vec_b200.cbow, DESIGN.md §4.14): which launches fwdbwd picks for
every preparation of a window list, the per-list records that the prepare_* methods fill, and the one configuration
check that train_cbow and CbowModel share."""
import gc
import itertools
import weakref

import numpy as np
import pytest
import torch

from g2vec_b200 import cbow
from tests import helpers

N, B = 1000, 256                      # list length; plan batches [0, 256) .. [768, 1000)
RANGES = {"whole": (0, N), "batch": (256, B), "other": (100, 300), "none": (0, N)}
PREPS = ["nothing", "csc", "slabs", "csc+slabs", "plan"]


def _record(prep, rng):
    """The _WindowList a model holds after ``prep`` on a list of N windows (slabs and CSC over the whole list, as
    train_cbow and bench.py prepare them), or None.  The None list ("none") can only hold slab workspaces."""
    if prep == "nothing" or (rng == "none" and "slabs" not in prep):
        return None
    rec = cbow._WindowList(None if rng == "none" else torch.zeros(N, dtype=torch.int32), N)
    if "csc" in prep and rng != "none":
        rec.cscptr, rec.pos, rec.dO = torch.zeros(1), torch.zeros(1), torch.zeros(N)
    if "slabs" in prep:
        rec.slabs[(0, N)] = torch.zeros(1)
    if prep == "plan":
        rec.plan, rec.B = object(), B
        rec.brp = [0, 70, 150, 220, 300]
    return rec


def _expected(algo, lazy, det, prep, rng):
    """The precedence, stated case by case: a route name, or the RuntimeError's message fragment."""
    whole_csc = "csc" in prep and rng == "whole"
    planned = prep == "plan" and rng == "batch"
    if lazy:
        return "batch_lazy" if planned else "optimizer='lazy_adam': windows"
    if algo == "rank1":
        return "r1_csc" if whole_csc else "r1"
    if det:
        if whole_csc:
            return "csc_det"
        if rng == "none":
            return "needs a window list given to prepare_csc or prepare_batches"
        return "batch_det" if planned else "deterministic=True: windows"
    if "slabs" in prep and rng in ("whole", "none"):
        return "slabs"
    return "csc" if whole_csc else "scatter"


@pytest.mark.parametrize("algo,optimizer", [("rows", "adam"), ("rows", "sgd"), ("rows", "lazy_adam"),
                                            ("rank1", "adam"), ("rank1", "sgd")])
def test_route_of_every_preparation_and_range(algo, optimizer):
    lazy = optimizer == "lazy_adam"
    seen = set()
    for det, prep, rng in itertools.product((False, True), PREPS, RANGES):
        lo, n = RANGES[rng]
        want = _expected(algo, lazy, det, prep, rng)
        args = (algo, lazy, det, _record(prep, rng), lo, n, rng == "none")
        if " " not in want:
            assert cbow.choose_route(*args) == want, (det, prep, rng)
            seen.add(want)
        else:
            with pytest.raises(RuntimeError, match=want.replace("[", r"\[").replace("(", r"\(")):
                cbow.choose_route(*args)
    every = {"rows": {"scatter", "csc", "csc_det", "slabs", "batch_det"}, "rank1": {"r1", "r1_csc"}}[algo]
    assert seen == ({"batch_lazy"} if lazy else every)


def test_precedence_spot_checks():
    both = _record("csc+slabs", "whole")
    assert cbow.choose_route("rows", False, False, both, 0, N) == "slabs"          # bench.py prepares both
    assert cbow.choose_route("rows", False, True, both, 0, N) == "csc_det"         # det never takes slabs
    plan = _record("plan", "batch")
    assert cbow.choose_route("rows", False, False, plan, 256, B) == "scatter"      # a plan alone serves lazy/det only
    assert cbow.choose_route("rows", True, False, plan, 768, N - 768) == "batch_lazy"      # the short last batch
    with pytest.raises(RuntimeError, match="prepare_batches"):
        cbow.choose_route("rows", True, False, plan, 768, B)
    assert plan.batch(512, B) == (150, 70) and plan.batch(768, N - 768) == (220, 80)
    assert plan.batch(1024, B) is None and plan.batch(-256, B) is None and plan.batch(0, 100) is None


def _bare_model(V=60, n_windows=40):
    """A CbowModel with only what the host-side preparation reads, on the CPU."""
    rowptr, gene, _ = helpers.random_windows(n_windows, V, 1, 6, seed=1)
    m = object.__new__(cbow.CbowModel)
    m.device, m.V, m.D, m.algo, m.lazy, m.det = torch.device("cpu"), V, 8, "rows", False, False
    m.rowptr, m.gene = torch.from_numpy(rowptr).int(), torch.from_numpy(gene).int()
    m._lists, m._pending, m._dO = {}, None, None
    return m


def test_record_keeps_its_list_alive():
    m = _bare_model()
    win = torch.arange(30, dtype=torch.int32)
    alive = weakref.ref(win)
    key = (win.data_ptr(), 30)
    m.prepare_csc(win)
    del win
    gc.collect()
    assert alive() is not None                    # the address cannot be handed to another list of 30 windows
    rec = m._lists[key]
    assert rec.win is alive() and m.prepared(alive()) is rec and rec.n == 30
    assert int(rec.cscptr[-1]) == rec.pos.shape[0] == int((m.rowptr[1:31] - m.rowptr[:30]).sum())


def test_preparing_again_replaces_and_other_lists_keep_theirs(monkeypatch):
    m = _bare_model()
    a, b = torch.arange(30, dtype=torch.int32), torch.arange(35, dtype=torch.int32).flip(0).contiguous()
    m.prepare_csc(a)
    first = m.prepared(a).cscptr
    m.prepare_csc(a)
    assert len(m._lists) == 1 and m.prepared(a).cscptr is not first
    m.prepare_csc(b)                              # another list: a keeps its CSC, so a loop over a keeps its route
    assert len(m._lists) == 2 and m.prepared(a).whole(0, 30) and m.prepared(b).whole(0, 35)
    assert m.route(a) == "csc" and m.route(b) == "csc" and m.route(a, 0, 29) == "scatter"

    made = []

    class Plan:                                   # _PlanBuffers without the device: batch k touches k + 1 genes
        def __init__(self, model, win, B):
            self.B = B
            made.append(self)

        def build(self, win):
            n_b = -(-int(win.shape[0]) // self.B)
            return None, None, None, np.cumsum(np.arange(n_b + 1))
    monkeypatch.setattr(cbow, "_PlanBuffers", Plan)
    m.prepare_batches(a, 8)
    m.prepare_batches(a, 8)                       # the same batch size: the buffers are reused
    assert len(made) == 1 and [m.batch_touched(a, 8 * k, min(8, 30 - 8 * k)) for k in range(4)] == [1, 2, 3, 4]
    m.prepare_batches(a, 10)                      # another batch size: a new plan replaces the old one
    assert len(made) == 2 and m.prepared(a).plan is made[1]
    with pytest.raises(KeyError):
        m.batch_touched(a, 8, 8)
    assert m.batch_touched(a, 20, 10) == 3 and len(m._lists) == 2 and m.prepared(a).whole(0, 30)

    class Lib:                                    # gene-slab entry points without the device: 3 slabs
        def g2v_cbow_slab_plan(self, V, D, s):
            s._obj.value = 3
            return 0

        def g2v_cbow_slab_workspace_bytes(self, n, D, S):
            return 16

        def g2v_cbow_slab_setup(self, *args):
            return 0
    m.lib, m._stream = Lib(), lambda: 0
    assert m.prepare_slabs(b) and m.prepare_slabs(b) and m.prepare_slabs(b, 5, 10)
    assert sorted(m.prepared(b).slabs) == [(0, 35), (5, 10)]
    assert m.route(b) == "slabs" and m.route(b, 5, 10) == "slabs" and m.route(b, 5, 11) == "scatter"
    assert m.prepare_slabs(None) and m.prepared(None).win is None and m.route(None, 0, 40) == "slabs"
    assert len(m._lists) == 3
    m.det = True
    assert not m.prepare_slabs(a) and m.prepared(a).slabs == {}


def _parent_train_cbow_refuses(algo, optimizer, det, several, batch, reshuffle):
    """train_cbow's checks before the single check, then those of the CbowModel it built."""
    return ((reshuffle and batch <= 0) or (det and several) or (det and algo == "rank1" and batch > 0)
            or (optimizer == "lazy_adam" and (algo != "rows" or several)) or algo not in ("rows", "rank1"))


def _parent_model_refuses(algo, optimizer, det, nvl_group):
    return ((optimizer == "lazy_adam" and (algo != "rows" or nvl_group)) or (det and nvl_group)
            or algo not in ("rows", "rank1"))


def test_one_config_check_refuses_what_both_copies_refused():
    for algo, opt, det, several, batch, reshuffle in itertools.product(("rows", "rank1", "dense"),
                                                                        ("adam", "sgd", "lazy_adam"), (False, True),
                                                                        (False, True), (0, 64), (False, True)):
        want = _parent_train_cbow_refuses(algo, opt, det, several, batch, reshuffle)
        if want:
            with pytest.raises(ValueError):
                cbow.check_config(algo, opt, det, several_gpus=several, batch=batch, reshuffle=reshuffle)
        else:
            cbow.check_config(algo, opt, det, several_gpus=several, batch=batch, reshuffle=reshuffle)
        if batch == 0 and not reshuffle:          # what CbowModel passes
            try:
                cbow.check_config(algo, opt, det, several_gpus=several)
                got = False
            except ValueError:
                got = True
            assert got == _parent_model_refuses(algo, opt, det, several), (algo, opt, det, several)
    with pytest.raises(ValueError, match="one GPU"):
        cbow.check_config("rows", "lazy_adam", False, several_gpus=True)
    with pytest.raises(ValueError, match="rank1"):
        cbow.check_config("rank1", "adam", True, batch=16)
    with pytest.raises(ValueError, match="reshuffle"):
        cbow.check_config("rows", "adam", False, reshuffle=True)
