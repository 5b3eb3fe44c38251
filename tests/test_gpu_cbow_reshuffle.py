"""GPU checks of reshuffled mini-batch epochs (DESIGN.md §4.12): the epoch-order kernel against the NumPy restatement
of P, the batch-plan builder against the torch.sort construction it replaced, and train_cbow(reshuffle=True) against
the CPU loops fed the restated orders."""
import re

import numpy as np
import pytest

import oracle
from tests import helpers, reshuffle_oracle as ro

pytestmark = pytest.mark.gpu
RTOL_VEC = 1e-4


@pytest.fixture(scope="module")
def g2v():
    import torch
    assert torch.cuda.is_available()
    import g2vec_b200
    return g2vec_b200


def rel_max(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("n", [1, 2, 3, 1000, 2 ** 20 + 3])
def test_epoch_order_kernel_equals_the_restatement(g2v, n):
    import torch
    from g2vec_b200 import cbow
    tr = np.random.RandomState(n % 97).permutation(n).astype(np.int32)
    td = torch.from_numpy(tr).cuda()
    for seed, epoch in ((0, 1), (3, 2), ((5 << 32) | 17, 9)):
        for rank, world in ((0, 1), (0, 2), (1, 2), (2, 3), (7, 8)):
            got = cbow.epoch_order(td, seed, epoch, rank, world).cpu().numpy()
            want = ro.epoch_list(tr, seed, epoch, rank, world)
            assert got.shape == want.shape and (got == want).all(), (seed, epoch, rank, world)


def _model(g2v, rowptr, gene, label, V, D=16):
    W0, Wo0 = helpers.init_weights(V, D, 0)
    return g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, optimizer="lazy_adam")


def _check_plan(m, win_np, B):
    import torch
    from g2vec_b200 import cbow
    wd = torch.from_numpy(np.ascontiguousarray(win_np, dtype=np.int32)).cuda()
    got = [x.cpu().numpy() for x in cbow.batch_plan(m, wd, B)]
    want = ro.batch_plan_torch(m.rowptr, m.gene, m.V, wd, B)
    for name, a, b in zip(("rows", "segptr", "pos", "batch_rowptr"), got, want):
        assert a.dtype == np.int32 and a.shape == b.shape and (a == b).all(), (name, B)


def test_batch_plan_equals_the_sort_construction(g2v):
    V, N = 600, 1500
    rowptr, gene, label = helpers.random_windows(N, V - 40, 1, 80, seed=4)
    rowptr[5] = rowptr[4]                                                 # window 4 empty
    gene = gene[:rowptr[N - 1]].copy(); rowptr[N] = rowptr[N - 1]
    gene[rowptr[5] + 1] = gene[rowptr[5]]                                 # window 5 lists a gene twice
    m = _model(g2v, rowptr, gene, label, V)
    rs = np.random.RandomState(0)
    for B in (1, 7, 64, 1000, 1499, 1500, 5000):                          # short last batches, B = 1, B >= n
        _check_plan(m, rs.permutation(N), B)
    _check_plan(m, rs.permutation(N)[:333], 100)


def test_batch_plan_long_segments(g2v):
    """Genes in more than 32 and more than 4096 windows of a batch (the shared-memory and the counting sorts)."""
    V, N = 50, 12000
    rs = np.random.RandomState(1)
    lens = rs.randint(1, 6, size=N)
    rowptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    gene = np.concatenate([np.sort(rs.choice(V, size=k, replace=False)) for k in lens]).astype(np.int32)
    gene[rowptr[:-1]] = 0                                                 # gene 0 in every window
    label = (rs.rand(N) < 0.5).astype(np.uint8)
    m = _model(g2v, rowptr, gene, label, V)
    for B in (300, 5000, 12000):
        _check_plan(m, rs.permutation(N), B)


def test_batch_plan_at_200k_genes(g2v):
    """V = 200k: waves of K = 2^22 // V = 20 batches.  B = 1024 and 5000 fit one wave; B = 64 (94 batches: 4 full waves
    and one of 14) and B = 70 (86 batches, the last one short: 4 waves and one of 6) carry the running row and
    incidence totals, batch_rowptr and segptr across wave boundaries."""
    V, N = 200_000, 6000
    rs = np.random.RandomState(2)
    lens = rs.randint(20, 81, size=N)
    rowptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    gene = np.concatenate([np.sort(rs.choice(V, size=k, replace=False)) for k in lens]).astype(np.int32)
    label = (rs.rand(N) < 0.5).astype(np.uint8)
    m = _model(g2v, rowptr, gene, label, V)
    for B in (1024, 5000, 64, 70):
        _check_plan(m, rs.permutation(N), B)
    _check_plan(m, rs.permutation(N)[:4321], 64)                         # 68 batches, last one short


def test_batch_plan_on_the_ex_windows(g2v):
    (rowptr, gene, label), _ = helpers.ex_windows(reps=2)
    V = 7523
    m = _model(g2v, rowptr, gene, label, V)
    tr, _ = oracle.split_indices(len(label), 0)
    for B in (1024, 16384):
        _check_plan(m, ro.epoch_list(tr, 0, 1), B)


def test_prepare_batches_keeps_one_plan_in_the_lists_record(g2v):
    """A second prepare_batches for the same list replaces its plan (and releases the buffers of the first batch
    size); the new plan is the builder's for the new batch size."""
    import torch
    V, N = 600, 1000
    rowptr, gene, label = helpers.random_windows(N, V, 1, 40, seed=7)
    m = _model(g2v, rowptr, gene, label, V)
    win = np.random.RandomState(3).permutation(N)
    wd = torch.from_numpy(win.astype(np.int32)).cuda()
    m.prepare_batches(wd, 64)
    assert m.batch_touched(wd, 64, 64) > 0
    m.prepare_batches(wd, 100)
    with pytest.raises(KeyError):
        m.batch_touched(wd, 64, 64)
    assert m.prepared(wd).plan.B == m.prepared(wd).B == 100
    _, _, _, brp = ro.batch_plan_torch(m.rowptr, m.gene, V, wd, 100)
    assert [m.batch_touched(wd, k * 100, 100) for k in range(10)] == list(np.diff(brp))


def _problem():
    V, N, D, B = 3000, 1200, 128, 256
    rowptr, gene, label = helpers.random_windows(N, V, 1, 30, seed=12)
    W0, Wo0 = helpers.init_weights(V, D, 4)
    tr, _ = oracle.split_indices(N, 0)
    return rowptr, gene, label, V, D, B, W0, Wo0, tr


@pytest.mark.parametrize("optimizer,algo", [("adam", "rows"), ("adam", "rank1"), ("sgd", "rows"), ("lazy_adam", "rows")])
def test_reshuffled_training_equals_the_oracle_loops(g2v, optimizer, algo):
    rowptr, gene, label, V, D, B, W0, Wo0, tr = _problem()
    lr = 0.5 if optimizer == "sgd" else 0.005        # SGD on batch-mean gradients moves W too little at 0.005 for the
    orders = ro.epoch_orders(tr, 0, 3)               # order to show above 10 * RTOL_VEC in 3 epochs
    if optimizer == "lazy_adam":
        want, _ = ro.lazy_minibatch_train_orders(rowptr, gene, label, orders, W0, Wo0, lr, B)
        fixed_want, _ = ro.lazy_minibatch_train_orders(rowptr, gene, label, [tr] * 3, W0, Wo0, lr, B)
    else:
        want, _ = ro.dense_minibatch_train_orders(rowptr, gene, label, orders, W0, Wo0, lr, B, optimizer)
        fixed_want, _ = ro.dense_minibatch_train_orders(rowptr, gene, label, [tr] * 3, W0, Wo0, lr, B, optimizer)
    kw = dict(seed=0, W_ih0=W0, W_ho0=Wo0, early_stop=False, log=None, batch=B, optimizer=optimizer, algo=algo)
    got = g2v.train_cbow(rowptr, gene, label, V, D, lr, max_epoch=3, reshuffle=True, **kw)
    assert rel_max(got, want) < RTOL_VEC
    fixed = g2v.train_cbow(rowptr, gene, label, V, D, lr, max_epoch=3, **kw)
    assert rel_max(fixed, fixed_want) < RTOL_VEC
    assert rel_max(got, fixed) > 10 * RTOL_VEC
    one = g2v.train_cbow(rowptr, gene, label, V, D, lr, max_epoch=1, reshuffle=True, **kw)
    one_fixed = g2v.train_cbow(rowptr, gene, label, V, D, lr, max_epoch=1, **kw)
    assert rel_max(one, one_fixed) < 1e-5


def test_reshuffle_argument_checks_and_full_batch(g2v):
    rowptr, gene, label, V, D, B, W0, Wo0, tr = _problem()
    kw = dict(seed=0, W_ih0=W0, W_ho0=Wo0, early_stop=False, log=None, max_epoch=2)
    with pytest.raises(ValueError):
        g2v.train_cbow(rowptr, gene, label, V, D, 0.005, batch=0, reshuffle=True, **kw)
    a = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, batch=10 * len(tr), reshuffle=True, **kw)
    b = g2v.train_cbow(rowptr, gene, label, V, D, 0.005, batch=10 * len(tr), **kw)
    assert rel_max(a, b) < 1e-5                      # full batch: the same launches (the scatter's atomics are unordered)


def test_order_and_plan_run_once_per_reshuffled_epoch(g2v, monkeypatch):
    from g2vec_b200 import _capi
    lib = _capi.load()
    calls = {k: 0 for k in ("g2v_cbow_epoch_order", "g2v_cbow_batch_plan")}

    def count(name, fn):
        def wrapped(*a):
            calls[name] += 1
            return fn(*a)
        return wrapped
    for k in calls:
        monkeypatch.setattr(lib, k, count(k, getattr(lib, k)))
    g = helpers.cbow_golden("cbow_small.npz")
    args = (g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"])
    epochs = 6
    for opt, reshuffle, order, plan in (("adam", False, 0, 0), ("lazy_adam", False, 0, 1),
                                        ("adam", True, epochs - 1, 0), ("lazy_adam", True, epochs - 1, epochs)):
        for k in calls:
            calls[k] = 0
        g2v.train_cbow(*args, max_epoch=epochs, seed=g["seed"], early_stop=False, log=None, batch=64, optimizer=opt,
                       reshuffle=reshuffle)
        assert calls == {"g2v_cbow_epoch_order": order, "g2v_cbow_batch_plan": plan}, (opt, reshuffle)


@pytest.mark.parametrize("optimizer", ["adam", "lazy_adam"])
def test_command_line_with_reshuffled_minibatches(g2v, tmp_path, capsys, optimizer):
    from g2vec_b200 import cli
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    prefix = str(tmp_path / "resh")
    cli.main([ef, cf, nf, prefix, "-r", "2", "-e", "3", "-n", "20", "--seed", "3", "--batch", "4096", "--reshuffle",
              "--optimizer", optimizer])
    log = capsys.readouterr().out
    assert "    - Epoch: 000\tACC[val]=" in log and "    Optimization Finish" in log
    vec = open(prefix + "_vectors.txt").read().splitlines()
    assert vec[0] == "GeneSymbol\t" + "\t".join("V%d" % i for i in range(128)) and len(vec) == 7524
    assert vec[1].split("\t")[0] == genes[0] and len(vec[1].split("\t")) == 129
    assert all(re.match(r"^-?\d+\.\d{6}$", x) for x in vec[1].split("\t")[1:])
    lg = open(prefix + "_lgroups.txt").read().splitlines()
    assert lg[0] == "GeneSymbol\tLgroup(0:good,1:poor,2:other)" and len(lg) == 7524
    assert {l.split("\t")[1] for l in lg[1:]} <= {"0", "1", "2"}
    bm = open(prefix + "_biomarkers.txt").read().splitlines()
    assert bm[0] == "GeneSymbol" and 1 <= len(bm) - 1 <= 40 and bm[1:] == sorted(bm[1:])
