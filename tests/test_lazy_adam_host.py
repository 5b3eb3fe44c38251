"""CPU checks of the lazy (touched-row) Adam pieces: the oracle restatement against the dense TF1 Adam oracle, the
command line's new options, and the byte model of bench_minibatch.py."""
import os
import sys

import numpy as np

import oracle
from tests import lazy_adam_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _state(V, D, rs):
    return [rs.randn(V, D).astype(np.float32) for _ in range(4)]


def test_lazy_adam_equals_dense_adam_when_untouched_rows_are_zero():
    rs = np.random.RandomState(0)
    V, D, rows = 50, 12, [3, 7, 7, 20, 49]
    var, m, v, g = _state(V, D, rs)
    v = np.abs(v)
    out = np.setdiff1d(np.arange(V), rows)
    m[out] = 0; v[out] = 0; g[out] = 0
    a = [x.copy() for x in (var, m, v)]
    b = [x.copy() for x in (var, m, v)]
    for t in (1, 2, 3):
        lazy_adam_oracle.lazy_adam_(a[0], a[1], a[2], g, rows, 0.005, t)
        oracle.adam_(b[0], b[1], b[2], g, 0.005, t)
    for x, y in zip(a, b):
        assert (x == y).all()


def test_lazy_adam_leaves_untouched_rows_alone():
    rs = np.random.RandomState(1)
    V, D, rows = 40, 8, np.array([0, 5, 39])
    var, m, v, g = _state(V, D, rs)
    v = np.abs(v)
    a = [x.copy() for x in (var, m, v)]
    lazy_adam_oracle.lazy_adam_(a[0], a[1], a[2], g, rows, 0.005, 4)
    out = np.setdiff1d(np.arange(V), rows)
    for x, x0 in zip(a, (var, m, v)):
        assert (x[out] == x0[out]).all() and not (x[rows] == x0[rows]).all()
    dense = [x.copy() for x in (var, m, v)]
    oracle.adam_(dense[0], dense[1], dense[2], g, 0.005, 4)
    for x, y in zip(a, dense):
        assert (x[rows] == y[rows]).all()           # the touched rows take exactly the dense step


def test_touched_counts_each_gene_once():
    rowptr = np.array([0, 3, 3, 5])
    gene = np.array([4, 1, 4, 9, 1])
    assert list(lazy_adam_oracle.touched(rowptr, gene, [0, 1, 2])) == [1, 4, 9]
    assert list(lazy_adam_oracle.touched(rowptr, gene, [1])) == []


def test_cli_batch_and_optimizer_options():
    from g2vec_b200 import cli
    a = cli.parse_arguments(["E", "C", "N", "R"])
    assert a.batch == 0 and a.optimizer == "adam"
    a = cli.parse_arguments(["E", "C", "N", "R", "--batch", "4096", "--optimizer", "lazy_adam"])
    assert a.batch == 4096 and a.optimizer == "lazy_adam"


def test_minibatch_byte_model():
    import bench_minibatch as bench
    V, D, B, L = 200_000, 512, 1024, 80
    T = bench.expected_touched(V, B, L)
    assert abs(T / V - 0.336) < 0.002                              # 1 - e^(-B*L/V)
    b = bench.minibatch_bytes(V, D, B, B * L, T)
    assert b["adam"] == B * L * (8 * D + 4) + 5 * B + 32 * V * D
    assert b["lazy_adam"] == int(B * L * (4 * D + 12) + 9 * B + 24 * D * T)
    assert 0.8e9 < 24 * D * T < 0.85e9 and abs(32 * V * D - 3.28e9) < 0.01e9
    assert abs(bench.expected_touched(10_000, 16384, 80) - 10_000) < 1e-6 * 10_000   # every gene, every batch
