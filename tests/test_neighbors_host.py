"""CPU checks of the nearest-genes search (DESIGN.md §4.25): the oracle of tests/nbr_oracle.py against exact rational
arithmetic and against W W^T cosines, every refusal of nearest_genes (raised before the library is loaded), the
--neighbors option and the _neighbors.txt writer."""
from fractions import Fraction

import numpy as np
import pytest

from g2vec_b200 import cli, neighbors
from tests import nbr_oracle


def _exact_chain(a, b):
    """The contract's dot with every addition rounded to float64 by hand: each product is exact as a Fraction, each
    partial sum is rounded to the nearest float64 (ties to even) through Python's float(Fraction)."""
    acc = 0.0
    for x, y in zip(a, b):
        acc = float(Fraction(acc) + Fraction(float(x)) * Fraction(float(y)))
    return acc


@pytest.mark.parametrize("m,D,seed", [(2, 1, 0), (3, 5, 1), (6, 17, 2), (9, 40, 3)])
def test_oracle_equals_the_per_pair_fraction_computation(m, D, seed):
    rs = np.random.RandomState(seed)
    W = (rs.standard_normal((m, D)) * np.exp2(rs.randint(-20, 20, size=(m, 1)))).astype(np.float32)
    W[-1] = 0.0 if m > 2 else W[-1]                     # a zero row (m > 2)
    dot = nbr_oracle.dots(W, W)
    for i in range(m):
        for j in range(m):
            assert dot[i, j] == _exact_chain(W[i], W[j])
    inv = nbr_oracle.inv_norms(W)
    for i in range(m):
        n = _exact_chain(W[i], W[i])
        assert inv[i] == (1.0 / np.sqrt(n) if n > 0 else 0.0)
    s = nbr_oracle.similarities(W)
    for i in range(m):
        for j in range(m):
            want = 0.0 if inv[i] == 0 or inv[j] == 0 else float(Fraction(float(Fraction(dot[i, j]) * Fraction(inv[i])))
                                                                  * Fraction(inv[j]))
            assert s[i, j] == want and not (s[i, j] == 0 and np.signbit(s[i, j]))
    idx, sim = nbr_oracle.nearest(W, m - 1)
    for i in range(m):
        cand = sorted((j for j in range(m) if j != i), key=lambda j: (-s[i, j], j))
        assert list(idx[i]) == cand and list(sim[i]) == [s[i, j] for j in cand]


def test_oracle_is_within_1e_12_of_the_matmul_cosines():
    rs = np.random.RandomState(4)
    W = rs.standard_normal((300, 128)).astype(np.float32)
    W64 = W.astype(np.float64)
    nrm = np.linalg.norm(W64, axis=1)
    cos = (W64 @ W64.T) / nrm[:, None] / nrm[None, :]
    assert np.abs(nbr_oracle.similarities(W) - cos).max() < 1e-12
    idx, sim = nbr_oracle.nearest(W, 10, block=64)
    assert np.abs(sim - np.take_along_axis(cos, idx, axis=1)).max() < 1e-12
    assert (np.diff(sim, axis=1) <= 0).all() and (idx != np.arange(300)[:, None]).all()


def test_oracle_orders_ties_by_index():
    W = np.array([[1, 0], [2, 0], [0, 1], [4, 0], [0, 0], [-1, 0]], np.float32)
    idx, sim = nbr_oracle.nearest(W, 5)
    assert list(idx[0]) == [1, 3, 2, 4, 5] and list(sim[0]) == [1.0, 1.0, 0.0, 0.0, -1.0]
    assert list(idx[4]) == [0, 1, 2, 3, 5] and (sim[4] == 0).all()


# ---------------------------------------------------------------------------------------------- refusals
def _no_library(monkeypatch):
    from g2vec_b200 import _capi

    def boom():
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(_capi, "load", boom)


@pytest.mark.parametrize("case", ["1d", "3d", "m0", "m1", "D0", "nan", "inf", "f32_overflow", "k0", "k_neg", "k_m",
                                  "k_65", "k_float", "k_str"])
def test_refusals_raise_before_the_library_is_loaded(case, monkeypatch):
    _no_library(monkeypatch)
    W = np.random.RandomState(0).standard_normal((100, 8)).astype(np.float32)
    k = 5
    if case == "1d":
        W = W[0]
    elif case == "3d":
        W = W.reshape(10, 10, 8)
    elif case == "m0":
        W = W[:0]
    elif case == "m1":
        W, k = W[:1], 1
    elif case == "D0":
        W = W[:, :0]
    elif case == "nan":
        W[3, 2] = np.nan
    elif case == "inf":
        W[3, 2] = -np.inf
    elif case == "f32_overflow":
        W = W.astype(np.float64); W[0, 0] = 1e300
    elif case == "k0":
        k = 0
    elif case == "k_neg":
        k = -1
    elif case == "k_m":
        W, k = W[:5], 5
    elif case == "k_65":
        k = 65
    elif case == "k_float":
        k = 2.0
    else:
        k = "3"
    with pytest.raises(ValueError):
        neighbors.nearest_genes(W, k)


def test_admitted_inputs():
    W = neighbors.check_inputs(np.ones((2, 1)), 1)
    assert W.dtype == np.float32 and W.shape == (2, 1)
    neighbors.check_inputs(np.zeros((65, 3), np.float32), 64)
    neighbors.check_inputs(np.zeros((65, 3), np.float32), np.int64(64))


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        neighbors.nearest_genes(np.ones((4, 2), np.float32), 2)


# ----------------------------------------------------------------------------------------- command line
def test_neighbors_option():
    a = cli.parse_arguments(["E", "C", "N", "R"])
    assert a.neighbors == 0 and "neighbors=0" in repr(a)
    assert cli.parse_arguments(["E", "C", "N", "R", "--neighbors", "10"]).neighbors == 10
    assert cli.parse_arguments(["E", "C", "N", "R", "--neighbors", "64"]).neighbors == 64
    for bad in ("-1", "65", "1.5", "x"):
        with pytest.raises(SystemExit):
            cli.parse_arguments(["E", "C", "N", "R", "--neighbors", bad])


def test_host_helpers():
    assert list(neighbors.genes_in_paths(np.array([-1, 0, 3, -1, 1], np.int8))) == [1, 2, 4]
    lg = np.array([0, 0, 1, 2])
    nbr = np.array([[1, 2], [0, 3], [3, 0], [2, 1]])
    assert neighbors.same_lgroup_share(lg, nbr) == 2 / 8


def test_neighbors_writer_format(tmp_path):
    p = str(tmp_path / "res")
    genes = np.array(["A1CF", "AAK1", "ABL1", "ACTB"])
    lgroup = np.array([1, 2, 0, 0])
    sub = np.array([0, 2, 3])                           # AAK1 is in no path
    idx = np.array([[2, 1], [2, 0], [0, 1]], np.int32)  # positions in sub
    sim = np.array([[0.5, -0.25], [1.0, 1 / 3.0], [-0.0, -1.0]])
    cli.write_neighbors(p, genes, lgroup, sub, idx, sim)
    assert open(p + "_neighbors.txt").read() == (
        "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tRank\tNeighbor\tNeighborLgroup\tCosine\n"
        "A1CF\t1\t1\tACTB\t0\t0.500000\n"
        "A1CF\t1\t2\tABL1\t0\t-0.250000\n"
        "ABL1\t0\t1\tACTB\t0\t1.000000\n"
        "ABL1\t0\t2\tA1CF\t1\t0.333333\n"
        "ACTB\t0\t1\tA1CF\t1\t-0.000000\n"
        "ACTB\t0\t2\tABL1\t0\t-1.000000\n")
