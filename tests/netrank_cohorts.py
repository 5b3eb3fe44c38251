"""Seeded cohorts of the NetRank GPU tests (tests/test_gpu_netrank.py), whose bounds were set from host oracle runs
over many seeds (DESIGN.md §4.35).

* ``bridge(seed)``: n = 60 samples (30 of each label) and G = 200 genes; genes 0..9 form a clique shifted by 1.5 SD in
  label 1, gene 10 (the bridge) is joined to the ten of them and to nothing else, and its values are the same multiset
  in both labels, so its own statistic is exactly 0; the other genes are noise on a random network.
* ``null(seed)``: n = 60, G = 300 genes of noise on a random network of 1 200 pairs, labels 30 / 30.

Host oracle runs over seeds 0..99 at B = 1000, d = 0.5: the bridge's count is at most 5 (P <= 0.006), and its own
permutation P is 1 (N_obs = 0).  Over seeds 0..59 at B = 200, d = 0.5, the null cohort's share of genes with P <= 0.05
lies in [0.017, 0.090], mean 0.050.
"""
import numpy as np

from g2vec_b200 import diffcoex

BRIDGE = 10


def _labels(rs, n0, n1):
    lab = np.array([0] * n0 + [1] * n1)
    rs.shuffle(lab)
    return lab


def bridge(seed):
    rs = np.random.RandomState(seed)
    n, G = 60, 200
    lab = _labels(rs, 30, 30)
    x = rs.standard_normal((n, G))
    x[lab == 1, :10] += 1.5
    v = rs.standard_normal(30)
    x[lab == 0, BRIDGE] = v
    x[lab == 1, BRIDGE] = rs.permutation(v)
    module = np.triu_indices(10, 1)
    src = np.r_[module[0], np.arange(10), rs.randint(11, G, 600)]
    dst = np.r_[module[1], np.full(10, BRIDGE), rs.randint(11, G, 600)]
    return x, lab, diffcoex.pairs_from_edges(src, dst)


def null(seed):
    rs = np.random.RandomState(seed)
    n, G = 60, 300
    lab = _labels(rs, 30, 30)
    x = rs.standard_normal((n, G))
    return x, lab, diffcoex.pairs_from_edges(rs.randint(0, G, 1200), rs.randint(0, G, 1200))
