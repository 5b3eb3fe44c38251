"""node2vec's in-out bias of the walk sampler, CPU side: the q -> (a_near, a_far) map and its refusals (library and
command line), the biased oracle (C against pure Python, equal multipliers against the unbiased oracle), and the
oracle's transition frequencies against the exact probabilities of the integer rule, including the direction of the
bias on a ring of cliques."""
import math

import numpy as np
import pytest

import oracle
from tests import helpers
from tests import walk_bias_oracle as wbo
from tests import walk_edge_graphs as weg

PAIRS = [(256, 128), (64, 256), (256, 1), (1, 256), (256, 85), (256, 256), (3, 7)]


# ------------------------------------------------------------------------------------------------ q -> multipliers
@pytest.mark.parametrize("q,want", [(1.0, (256, 256)), (2.0, (256, 128)), (0.5, (128, 256)), (4, (256, 64)),
                                    (0.25, (64, 256)), (256.0, (256, 1)), (1 / 256, (1, 256)), (3.0, (256, 85)),
                                    (1 / 3, (85, 256)), (1.5, (256, 171)), (0.7, (179, 256)), (255.0, (256, 1)),
                                    (171.0, (256, 1)), (170.0, (256, 2))])
def test_walk_bias_maps_q_to_multipliers(q, want):
    from g2vec_b200 import walks
    assert walks.walk_bias(q) == want
    a_near, a_far = want
    assert all(isinstance(a, int) and 1 <= a <= 256 for a in want)
    if q in (1.0, 2.0, 0.5, 4, 0.25, 256.0, 1 / 256):             # powers of two are exact
        assert walks.effective_q(q) == q
    # rint: the rounded multiplier is within 0.5 of 256 / q (q >= 1) or 256 q (q < 1)
    if q >= 1:
        assert a_near == 256 and abs(a_far - 256 / q) <= 0.5
    else:
        assert a_far == 256 and abs(a_near - 256 * q) <= 0.5


@pytest.mark.parametrize("q", [0.0, -1.0, -0.5, float("nan"), float("inf"), -float("inf"), 256.0001, 1000.0,
                               1 / 256 * 0.999, 1e-9, "abc", None])
def test_walk_bias_refuses(q):
    from g2vec_b200 import walks
    with pytest.raises(ValueError):
        walks.walk_bias(q)


def _parse(extra):
    from g2vec_b200 import cli
    return cli.parse_arguments(["E", "C", "N", "R"] + extra)


def test_walk_q_option_defaults_to_one_and_parses():
    assert _parse([]).walk_q == 1.0
    assert _parse(["--walk-q", "0.5"]).walk_q == 0.5
    assert _parse(["--walk-q", "256"]).walk_q == 256.0
    assert _parse(["--walk-q=0.00390625"]).walk_q == 1 / 256


@pytest.mark.parametrize("bad", ["0", "-1", "nan", "inf", "-inf", "256.5", "0.003", "x"])
def test_walk_q_option_refuses(bad, capsys):
    with pytest.raises(SystemExit) as e:
        _parse(["--walk-q=" + bad])
    assert e.value.code == 2 and "--walk-q" in capsys.readouterr().err


# --------------------------------------------------------------------------------------------------- the oracle
def _small_graphs():
    out = []
    for V, deg, seed in ((12, 3, 1), (30, 5, 2), (60, 8, 3), (25, 12, 4)):
        rp, col, w = helpers.random_graph(V, deg, seed)
        out.append(("random%d" % V, rp, col, oracle.quantise_weights(w)))
    rs = np.random.RandomState(5)
    rp, col, w = helpers.random_graph(40, 6, 6)
    qw = rs.randint(1, (1 << 24) + 1, size=len(col)).astype(np.uint32)          # the whole quantised range
    qw[::7] = 1 << 24
    out.append(("wide40", rp, col, qw))
    return out


@pytest.mark.parametrize("pair", PAIRS)
def test_c_oracle_equals_python_on_random_graphs(pair):
    for name, rp, col, qw in _small_graphs():
        V = len(rp) - 1
        for L, seed, group in ((2, 3, 0), (8, 11, 1), (40, 0x5EED, 1)):
            nodes, lens = wbo.walks(rp, col, qw, L, seed, group, 0, 3 * V, 1, *pair)
            py = wbo.walks_py(rp, col, qw, L, seed, group, range(3 * V), *pair)
            for i, p in enumerate(py):
                assert list(nodes[i, :lens[i]]) == p, (name, L, pair, i)
                assert (nodes[i, lens[i]:] == -1).all()


def _gadget_cases():
    """the edge gadgets small enough for the pure-Python restatement"""
    cs = [weg.forced_case(False, weg.FORCED_GROUPS[0]), weg.forced_case(True, weg.FORCED_GROUPS[1]),
          weg.hash_case(21), weg.walker_count_case(), weg.length_case(33), weg.small_v_case(65)]
    return {c.name: c for c in cs}


@pytest.mark.parametrize("pair", [(256, 128), (1, 256), (256, 1), (256, 256)])
def test_c_oracle_equals_python_on_edge_gadgets(pair):
    for c in _gadget_cases().values():
        for b, e, s in c.ranges[:3]:
            ids = list(range(b, e, s))[:64]
            nodes, lens = wbo.walks(c.rowptr, c.col, c.qw, c.L, c.seed, c.group, ids[0], ids[-1] + 1, s, *pair)
            py = wbo.walks_py(c.rowptr, c.col, c.qw, c.L, c.seed, c.group, ids, *pair)
            for i, p in enumerate(py):
                assert list(nodes[i, :lens[i]]) == p, (c.name, pair, i)


@pytest.mark.parametrize("a", [1, 2, 7, 128, 256])
def test_equal_multipliers_are_the_unbiased_walk(a):
    """scale invariance: the first prefix P_k > floor(x T / 2^64) is the first P_k > x T / 2^64, so scaling every
    weight by the same a picks the same neighbour"""
    graphs = [(n, rp, col, qw, 40, [(0, 3 * (len(rp) - 1), 1)], 9, 1) for n, rp, col, qw in _small_graphs()]
    for g in (0, 1):
        rp, col, w = helpers.ex_graph(g)
        graphs.append(("ex%d" % g, rp, col, oracle.quantise_weights(w), 80, [(0, 2 * (len(rp) - 1), 1)], 7, g))
    for c in weg.all_cases():
        graphs.append((c.name, c.rowptr, c.col, c.qw, c.L, c.ranges, c.seed, c.group))
    for name, rp, col, qw, L, ranges, seed, group in graphs:
        for rng in ranges:
            want, wl = oracle.walks(rp, col, qw, L, seed, group, *rng)
            got, gl = wbo.walks(rp, col, qw, L, seed, group, *rng, a, a)
            assert (gl == wl).all() and (got == want).all(), (name, rng, a)


def test_step_zero_is_unbiased():
    """L = 2: only the first step is drawn, and it ignores the multipliers"""
    for name, rp, col, qw in _small_graphs():
        V = len(rp) - 1
        want, wl = oracle.walks(rp, col, qw, 2, 5, 0, 0, 4 * V)
        for pair in PAIRS:
            got, gl = wbo.walks(rp, col, qw, 2, 5, 0, 0, 4 * V, 1, *pair)
            assert (gl == wl).all() and (got == want).all(), (name, pair)


# ------------------------------------------------------------------------------------------------- statistics
def _paths_with_probs(rp, col, qw, start, L, pair):
    """every walk of at most L nodes from `start` with its exact probability under the integer rule"""
    out = {}

    def rec(path, p):
        if len(path) == L:
            out[tuple(path)] = out.get(tuple(path), 0.0) + p
            return
        probs = wbo.step_probs(rp, col, qw, path, *pair)
        if not probs:
            out[tuple(path)] = out.get(tuple(path), 0.0) + p
            return
        for x, px in probs.items():
            if px > 0:
                rec(path + [x], p * px)

    rec([start], 1.0)
    return out


def _chi2_pvalue(rp, col, qw, start, L, pair, n_walkers, seed):
    from scipy import stats
    V = len(rp) - 1
    exact = _paths_with_probs(rp, col, qw, start, L, pair)
    assert abs(sum(exact.values()) - 1.0) < 1e-9
    nodes, lens = wbo.walks(rp, col, qw, L, seed, 0, start, start + n_walkers * V, V, *pair)
    counts = {}
    for row, n in zip(nodes, lens):
        k = tuple(int(x) for x in row[:n])
        assert k in exact, k
        counts[k] = counts.get(k, 0) + 1
    keys = sorted(exact, key=lambda k: exact[k])
    obs, exp, o_acc, e_acc = [], [], 0, 0.0
    for k in keys:                               # merge the rarest paths until every bin expects >= 5
        o_acc += counts.get(k, 0)
        e_acc += exact[k] * n_walkers
        if e_acc >= 5:
            obs.append(o_acc); exp.append(e_acc); o_acc, e_acc = 0, 0.0
    if e_acc > 0:
        obs[-1] += o_acc; exp[-1] += e_acc
    exp = np.array(exp) * (n_walkers / np.sum(exp))
    return stats.chisquare(obs, exp).pvalue, exact, counts


@pytest.mark.parametrize("pair", [(256, 64), (64, 256), (256, 85), (256, 1)])
def test_transition_frequencies_match_the_exact_probabilities(pair):
    rp, col, w = helpers.random_graph(9, 4, 17, dead_frac=0.0)
    qw = oracle.quantise_weights(w)
    p, _, _ = _chi2_pvalue(rp, col, qw, 0, 4, pair, 20000, seed=101)
    assert p > 1e-4, (pair, p)


def _ring_of_cliques(k=6, m=5):
    """k cliques of m nodes (every ordered pair an edge); node 0 of each clique, its gate, also links both ways to
    the gates of the two neighbouring cliques.  Equal weights."""
    adj = {v: set() for v in range(k * m)}
    for c in range(k):
        nodes = range(c * m, (c + 1) * m)
        for a in nodes:
            adj[a] |= {b for b in nodes if b != a}
        g, nxt = c * m, ((c + 1) % k) * m
        adj[g].add(nxt)
        adj[nxt].add(g)
    V = k * m
    rp = np.zeros(V + 1, np.int32)
    rp[1:] = np.cumsum([len(adj[v]) for v in range(V)])
    col = np.array([b for v in range(V) for b in sorted(adj[v])], np.int32)
    return rp, col, np.full(len(col), 65536, np.uint32), m


def test_ring_of_cliques_q_above_one_stays_and_below_one_leaves():
    """From a non-gate node of clique 0 the walk steps to the gate (sometimes), then either stays in the clique
    (distance 1 from the previous node: a_near) or crosses to a neighbouring gate (distance 2: a_far).  q = 4 must
    leave less often than q = 1, and q = 1/4 more often, as the exact probabilities say."""
    from g2vec_b200 import walks
    rp, col, qw, m = _ring_of_cliques()
    start, L, n = 1, 6, 40000

    def left(nodes, lens):
        """fraction of walks that reach a node outside clique 0"""
        return float(np.mean([(row[:k] >= m).any() for row, k in zip(nodes, lens)]))

    frac = {}
    for q in (4.0, 1.0, 0.25):
        pair = walks.walk_bias(q)
        p, exact, _ = _chi2_pvalue(rp, col, qw, start, L, pair, n, seed=7)
        assert p > 1e-4, (q, p)
        want = sum(pr for path, pr in exact.items() if any(x >= m for x in path))
        nodes, lens = wbo.walks(rp, col, qw, L, 7, 0, start, start + n * len(rp[:-1]), len(rp) - 1, *pair)
        frac[q] = left(nodes, lens)
        assert abs(frac[q] - want) < 5 * math.sqrt(want * (1 - want) / n) + 1e-9, (q, frac[q], want)
    assert frac[4.0] < frac[1.0] < frac[0.25], frac
