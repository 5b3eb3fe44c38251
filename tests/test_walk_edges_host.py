"""CPU checks of the walk-sampler gadget graphs (tests/walk_edge_graphs.py): each builder produces the walks it states,
the C oracle equals the pure-Python oracle on every gadget, and the random draws reach every chunk and slot the GPU
kernels split a row into."""
import functools

import numpy as np
import pytest

import oracle
from tests import walk_edge_graphs as weg


@functools.lru_cache(maxsize=None)
def cases():
    return {c.name: c for c in weg.all_cases()}


@functools.lru_cache(maxsize=None)
def oracle_runs(name):
    c = cases()[name]
    return [(rng,) + oracle.walks(c.rowptr, c.col, c.qw, c.L, c.seed, c.group, *rng) for rng in c.ranges]


def walks_by_id(name):
    out = {}
    for (b, e, s), nodes, lens in oracle_runs(name):
        for i, w in enumerate(range(b, e, s)):
            out[w] = list(nodes[i, :lens[i]])
    return out


def test_every_case_is_a_valid_csr_graph():
    for c in cases().values():
        assert c.rowptr[0] == 0 and (np.diff(c.rowptr) >= 0).all() and c.rowptr[-1] == c.E
        assert c.E == 0 or (c.col.min() >= 0 and c.col.max() < c.V)
        assert c.E == 0 or (c.qw.min() >= 1 and c.qw.max() <= weg.Q_WIDE)
        for v in range(c.V):
            r = c.col[c.rowptr[v]:c.rowptr[v + 1]]
            assert (np.diff(r) > 0).all(), (c.name, v)              # ascending, no duplicate edge
        for b, e, s in c.ranges:
            assert 0 <= b < e and s >= 1


@pytest.mark.parametrize("name", [c.name for c in weg.all_cases() if c.forced or c.prefix])
def test_forced_walks_follow_their_stated_path(name):
    c = cases()[name]
    got = walks_by_id(name)
    assert set(c.forced) | set(c.prefix) <= set(got)
    for w, path in c.forced.items():
        assert got[w] == path, (name, w)
    for w, (seq, free) in c.prefix.items():
        assert got[w][:len(seq)] == seq and len(got[w]) == len(seq) + 1 and got[w][-1] in free, (name, w)


def test_forced_gadgets_cover_every_degree_and_position():
    for wide in (False, True):
        stops, picks, halves = set(), set(), set()
        for ds in weg.FORCED_GROUPS:
            c = cases()["forced_%s_d%d" % ("wide" if wide else "pcc", max(ds))]
            deg = np.diff(c.rowptr)
            for w, path in c.forced.items():
                X = path[-1] if deg[path[-1]] else path[-2]         # the walk stops at the hub or one past it
                row = list(c.col[c.rowptr[X]:c.rowptr[X + 1]])
                if path[-1] == X:
                    stops.add(len(row))                             # T = 0 at the hub
                else:
                    picks.add((len(row), row.index(path[-1])))
                    if wide:                                        # the one unvisited neighbour has weight 1
                        assert c.qw[c.rowptr[X] + row.index(path[-1])] == 1
            halves |= {int(deg[seq[-1]]) for seq, _ in c.prefix.values()}
            # the half-visited walks draw more than one of the free neighbours
            got = walks_by_id(c.name)
            by_start = {}
            for w, (seq, free) in c.prefix.items():
                by_start.setdefault(seq[0], set()).add(got[w][-1])
            assert sum(len(v) > 1 for v in by_start.values()) >= len(by_start) // 2
        assert stops == set(weg.FORCED_DEGREES)
        assert picks == {(d, p) for d in weg.FORCED_DEGREES for p in weg.FORCED_POSITIONS + (d - 1,) if p < d}
        assert halves == {d for d in weg.FORCED_DEGREES if d > 1}             # every degree with an odd position


@pytest.mark.parametrize("name", [c.name for c in weg.all_cases()])
def test_c_oracle_equals_python_oracle(name):
    """Every forced gadget walks once; every other range is sampled (the heavy rows' T > 2^32 included: the Python
    restatement uses big integers)."""
    c = cases()[name]
    for (b, e, s), nodes, lens in oracle_runs(name):
        ids = list(range(b, e, s))
        pick = list(range(len(ids))) if len(ids) <= 300 else list(range(0, len(ids), max(1, len(ids) // 64)))
        want = oracle.walks_py(c.rowptr, c.col, c.qw, c.L, c.seed, c.group, [ids[i] for i in pick])
        for i, path in zip(pick, want):
            assert list(nodes[i, :lens[i]]) == path and (nodes[i, lens[i]:] == -1).all(), (name, ids[i])


def _hub_picks(name):
    """hub -> positions (in its row) of the neighbour each of its walks drew"""
    c = cases()[name]
    out = {}
    for (b, e, s), nodes, lens in oracle_runs(name):
        X = b % c.V
        row = c.col[c.rowptr[X]:c.rowptr[X + 1]]
        assert (lens == 2).all() and (nodes[:, 0] == X).all()
        out[X] = np.searchsorted(row, nodes[:, 1])
    return out


@pytest.mark.parametrize("name", ["random_pcc", "random_wide"])
def test_random_draws_hit_every_chunk_and_slot(name):
    """Plain CSR: chunks of 32 (two in registers, then the tail).  Packed one-walker kernel: chunks of 64, two neighbours
    per lane (pair slots).  Two-walker kernel: 64 per tile request, four per lane (quad slots)."""
    c = cases()[name]
    picks = _hub_picks(name)
    assert sorted(picks) == sorted(c.hubs) and len(picks) == len(c.hubs)
    for X, pos in picks.items():
        d = c.hubs[X]
        assert len(pos) == weg.RANDOM_REPS
        assert set(np.minimum(pos // 32, 2)) == {0, 1, 2}, (X, d)
        assert set(np.minimum(pos // 64, 2)) == ({0, 1, 2} if d > 128 else {0, 1}), (X, d)
        assert set(pos % 2) == {0, 1} and set(pos % 4) == {0, 1, 2, 3}, (X, d)
        if d > 128:
            assert set(pos // 64) == set(range((d + 63) // 64)), (X, d)   # every 64-neighbour request of the row


def test_heavy_rows_need_64_bit_totals():
    """Rows of 257-400 neighbours at 2^24: T > 2^32, and the draws past neighbour 256 are exactly those with
    rem >= 2^32."""
    c = cases()["random_wide"]
    picks = _hub_picks("random_wide")
    heavy = [X for X in c.hubs if (c.qw[c.rowptr[X]:c.rowptr[X + 1]] == weg.Q_WIDE).all()]
    assert sorted(c.hubs[X] for X in heavy) == sorted(weg.HEAVY_DEGREES)
    for X in heavy:
        T = int(c.qw[c.rowptr[X]:c.rowptr[X + 1]].astype(np.int64).sum())
        assert T > 2**32
        assert (picks[X] >= 256).sum() > 0 and (picks[X] < 256).sum() > 100
    assert sum((picks[X] >= 256).sum() for X in heavy) > 100


def test_layout_boundary_cases_admit_what_they_should():
    cs = cases()
    assert cs["qw_32768_65536"].packable
    assert cs["qw_32768_65536"].qw.min() == weg.Q_PCC_LO and cs["qw_32768_65536"].qw.max() == weg.Q_PCC_HI
    assert not cs["qw_32767"].packable and not cs["qw_65537"].packable
    assert cs["V65535"].packable and not cs["V65536"].packable
    assert cs["V65535"].col.max() == 65534 and cs["V65536"].col.max() == 65535
    # the largest packed graph's bitmap (65536 bits) is too large for two walkers per warp
    assert "e4w2" not in weg.routes_for(cs["V65535"]) and "e4w1_bitmap" in weg.routes_for(cs["V65535"])
    assert weg.routes_for(cs["V65536"]) == [r for r in weg.ROUTES if not r.startswith("e4")]
    for name in [c.name for c in cs.values() if c.packable and c.name != "V65535" and c.name != "hashL1365"]:
        assert weg.routes_for(cs[name]) == list(weg.ROUTES), name
    for name in [c.name for c in cs.values() if not c.packable]:
        assert weg.routes_for(cs[name]) == [r for r in weg.ROUTES if not r.startswith("e4")], name


def test_hash_clusters_wrap_around():
    """The chain's nodes all hash to slot H-1 (computed here with 64-bit NumPy arithmetic), so a set holding them
    fills slots H-1, 0, 1, ... and the unvisited node's lookup probes past the wrap."""
    for L, H in zip(weg.HASH_L, (64, 128, 256, 4096)):
        c = cases()["hashL%d" % L]
        assert weg.hash_size(L) == H and c.cluster[0] == H
        ids = np.array(c.cluster[1] + [c.cluster[2]], np.uint64)
        slot = ((ids * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(32 - int(np.log2(H)))
        assert (slot == H - 1).all()
        assert c.packable and max(ids) < 65535


def test_small_v_walks_reach_the_bitmap_word_edges():
    for V in weg.SMALL_V:
        c = cases()["smallV%d" % V]
        got = walks_by_id(c.name)
        multi = [set(p) for p in got.values() if len(p) > 1]
        for v in set(weg.SPECIAL + (V - 1,)):
            if v < V and V > 1:
                assert any(v in p for p in multi), (V, v)
        assert got[0] == sorted({s for s in weg.SPECIAL if s < V} | {V - 1})


def test_length_sweep_walks_reach_L():
    for L in weg.SWEEP_L:
        _, nodes, lens = oracle_runs("lenL%d" % L)[0]
        assert (lens == L).all()


def test_walker_ranges_cross_2_32_and_leave_partial_warps():
    c = cases()["walkers"]
    counts = [len(range(*r)) for r in c.ranges]
    assert set(weg.WALKER_COUNTS) <= set(counts)
    assert all(b >= 2**32 for b, _, _ in c.ranges) and any(s > 1 for _, _, s in c.ranges)
    # the walker ids' high words differ from the low ones: w % V and the Philox subsequence both see them
    assert len({b % c.V for b, _, _ in c.ranges} | {b & 0xFFFFFFFF for b, _, _ in c.ranges}) > 1


@pytest.mark.parametrize("layout", [1, 2])
def test_packed_layout_restatement(layout):
    """The NumPy restatement of g2v_walk_prepare that the GPU test compares against: begins aligned to 2 / 4, rows
    in order, pads {0, 0} / sentinel V, everything past the last row zero."""
    for V in (1, 1023, 1024, 1025, 3000):
        for r in range(6):
            rp, col, qw = weg.packing_graph(V, r)
            assert (np.diff(rp)[-1]) == min(V, r)
            rows, edges = weg.packed_layout(rp, col, qw, layout)
            rows = rows.view(np.int32).reshape(-1, 2)
            al = 4 if layout == 2 else 2
            assert (rows[:, 0] % al == 0).all() and (rows[:, 1] - rows[:, 0] == np.diff(rp)).all()
            assert (rows[1:, 0] == (rows[:-1, 1] + al - 1) // al * al).all()
            end = (int(rows[-1, 1]) + al - 1) // al * al
            if layout == 2:
                w = edges.view(np.uint32)
                for v in range(V):
                    b, e = rows[v]
                    assert (w[e:(e + 3) // 4 * 4] == V).all()
                    assert ((w[b:e] & 0xFFFF) == col[rp[v]:rp[v + 1]]).all()
                    assert ((w[b:e] >> 16) + 32768 == qw[rp[v]:rp[v + 1]]).all()
                assert (w[end:] == 0).all()
            else:
                w = edges.view(np.uint32).reshape(-1, 2)
                assert (w[end:] == 0).all()
                assert sum((w[b:e, 1] > 0).sum() for b, e in rows) == len(col)
