"""The walk sampler at its internal boundaries (tests/walk_edge_graphs.py), on every kernel instantiation that admits
each gadget graph: plain CSR x {bitmap, hash}; {col, qw} pairs x {bitmap, hash} x {visit order, canonical}; packed
16+16-bit edges with one walker per warp x {bitmap, hash} x {visit order, canonical}; packed edges with two walkers
per warp x {visit order, canonical}.  Every launch is bit-exact against the oracle, every forced walk equals its
hand-stated path, and every case asserts which kernel its hooks selected."""
import functools

import numpy as np
import pytest

import oracle
from tests import walk_edge_graphs as weg

pytestmark = pytest.mark.gpu

CASES = {c.name: c for c in weg.all_cases()}
_graphs = {}


@pytest.fixture(scope="module")
def g2v():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import g2vec_b200
    return g2vec_b200


@pytest.fixture(scope="module")
def optin(g2v):
    import torch
    return int(torch.cuda.get_device_properties(0).shared_memory_per_block_optin)


@functools.lru_cache(maxsize=None)
def oracle_runs(name):
    c = CASES[name]
    return [(rng,) + oracle.walks(c.rowptr, c.col, c.qw, c.L, c.seed, c.group, *rng) for rng in c.ranges]


def graph_for(g2v, case, route):
    edges = weg.route_env(route)[0]
    key = (case.name, edges == "e8")
    if key not in _graphs:
        if len(_graphs) >= 4:                            # the parameters run case by case: keep the recent graphs
            _graphs.clear()
        _graphs[key] = weg.walk_graph(g2v, case, edges)
    g = _graphs[key]
    assert g.layout == (2 if case.packable and edges != "e8" else 1), (case.name, route, g.layout)
    return g


@pytest.mark.parametrize("name,route", [(c.name, r) for c in CASES.values() for r in weg.routes_for(c)])
def test_gadgets_bit_exact_on_every_route(g2v, optin, name, route):
    c = CASES[name]
    edges, canon, env = weg.route_env(route)
    g = graph_for(g2v, c, route)
    layout = 0 if edges == "csr" else g.layout
    # the hooks took: launch_walk's routing (restated) selects the instantiation the route names
    assert weg.route_of(c.V, c.E, c.L, layout, canon, env["G2V_WALK_VISITED"], env["G2V_WALK_TILE"], optin) \
        == weg.intended_kernel(route)
    for rng, want, wl in oracle_runs(name):
        nodes, lens, key = weg.run_route(g2v, g, c, route, *rng)
        weg.check_walks(c, route, rng, nodes, lens, key, want, wl)


def _profiled_kernels(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    return names, {k for k in map(weg.parse_kernel_name, names) if k is not None}


# the mirror once per route, and for the hook-free routing of three graphs (two walkers per warp; the hash set at
# V = 65535; the hash set at L = 1365)
MIRROR = [("walkers", r) for r in weg.ROUTES] + [("walkers", None), ("V65535", None), ("hashL1365", None)]


@pytest.mark.parametrize("name,route", MIRROR)
def test_route_mirror_names_the_kernel_that_ran(g2v, optin, name, route):
    """torch.profiler (CUDA activity tracing) reports exactly the walk kernel that route_of predicts."""
    c = CASES[name]
    g = weg.walk_graph(g2v, c, "e4")
    b, e, s = c.ranges[0]
    if route is None:
        want = weg.route_of(c.V, c.E, c.L, g.layout, False, None, None, optin)
        fn = lambda: g2v.generate_paths(g, c.L, 1, seed=c.seed, group=c.group, walker_begin=b, walker_end=e,
                                        walker_stride=s)
    else:
        edges, canon, env = weg.route_env(route)
        g = weg.walk_graph(g2v, c, edges)
        want = weg.route_of(c.V, c.E, c.L, 0 if edges == "csr" else g.layout, canon, env["G2V_WALK_VISITED"],
                            env["G2V_WALK_TILE"], optin)
        assert want == weg.intended_kernel(route)
        fn = lambda: weg.run_route(g2v, g, c, route, b, e, s)
    names, kernels = _profiled_kernels(fn)
    if names and not kernels:
        # the activity record of a single short kernel was once missing while its cudaLaunchKernel was recorded:
        # profile the same launch once more rather than read a lost record as a routing error
        names, kernels = _profiled_kernels(fn)
    if not names:
        pytest.skip("torch.profiler recorded no CUDA events on this device: the route mirror is not cross-checked")
    assert kernels == {want}, ([n for n in names if not n.startswith("cuda")], want)


@pytest.mark.parametrize("layout", ["e8", "e4"])
@pytest.mark.parametrize("V", [1, 1023, 1024, 1025, 3000])
def test_packed_buffers_equal_their_restatement(g2v, V, layout):
    """g2v_walk_prepare's rows and edges, byte for byte: begins aligned to 2 / 4, {0, 0} pad pairs, sentinel words,
    zeros past the last row; every degree residue mod 6 as the last row, and a graph without edges."""
    graphs = [weg.packing_graph(V, r) for r in range(6)]
    graphs.append((np.zeros(V + 1, np.int32), np.zeros(0, np.int32), np.zeros(0, np.uint32)))
    for rp, col, qw in graphs:
        c = weg.Case("pack", rp, col, qw, L=8, ranges=[])
        g = weg.walk_graph(g2v, c, layout)
        assert g.layout == (2 if layout == "e4" else 1)
        rows, edges = weg.packed_layout(rp, col, qw, g.layout)
        got_rows = g.rows.cpu().numpy()[:len(rows)]
        got_edges = g.edges.cpu().numpy()[:len(edges)]
        assert len(got_edges) == len(edges)
        assert (got_rows == rows).all(), (V, len(col))
        assert (got_edges == edges).all(), (V, len(col))
