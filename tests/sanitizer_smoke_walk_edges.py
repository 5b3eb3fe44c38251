"""The walk sampler's boundary gadgets (tests/walk_edge_graphs.py) once per kernel route, meant to be executed under
compute-sanitizer on a GPU box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_walk_edges.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  Forced-position gadgets up to degree
65, the layout-boundary graphs (qw 32767 / 32768 / 65536 / 65537, V 65535 / 65536 on a few walkers), the small-V
bitmaps, and graphs whose LAST packed row has each degree residue 0-5 (the loads past a row's end then meet the end
of the edge buffer).  Results are still checked against the oracle."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import g2vec_b200 as g2v
    import oracle
    from tests import walk_edge_graphs as weg

    cases = [weg.forced_case(False, weg.FORCED_GROUPS[0]), weg.forced_case(True, weg.FORCED_GROUPS[0])]
    cases += weg.layout_q_cases()
    for V in (65535, 65536):
        c = weg.layout_v_case(V)
        c.ranges = c.ranges[:1] + [(0, 8 * V, V)]
        cases.append(c)
    cases += [weg.small_v_case(V) for V in weg.SMALL_V]
    for r in range(6):
        for V in (1, 33, 1025):
            rp, col, qw = weg.packing_graph(V, r)
            cases.append(weg.Case("last_residue%d_V%d" % (r, V), rp, col, qw, L=24, ranges=[(0, 2 * V, 1)]))
    launches = 0
    for c in cases:
        runs = [(rng,) + oracle.walks(c.rowptr, c.col, c.qw, c.L, c.seed, c.group, *rng) for rng in c.ranges]
        graphs = {}
        for route in weg.routes_for(c):
            edges = weg.route_env(route)[0]
            if (edges == "e8") not in graphs:
                graphs[edges == "e8"] = weg.walk_graph(g2v, c, edges)
            g = graphs[edges == "e8"]
            for rng, want, wl in runs:
                nodes, lens, key = weg.run_route(g2v, g, c, route, *rng)
                weg.check_walks(c, route, rng, nodes, lens, key, want, wl)
                launches += 1
    print("sanitizer smoke (walk edges) OK: %d cases, %d launches" % (len(cases), launches))


if __name__ == "__main__":
    main()
