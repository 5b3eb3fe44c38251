"""The biased walk kernel (walk_bias_kernel, node2vec's in-out bias) once per route over the forced-position gadgets
and the hub gadgets, meant to be executed under compute-sanitizer on a GPU box:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_walk_bias.py

(not a pytest test: sizes are small because the sanitizer slows kernels down).  One launch per biased route ({plain
CSR, {col, qw} pairs, packed 16+16-bit edges} x {bitmap, hash set} x {visit order, canonical}) and case, at
(a_near, a_far) = (256, 1), so that the membership search runs on every candidate; results are still checked
against the biased oracle."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import g2vec_b200 as g2v
    from tests import test_gpu_walk_bias as t
    from tests import walk_bias_graphs as wbg
    from tests import walk_bias_oracle as wbo
    from tests import walk_edge_graphs as weg

    cases = [weg.forced_case(False, weg.FORCED_GROUPS[0]), weg.forced_case(True, weg.FORCED_GROUPS[0])]
    for wide in (False, True):
        c = wbg.hub_case(wbg.HUB_GROUPS[1], wide)
        V = c.V
        c.ranges = [(s, s + 8 * V, V) for s, _, _ in c.ranges]
        cases.append(c)
    launches = 0
    for c in cases:
        for route in t.BIAS_ROUTES:
            if not t._route_ok(c, route):
                continue
            g = t.graph(g2v, c, route)
            for rng in c.ranges:
                want, wl = wbo.walks(c.rowptr, c.col, c.qw, c.L, c.seed, c.group, *rng, 256, 1)
                got = t.run_biased(g2v, g, c.L, c.seed, c.group, route, *rng, 256, 1)
                t.check((c.name, route, rng), *got, want, wl)
                launches += 1
    print("sanitizer smoke (walk bias) OK: %d cases, %d launches" % (len(cases), launches))


if __name__ == "__main__":
    main()
