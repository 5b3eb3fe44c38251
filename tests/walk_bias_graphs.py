"""Gadget graphs for the in-out bias of the walk sampler (walk_bias_kernel in csrc/g2v_walk.cu).

Each start node S has one edge, to a hub H of degree d; H's ascending row N_0 .. N_{d-1} is the previous node's row when
the walker stands on N_i, whose own row holds every other N_j (candidates inside row(H): distance 1, a_near) and
outsiders O_0 .. O_{k-1} interleaved with them in id order (distance 2, a_far).  Degrees straddle 32 and 64 (one
chunk of the plain CSR and of the packed layouts) and the hub rows straddle 32 .. 256 entries, so the membership
search runs over rows of every length class and the candidates of the chosen N_i fill one or several chunks.  Every
S is walked by 256 walkers (different Philox streams), so the draws land across all chunk positions.  Weights are
either in the |PCC| range (packed 16+16-bit layout) or 2^24 ("wide": the effective weight reaches 2^32 with
a = 256; only the plain CSR and {col, qw} pair layouts hold them).
"""
import numpy as np

from tests.walk_edge_graphs import Builder, Case, Q_WIDE

HUB_GROUPS = ((31, 32, 33), (63, 64, 65), (127, 128, 129), (255, 256, 257))
REPS = 256


def hub_case(degrees, wide, k_out=9):
    b = Builder(77 + max(degrees) + (1 if wide else 0))
    for d in degrees:
        S = b.new(start=True)[0]
        H = b.new()[0]
        # hub neighbours and outsiders interleaved in id order: ids alternate between the two sets in blocks
        ids = b.new(d + k_out)
        outs = set(ids[1::max(2, (d + k_out) // k_out)][:k_out])
        N = [x for x in ids if x not in outs]
        O = [x for x in ids if x in outs]
        w = lambda: Q_WIDE if wide else int(b.q_pcc())
        b.edge(S, H, w())
        for x in N:
            b.edge(H, x, w())
        # only some of the N_i have rows (the others are dead ends): rows at the first, middle and last positions
        for i in sorted({0, 1, d // 2, d - 2, d - 1}):
            v = N[i]
            for x in N:
                if x != v:
                    b.edge(v, x, w())
            for x in O:
                b.edge(v, x, w())
    rowptr, col, qw, _ = b.finish()
    V = len(rowptr) - 1
    K = len(b.starts)
    name = "bias_hub%d_%s" % (max(degrees), "wide" if wide else "pcc")
    return Case(name, rowptr, col, qw, L=6, ranges=[(s, s + REPS * V, V) for s in range(K)])


def all_cases():
    return [hub_case(ds, wide) for ds in HUB_GROUPS for wide in (False, True)]
