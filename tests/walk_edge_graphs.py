"""CPU builders of "gadget" graphs that put the walk sampler (csrc/g2v_walk.cu) at its internal boundaries.

Each builder returns a ``Case``: one merged CSR graph (ascending columns, integer weights ``qw``), the walker ranges
to run on it, and what some of those walks must be, stated by hand:

* forced position -- hub X has d ascending neighbours N_0..N_{d-1}; a one-edge chain S -> N_i (i != p) -> X visits
  every neighbour but N_p, so the walk must be S, chain, X, N_p.  Variants: every N_i visited (T = 0 at X: the walk
  stops at X) and the even positions visited (the draw lands on an odd one).  Degrees straddle the chunk sizes of
  every kernel (32 plain CSR lanes, 64 packed neighbours, 2 chunks of 64 in registers, then the tail).
* random position -- hubs whose neighbours are dead-end leaves, each walked >= 512 times, so that the draws land in
  chunk 0, chunk 1 and the tail and in every pair / quad slot; rows of 2^24-weight neighbours with T > 2^32.
* layout boundaries (qw 32767 / 32768 / 65536 / 65537, V 65535 / 65536), small-V bitmaps, hash clusters whose
  probes wrap from slot H-1 to slot 0, partial warps, walker ids >= 2^32, and walk lengths around the Philox refills.

``route_of`` restates ``launch_walk``'s choice of kernel, so that a test can assert which instantiation ran.
"""
import os
import re
from dataclasses import dataclass, field

import numpy as np

Q_PCC_LO, Q_PCC_HI = 32768, 65536           # packed 16+16-bit edges hold exactly these weights
Q_WIDE = 1 << 24                            # largest quantised weight (g2vec_b200.graph.Q_MAX)
GOLDEN = 2654435761                         # hash_slot multiplier
PAD = 2**31 - 1                             # canonical rows' padding (g2vec_b200.paths.PAD)

FORCED_GROUPS = ((1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65), (127, 128, 129), (191, 192, 193), (255, 256, 257))
FORCED_DEGREES = tuple(d for g in FORCED_GROUPS for d in g)
FORCED_POSITIONS = (0, 1, 31, 32, 63, 64, 127, 128)
RANDOM_DEGREES = (65, 100, 128, 129, 193, 257)
HEAVY_DEGREES = (257, 300, 400)
RANDOM_REPS = 512
SMALL_V = (1, 2, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025)
HASH_L = (21, 22, 80, 1365)
WALKER_COUNTS = (1, 7, 8, 9, 15, 16, 17)
SWEEP_L = (16, 17, 32, 33, 48, 49, 64, 65)


@dataclass
class Case:
    name: str
    rowptr: np.ndarray
    col: np.ndarray
    qw: np.ndarray
    L: int
    ranges: list                            # (walker_begin, walker_end, walker_stride)
    forced: dict = field(default_factory=dict)      # walker id -> the whole walk
    prefix: dict = field(default_factory=dict)      # walker id -> (walk up to the draw, the allowed next nodes)
    hubs: dict = field(default_factory=dict)        # hub node -> its degree (random-position hubs)
    cluster: tuple = None                           # hash cases: (H, chain nodes of slot H-1, the unvisited one)
    seed: int = 0x5EED
    group: int = 1

    @property
    def V(self):
        return len(self.rowptr) - 1

    @property
    def E(self):
        return len(self.col)

    @property
    def packable(self):
        """layout 2 (packed 16+16-bit edges) admits the graph: V <= 65535 and every qw in [32768, 65536]."""
        return self.V <= 65535 and (self.E == 0 or (int(self.qw.min()) >= Q_PCC_LO and int(self.qw.max()) <= Q_PCC_HI))


class Builder:
    """Nodes are numbered at the end: walk starts first, every other node after them, each class in creation order
    (so a hub's neighbours, created in a block, stay consecutive and ascending)."""

    def __init__(self, seed):
        self.rs = np.random.RandomState(seed)
        self.n = 0
        self.starts = []
        self.adj = {}

    def new(self, k=1, start=False):
        ids = list(range(self.n, self.n + k))
        self.n += k
        if start:
            self.starts += ids
        return ids

    def edge(self, a, b, q):
        assert b not in self.adj.setdefault(a, {}), "duplicate edge"
        self.adj[a][b] = int(q)

    def q_pcc(self, k=None):
        """weights of the |PCC| in [0.5, 1] range, both ends included"""
        x = self.rs.randint(Q_PCC_LO, Q_PCC_HI + 1, size=k)
        if k is not None and k >= 4:
            x[self.rs.choice(k, 2, replace=False)] = (Q_PCC_LO, Q_PCC_HI)
        return x

    def finish(self, V=None):
        """-> (rowptr, col, qw, relabel) with relabel[provisional id] = final id"""
        n = self.n if V is None else V
        starts = set(self.starts)
        order = self.starts + [v for v in range(self.n) if v not in starts]
        relabel = np.empty(self.n, np.int64)
        relabel[order] = np.arange(self.n)
        rows = [[] for _ in range(n)]
        for a, nb in self.adj.items():
            rows[relabel[a]] = sorted((int(relabel[b]), q) for b, q in nb.items())
        rowptr = np.zeros(n + 1, np.int32)
        rowptr[1:] = np.cumsum([len(r) for r in rows])
        col = np.array([c for r in rows for c, _ in r], np.int32)
        qw = np.array([q for r in rows for _, q in r], np.uint32)
        return rowptr, col, qw, relabel


def _forced_gadget(b, d, p, mode, wide):
    """Hub with d neighbours; mode 'one' (only N_p unvisited), 'none' (all visited) or 'half' (even ones visited).
    Returns (start, walk up to X, allowed next nodes) in provisional ids."""
    S = b.new(start=True)[0]
    X = b.new()[0]
    N = b.new(d)
    if mode == "one":
        chain = [i for i in range(d) if i != p]
        free = [p]
    elif mode == "none":
        chain, free = list(range(d)), []
    else:
        chain = [i for i in range(0, d, 2)]
        free = [i for i in range(1, d, 2)]
    seq = [S] + [N[i] for i in chain] + [X]
    for a, c in zip(seq, seq[1:]):
        b.edge(a, c, Q_WIDE if wide else b.q_pcc())
    if wide:
        # visited neighbours at the largest weight, so that a neighbour wrongly left unmasked dominates the draw
        q = np.full(d, Q_WIDE, np.int64)
        if mode == "one":
            q[p] = 1
        elif mode == "half":
            q[free] = b.rs.randint(1, Q_WIDE + 1, size=len(free))
    else:
        q = b.q_pcc(d)
    for i in range(d):
        b.edge(X, N[i], q[i])
    return S, seq, [N[i] for i in free]


def forced_case(wide, degrees):
    """Every (degree, position) gadget, the all-visited and the half-visited variant of every degree.  The degrees
    come in groups so that each graph stays small enough for two walkers per warp (both tiles' bitmaps in 56 KB)."""
    b = Builder((11 if wide else 12) + max(degrees))
    gadgets = []
    for d in degrees:
        for p in sorted({p for p in FORCED_POSITIONS + (d - 1,) if p < d}):
            gadgets.append(("one", _forced_gadget(b, d, p, "one", wide)))
        gadgets.append(("none", _forced_gadget(b, d, 0, "none", wide)))
        gadgets.append(("half", _forced_gadget(b, d, 0, "half", wide)))
    rowptr, col, qw, rl = b.finish()
    V = len(rowptr) - 1
    K = len(b.starts)
    c = Case("forced_%s_d%d" % ("wide" if wide else "pcc", max(degrees)), rowptr, col, qw, L=max(degrees) + 3,
             ranges=[(0, K, 1)])
    for mode, (S, seq, free) in gadgets:
        s = int(rl[S])
        seq = [int(rl[x]) for x in seq]
        free = [int(rl[x]) for x in free]
        if mode == "one":
            c.forced[s] = seq + free
        elif mode == "none" or not free:
            c.forced[s] = seq
        else:
            c.prefix[s] = (seq, free)
            c.ranges.append((s + V, s + 16 * V, V))          # the same walk under 15 more draws
            for w in range(s + V, s + 16 * V, V):
                c.prefix[w] = (seq, free)
    return c


def random_case(wide):
    """Hubs of dead-end leaves walked RANDOM_REPS times each; the wide case adds rows of 2^24-weight neighbours whose
    total exceeds 2^32."""
    b = Builder(21 if wide else 22)
    hubs = []
    for d, heavy in [(d, False) for d in RANDOM_DEGREES] + [(d, True) for d in (HEAVY_DEGREES if wide else ())]:
        X = b.new(start=True)[0]
        leaves = b.new(d)
        if heavy:
            q = np.full(d, Q_WIDE)
        else:
            q = b.rs.randint(1, Q_WIDE + 1, size=d) if wide else b.q_pcc(d)
        for leaf, x in zip(leaves, q):
            b.edge(X, leaf, x)
        hubs.append((X, d))
    rowptr, col, qw, rl = b.finish()
    V = len(rowptr) - 1
    c = Case("random_wide" if wide else "random_pcc", rowptr, col, qw, L=4, ranges=[])
    for X, d in hubs:
        x = int(rl[X])
        c.hubs[x] = d
        c.ranges.append((x, x + RANDOM_REPS * V, V))
    return c


def _pcc_graph(V, deg, seed, dead_frac=0.1):
    rs = np.random.RandomState(seed)
    rows = []
    for v in range(V):
        k = 0 if rs.rand() < dead_frac else min(V - 1, max(1, rs.poisson(deg)))
        nb = rs.choice(V - 1, size=k, replace=False)
        rows.append(np.sort(np.where(nb >= v, nb + 1, nb)))
    rowptr = np.zeros(V + 1, np.int32)
    rowptr[1:] = np.cumsum([len(r) for r in rows])
    col = np.concatenate(rows).astype(np.int32) if rowptr[-1] else np.zeros(0, np.int32)
    qw = rs.randint(Q_PCC_LO, Q_PCC_HI + 1, size=len(col)).astype(np.uint32)
    return rowptr, col, qw


def layout_q_cases():
    """Weights at the packed layout's limits: 32768 and 65536 stay packed, one 32767 or 65537 edge does not."""
    out = []
    for odd in (None, 32767, 65537):
        rowptr, col, qw = _pcc_graph(400, 20, seed=31)
        qw[0], qw[1] = Q_PCC_LO, Q_PCC_HI
        if odd is not None:
            qw[len(qw) // 2] = odd
        out.append(Case("qw_%s" % (odd or "32768_65536"), rowptr, col, qw, L=40, ranges=[(0, 2 * 400, 1)]))
    return out


def layout_v_case(V):
    """V = 65535 (the largest packed graph: node 65534, sentinel 0xFFFF) or 65536 (pairs).  A forced walk ends on
    node V-1; a hub at node 0 reaches both ends of the id range.  Only a few walker ids run."""
    d = 65
    rs = np.random.RandomState(V)
    N = list(range(V - d, V))
    X, S = V - d - 1, V - d - 2
    edges = {}
    seq = [S] + N[:-1] + [X]
    for a, c in zip(seq, seq[1:]):
        edges[(a, c)] = rs.randint(Q_PCC_LO, Q_PCC_HI + 1)
    for c in N:
        edges[(X, c)] = rs.randint(Q_PCC_LO, Q_PCC_HI + 1)
    for c in list(range(1, 40)) + [V - 40, V - 2, V - 1]:
        edges[(0, c)] = rs.randint(Q_PCC_LO, Q_PCC_HI + 1)
    for a in range(1, 40):
        edges[(a, V - 1 - a)] = Q_PCC_HI
    src = np.array([a for a, _ in sorted(edges)], np.int64)
    col = np.array([c for _, c in sorted(edges)], np.int32)
    qw = np.array([edges[k] for k in sorted(edges)], np.uint32)
    rowptr = np.zeros(V + 1, np.int32)
    np.add.at(rowptr, src + 1, 1)
    rowptr = np.cumsum(rowptr).astype(np.int32)
    c = Case("V%d" % V, rowptr, col, qw, L=80,
             ranges=[(S, S + 1, 1), (0, 256 * V, V), (V - d - 2, V, 1)])
    c.forced[S] = seq + [V - 1]
    return c


SPECIAL = (0, 31, 32, 63, 64)


def small_v_case(V):
    """Chain through nodes 0, 31, 32, 63, 64, V-1 (those below V) that closes back on node 0 (visited: the walk stops
    there), every other node with a few random out-edges.  V = 1 is one self-loop."""
    rs = np.random.RandomState(100 + V)
    special = sorted({s for s in SPECIAL if s < V} | {V - 1})
    adj = {v: set() for v in range(V)}
    for a, c in zip(special, special[1:] + [special[0]]):
        adj[a].add(c)
    for v in range(V):
        if v in special or V == 1:
            continue
        others = [u for u in range(V) if u != v]
        adj[v] |= set(int(x) for x in rs.choice(others, size=rs.randint(0, min(len(others), 6) + 1), replace=False))
    rowptr = np.zeros(V + 1, np.int32)
    rowptr[1:] = np.cumsum([len(adj[v]) for v in range(V)])
    col = np.array([c for v in range(V) for c in sorted(adj[v])], np.int32)
    qw = rs.randint(Q_PCC_LO, Q_PCC_HI + 1, size=len(col)).astype(np.uint32)
    c = Case("smallV%d" % V, rowptr, col, qw, L=80, ranges=[(0, 4 * V, 1)])
    c.forced[0] = special
    return c


def hash_slot(c, H):
    return ((int(c) * GOLDEN) & 0xFFFFFFFF) >> (32 - (H.bit_length() - 1))


def hash_size(L):
    """the kernel's hash set: >= 3L slots, a power of two, at least 64"""
    H = 64
    while H < 3 * L:
        H <<= 1
    return H


def hash_case(L, k=5):
    """Chain c_1 .. c_k -> X of nodes whose hash slot is H-1, so that they fill slots H-1, 0, 1, ...; X's row holds
    them all and one more slot-(H-1) node u, whose lookup probes through the wrapped cluster to an empty slot."""
    H = hash_size(L)
    ids = [c for c in range(1, 65535) if hash_slot(c, H) == H - 1][:k + 1]
    assert len(ids) == k + 1
    cl, u = ids[:k], ids[k]
    V = max(ids) + 3
    X, S = V - 1, V - 2
    adj = {v: {} for v in range(V)}
    rs = np.random.RandomState(L)
    seq = [S] + cl + [X]
    for a, c in zip(seq, seq[1:]):
        adj[a][c] = rs.randint(Q_PCC_LO, Q_PCC_HI + 1)
    for c in cl + [u]:
        adj[X][c] = rs.randint(Q_PCC_LO, Q_PCC_HI + 1)
    rowptr = np.zeros(V + 1, np.int32)
    rowptr[1:] = np.cumsum([len(adj[v]) for v in range(V)])
    col = np.array([c for v in range(V) for c in sorted(adj[v])], np.int32)
    qw = np.array([adj[v][c] for v in range(V) for c in sorted(adj[v])], np.uint32)
    c = Case("hashL%d" % L, rowptr, col, qw, L=L, ranges=[(S, S + 4 * V, V)], cluster=(H, cl, u))
    for w in range(S, S + 4 * V, V):
        c.forced[w] = seq + [u]
    return c


def walker_count_case():
    """Partial last warps / tiles: walker counts around 8 (warps per CTA) and 16 (walkers per pair-kernel CTA), walker
    ids past 2^32 (the Philox subsequence's high word, w % V) and strides > 1."""
    rowptr, col, qw = _pcc_graph(300, 30, seed=41)
    base = (1 << 32) + 123
    ranges = [(base, base + n * s, s) for n in WALKER_COUNTS for s in (1, 3)]
    ranges.append(((5 << 32) + 7, (5 << 32) + 7 + 300 * 301, 301))
    return Case("walkers", rowptr, col, qw, L=40, ranges=ranges)


def length_case(L):
    """A complete 100-node digraph: every walk reaches L, across the Philox refills (every 16 steps in the pair
    kernel, every 32 in the one-walker kernel), on rows of 99 neighbours."""
    V = 100
    rs = np.random.RandomState(L)
    rowptr = (np.arange(V + 1) * (V - 1)).astype(np.int32)
    col = np.array([c for v in range(V) for c in range(V) if c != v], np.int32)
    qw = rs.randint(Q_PCC_LO, Q_PCC_HI + 1, size=len(col)).astype(np.uint32)
    return Case("lenL%d" % L, rowptr, col, qw, L=L, ranges=[(0, 2 * V, 1)])


def all_cases():
    cs = [forced_case(wide, ds) for wide in (False, True) for ds in FORCED_GROUPS]
    cs += [random_case(False), random_case(True)]
    cs += layout_q_cases() + [layout_v_case(65535), layout_v_case(65536)]
    cs += [small_v_case(V) for V in SMALL_V] + [hash_case(L) for L in HASH_L]
    cs += [walker_count_case()] + [length_case(L) for L in SWEEP_L]
    return cs


def packing_graph(V, last_residue, seed=0):
    """Degrees through every residue mod 4 and 2 (0..17), the last row's degree = last_residue (mod 6)."""
    rs = np.random.RandomState(seed + 7 * V + last_residue)
    deg = [min(V, ((v - (V - 1) + last_residue) % 6) + 6 * ((v // 6) % 3)) for v in range(V)]
    deg[-1] = min(V, last_residue)
    rows = [np.sort(rs.choice(V, size=k, replace=False)) for k in deg]
    rowptr = np.zeros(V + 1, np.int32)
    rowptr[1:] = np.cumsum(deg)
    col = np.concatenate(rows).astype(np.int32) if rowptr[-1] else np.zeros(0, np.int32)
    qw = rs.randint(Q_PCC_LO, Q_PCC_HI + 1, size=len(col)).astype(np.uint32)
    return rowptr, col, qw


def packed_layout(rowptr, col, qw, layout):
    """NumPy restatement of g2v_walk_prepare's output: rows {begin, end} int32 pairs and the edge buffer
    (layout 1: {col, qw} uint32 pairs from begins aligned to 2, {0, 0} pad pairs; layout 2: col | (qw - 32768) << 16
    words from begins aligned to 4, sentinel words V up to the next multiple of 4), both as bytes of the sizes
    g2v_walk_packed_bytes reports; everything past the last row is zero."""
    V, E = len(rowptr) - 1, len(col)
    deg = np.diff(rowptr).astype(np.int64)
    al = 4 if layout == 2 else 2
    span = (deg + al - 1) // al * al
    begin = np.concatenate([[0], np.cumsum(span)[:-1]]).astype(np.int64)
    rows = np.stack([begin, begin + deg], 1).astype(np.int32)
    nbytes = max(8 * (E + V + 4), 4 * (E + 3 * V + 8))
    if layout == 2:
        edges = np.zeros(nbytes // 4, np.uint32)
        for v in range(V):
            b, e = int(begin[v]), int(begin[v] + deg[v])
            r = slice(rowptr[v], rowptr[v + 1])
            edges[b:e] = col[r].astype(np.uint32) | ((qw[r].astype(np.uint32) - Q_PCC_LO) << 16)
            edges[e:b + int(span[v])] = V
    else:
        edges = np.zeros((nbytes // 8, 2), np.uint32)
        for v in range(V):
            b, e = int(begin[v]), int(begin[v] + deg[v])
            r = slice(rowptr[v], rowptr[v + 1])
            edges[b:e, 0] = col[r]
            edges[b:e, 1] = qw[r]
    return rows.view(np.uint8).reshape(-1), edges.view(np.uint8).reshape(-1)[:nbytes]


# ------------------------------------------------------------------------------------------------ kernel routing
ROUTES = ("csr_bitmap", "csr_hash",
          "e8_bitmap", "e8_hash", "e8_bitmap_canon", "e8_hash_canon",
          "e4w1_bitmap", "e4w1_hash", "e4w1_bitmap_canon", "e4w1_hash_canon",
          "e4w2", "e4w2_canon")


def route_env(route):
    """-> (edges 'csr' / 'e8' / 'e4', canonical, {G2V_WALK_VISITED, G2V_WALK_TILE}) forcing the route"""
    parts = route.split("_")
    canon = parts[-1] == "canon"
    if parts[0] == "e4w2":
        return "e4", canon, {"G2V_WALK_VISITED": "bitmap", "G2V_WALK_TILE": "16"}
    edges = "e4" if parts[0] == "e4w1" else parts[0]
    return edges, canon, {"G2V_WALK_VISITED": parts[1], "G2V_WALK_TILE": "32"}


def intended_kernel(route):
    """the instantiation a route names: ('pair', canon) or ('walk', bitmap, layout, canon)"""
    edges, canon, env = route_env(route)
    if route.startswith("e4w2"):
        return ("pair", canon)
    return ("walk", env["G2V_WALK_VISITED"] == "bitmap", {"csr": 0, "e8": 1, "e4": 2}[edges], canon)


def route_of(V, E, L, layout, canon, visited=None, tile=None, smem_optin=232448):
    """launch_walk's routing restated: which kernel runs for this graph, walk length and hooks."""
    Lpad = (L + 31) & ~31
    if canon:
        Lpad = 32
        while Lpad < L:
            Lpad <<= 1
    bm_words = (V + 32) // 32
    Hh = 64
    while Hh < 3 * L:
        Hh <<= 1
    per_warp = 8 * 4
    bm_smem, hash_smem = per_warp * (Lpad + bm_words), per_warp * (Lpad + Hh)
    bitmap = bm_smem <= 56 * 1024 or bm_smem <= hash_smem
    if visited and visited[0] == "h":
        bitmap = False
    if visited and visited[0] == "b" and bm_smem <= smem_optin:
        bitmap = True
    pair_smem = 2 * per_warp * (Lpad + bm_words)
    short_rows = 8 * V <= E <= 56 * V
    if layout == 2 and bitmap and pair_smem <= 56 * 1024 and (int(tile) == 16 if tile else short_rows):
        return ("pair", canon)
    return ("walk", bitmap, layout, canon)


def parse_kernel_name(name):
    """a profiler kernel name -> the tuple route_of returns (None for any other kernel)"""
    m = re.search(r"walk_(pair_)?kernel<([^>]*)>", name)
    if not m:
        return None
    vals = []
    for a in m.group(2).split(","):
        a = re.sub(r"^\(.*\)", "", a.strip()).strip()
        vals.append(1 if a == "true" else 0 if a == "false" else int(re.sub(r"[^0-9]", "", a)))
    if m.group(1):
        return ("pair", bool(vals[0]))
    return ("walk", bool(vals[0]), vals[1], bool(vals[2]))


# ------------------------------------------------------------------------------------------- running on the GPU
def walk_graph(g2v, case, edges):
    """WalkGraph of the case; edges 'e8' forces the pair layout at construction"""
    old = os.environ.pop("G2V_WALK_LAYOUT", None)
    try:
        if edges == "e8":
            os.environ["G2V_WALK_LAYOUT"] = "e8"
        return g2v.WalkGraph(case.rowptr, case.col, qw=case.qw)
    finally:
        os.environ.pop("G2V_WALK_LAYOUT", None)
        if old is not None:
            os.environ["G2V_WALK_LAYOUT"] = old


def run_route(g2v, g, case, route, b, e, s):
    """One launch with the route's hooks set -> (nodes, lens, keys or None) as NumPy arrays"""
    import torch
    edges, canon, env = route_env(route)
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        out = g2v.generate_paths(g, case.L, 1, seed=case.seed, group=case.group, walker_begin=b, walker_end=e,
                                 walker_stride=s, canonical=canon, plain_csr=(edges == "csr"))
        torch.cuda.synchronize()
    finally:
        for k, v in saved.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v
    out = [x.cpu().numpy() for x in out]
    return out[0], out[1], (out[2] if canon else None)


def canon_key_ref(want):
    """g2v_paths_canonicalise's keys of the oracle's visit-order rows"""
    import torch
    from g2vec_b200 import paths
    _, key = paths._canon(torch.from_numpy(np.ascontiguousarray(want)).cuda())
    return key.cpu().numpy()


def check_walks(case, route, rng, nodes, lens, key, want, wl):
    """GPU rows == the oracle's (visit order, or sorted + PAD with the keys of g2v_paths_canonicalise), and every
    forced walk == its hand-stated path"""
    tag = (case.name, route, rng)
    assert (lens == wl).all(), tag
    if key is None:
        assert (nodes == want).all(), tag
    else:
        assert (nodes == np.sort(np.where(want < 0, PAD, want), axis=1)).all(), tag
        assert (key == canon_key_ref(want)).all(), tag
    for i, w in enumerate(range(*rng)):
        path = case.forced.get(w)
        if path is None and w in case.prefix:
            path = case.prefix[w][0] + [int(want[i, len(case.prefix[w][0])])]
            assert path[-1] in case.prefix[w][1], tag + (w,)
        if path is not None:
            row = list(nodes[i, :lens[i]])
            assert row == (sorted(path) if key is not None else path), tag + (w,)


def routes_for(case, smem_optin=232448):
    """every route that admits the case: the packed routes need layout 2, and two walkers per warp also need both
    tiles' bitmaps within 56 KB (never at V = 65535)"""
    out = []
    for r in ROUTES:
        if r.startswith("e4") and not case.packable:
            continue
        edges, canon, env = route_env(r)
        if r.startswith("e4w2") and route_of(case.V, case.E, case.L, 2, canon, env["G2V_WALK_VISITED"],
                                             env["G2V_WALK_TILE"], smem_optin)[0] != "pair":
            continue
        out.append(r)
    return out
