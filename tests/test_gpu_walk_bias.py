"""node2vec's in-out bias on the H100: walk_bias_kernel on every route ({plain CSR, {col, qw} pairs, packed 16+16-bit
edges} x {bitmap, hash set} x {visit order, canonical}) bit-exact against the biased oracle (tests/walk_bias_oracle.c),
the forced biased kernel at equal multipliers against the unbiased kernels, q = 1 on the unchanged launches, walker
shards, and the command line."""
import os

import numpy as np
import pytest

import oracle
from tests import helpers
from tests import walk_bias_graphs as wbg
from tests import walk_bias_oracle as wbo
from tests import walk_edge_graphs as weg

pytestmark = pytest.mark.gpu

PAIRS = [(256, 128), (64, 256), (256, 1), (1, 256), (256, 85), (256, 256)]
BIAS_ROUTES = [r for r in weg.ROUTES if not r.startswith("e4w2")]      # the biased walk has no two-walker kernel


@pytest.fixture(scope="module")
def g2v():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import g2vec_b200
    return g2vec_b200


class _Env:
    def __init__(self, env):
        self.env = env

    def __enter__(self):
        self.saved = {k: os.environ.get(k) for k in self.env}
        os.environ.update(self.env)

    def __exit__(self, *a):
        for k, v in self.saved.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v


def run_biased(g2v, g, L, seed, group, route, b, e, s, a_near, a_far, force=True):
    """one launch of the biased entry point of the route (G2V_WALK_BIAS=kernel: the biased kernel even at equal
    multipliers) -> (nodes, lens, keys or None) as NumPy arrays"""
    import torch
    from g2vec_b200 import _capi, walks
    edges, canon, env = weg.route_env(route)
    env = dict(env, G2V_WALK_BIAS="kernel" if force else "off")
    lib = _capi.load()
    n = walks.num_walkers(g.V, 1, b, e, s)
    nodes = torch.empty((n, L), dtype=torch.int32, device=g.device)
    lens = torch.empty((n,), dtype=torch.int32, device=g.device)
    key = torch.empty((n,), dtype=torch.int64, device=g.device) if canon else None
    st = torch.cuda.current_stream().cuda_stream
    with _Env(env):
        if edges == "csr":
            rc = lib.g2v_walk_launch_biased(g.rowptr.data_ptr(), g.col.data_ptr(), g.qw.data_ptr(), g.V, g.E, L, seed,
                                            group, b, e, s, nodes.data_ptr(), lens.data_ptr(), a_near, a_far,
                                            g._ws.data_ptr(), st)
        else:
            rc = lib.g2v_walk_launch_packed_biased(g.rows.data_ptr(), g.edges.data_ptr(), g.layout, g.V, g.E, L, seed,
                                                   group, b, e, s, nodes.data_ptr(), lens.data_ptr(),
                                                   0 if key is None else key.data_ptr(), a_near, a_far,
                                                   g._ws.data_ptr(), st)
        _capi.check(rc, "g2v_walk_launch_biased")
        torch.cuda.synchronize()
    return nodes.cpu().numpy(), lens.cpu().numpy(), (key.cpu().numpy() if canon else None)


def check(tag, nodes, lens, key, want, wl):
    assert (lens == wl).all(), tag
    if key is None:
        assert (nodes == want).all(), tag
    else:
        assert (nodes == np.sort(np.where(want < 0, weg.PAD, want), axis=1)).all(), tag
        assert (key == weg.canon_key_ref(want)).all(), tag


def graph(g2v, case, route):
    g = weg.walk_graph(g2v, case, weg.route_env(route)[0])
    assert g.layout == (2 if case.packable and weg.route_env(route)[0] != "e8" else 1), (case.name, route)
    return g


def _golden_cases():
    from oracle import legacy
    z = np.load(os.path.join(helpers.GOLDEN, "walk_small.npz"))
    out = []
    for i in range(int(z["n_cases"])):
        A = z["A%d" % i]
        L, iters, seed = (int(x) for x in z["meta%d" % i])
        rp, col, w = legacy.csr_from_dense(A)
        for grp in (0, 1):
            out.append(weg.Case("small%d_g%d" % (i, grp), rp, col, oracle.quantise_weights(w), L=L,
                                ranges=[(0, iters * A.shape[0], 1)], seed=seed, group=grp))
    for grp in (0, 1):
        rp, col, w = helpers.ex_graph(grp)
        for L in (1, 2, 3, 80, 160):
            out.append(weg.Case("ex%d_L%d" % (grp, L), rp, col, oracle.quantise_weights(w), L=L,
                                ranges=[(0, 2 * (len(rp) - 1), 1)], seed=7, group=grp))
    return out


def _route_ok(case, route):
    return not route.startswith("e4") or case.packable


GOLDEN = {c.name: c for c in _golden_cases()}
EDGE = {c.name: c for c in weg.all_cases() + wbg.all_cases()}


@pytest.mark.parametrize("name", sorted(GOLDEN))
@pytest.mark.parametrize("route", BIAS_ROUTES)
def test_goldens_bit_exact(g2v, name, route):
    c = GOLDEN[name]
    if not _route_ok(c, route):
        pytest.skip("the packed 16+16-bit layout does not admit this graph")
    g = graph(g2v, c, route)
    for pair in PAIRS:
        for rng in c.ranges:
            want, wl = wbo.walks(c.rowptr, c.col, c.qw, c.L, c.seed, c.group, *rng, *pair)
            check((name, route, pair), *run_biased(g2v, g, c.L, c.seed, c.group, route, *rng, *pair), want, wl)


@pytest.mark.parametrize("name", sorted(EDGE))
def test_edge_gadgets_bit_exact_on_every_route(g2v, name):
    c = EDGE[name]
    pairs = [(256, 256), (256, 1), (1, 256)] if name.startswith(("random", "V6553")) else PAIRS
    for route in BIAS_ROUTES:
        if not _route_ok(c, route):
            continue
        g = graph(g2v, c, route)
        for pair in pairs:
            for rng in c.ranges:
                want, wl = wbo.walks(c.rowptr, c.col, c.qw, c.L, c.seed, c.group, *rng, *pair)
                got = run_biased(g2v, g, c.L, c.seed, c.group, route, *rng, *pair)
                check((name, route, pair, rng), *got, want, wl)


@pytest.mark.parametrize("route", BIAS_ROUTES)
@pytest.mark.parametrize("a", [1, 256])
def test_forced_biased_kernel_at_equal_multipliers_is_the_unbiased_kernel(g2v, route, a):
    for name in ("ex0_L80", "ex1_L160", "small2_g1"):
        c = GOLDEN[name]
        if not _route_ok(c, route):
            continue
        g = graph(g2v, c, route)
        for rng in c.ranges:
            base = weg.run_route(g2v, g, c, route, *rng)
            got = run_biased(g2v, g, c.L, c.seed, c.group, route, *rng, a, a)
            assert (got[1] == base[1]).all() and (got[0] == base[0]).all(), (name, route, a)
            if base[2] is not None:
                assert (got[2] == base[2]).all()


def _kernels(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "walk" in e.name and "kernel" in e.name]


def test_q_one_launches_the_unbiased_kernels_and_other_q_the_biased(g2v):
    c = GOLDEN["ex0_L80"]
    g = weg.walk_graph(g2v, c, "e4")
    names = {}
    for q in (1.0, 2.0):
        names[q] = _kernels(lambda: g2v.generate_paths(g, c.L, 2, seed=7, group=0, canonical=True, q=q))
    if not names[1.0] and not names[2.0]:
        pytest.skip("torch.profiler recorded no CUDA kernels on this device")
    assert names[1.0] and all("walk_bias_kernel" not in n for n in names[1.0]), names
    assert names[2.0] and all("walk_bias_kernel" in n for n in names[2.0]), names
    a, b = g2v.generate_paths(g, c.L, 2, seed=7, group=0, q=1.0)
    want, wl = oracle.walks(c.rowptr, c.col, c.qw, c.L, 7, 0, 0, 2 * g.V)
    assert (a.cpu().numpy() == want).all() and (b.cpu().numpy() == wl).all()


@pytest.mark.parametrize("q", [0.5, 2.0, 1 / 3])
def test_generate_paths_q_equals_the_oracle_and_shards_reassemble(g2v, q):
    from g2vec_b200 import walks
    pair = walks.walk_bias(q)
    for grp in (0, 1):
        rp, col, w = helpers.ex_graph(grp)
        qw = oracle.quantise_weights(w)
        g = g2v.WalkGraph(rp, col, qw=qw)
        V, L, reps = g.V, 80, 2
        want, wl = wbo.walks(rp, col, qw, L, 3, grp, 0, reps * V, 1, *pair)
        full, fl = g2v.generate_paths(g, L, reps, seed=3, group=grp, q=q)
        assert (fl.cpu().numpy() == wl).all() and (full.cpu().numpy() == want).all()
        world = 3
        nodes = np.empty_like(want)
        lens = np.empty_like(wl)
        for r in range(world):
            a, b = g2v.generate_paths(g, L, reps, seed=3, group=grp, walker_begin=r, walker_stride=world, q=q)
            nodes[r::world] = a.cpu().numpy()
            lens[r::world] = b.cpu().numpy()
        assert (nodes == want).all() and (lens == wl).all()
        hn, hl = g2v.generate_paths_host(rp, col, qw, L, reps, seed=3, group=grp, q=q)
        assert (hn == want).all() and (hl == wl).all()
        ps = g2v.generate_pathSet(g, L, reps, seed=3, group=grp, q=q)
        assert ps == oracle.path_set(want, wl)


def test_biased_entry_points_refuse_bad_multipliers(g2v):
    from g2vec_b200 import _capi
    c = GOLDEN["small0_g0"]
    g = weg.walk_graph(g2v, c, "e4")
    for bad in ((0, 1), (1, 0), (257, 1), (1, 257), (0, 0), (2**32 - 1, 1)):
        with pytest.raises(RuntimeError):
            run_biased(g2v, g, c.L, c.seed, c.group, "e8_bitmap", 0, 4, 1, *bad)
        lib = _capi.load()
        a = np.zeros(16, np.int32)
        rc = lib.g2v_walk_host_biased(a.ctypes.data, a.ctypes.data, a.ctypes.data, 3, 0, 5, 0, 0, 0, 3, 1,
                                      a.ctypes.data, a.ctypes.data, *bad)
        assert rc != 0 and b"[1, 256]" in lib.g2v_last_error()
    for q in (0.0, float("nan"), 300.0):
        with pytest.raises(ValueError):
            g2v.generate_paths(g, c.L, 1, q=q)


def test_command_line(g2v, tmp_path, capsys, monkeypatch):
    from g2vec_b200 import cli, walks
    ef, cf, nf, _ = helpers.write_ex_tsv(tmp_path)
    base = [ef, cf, nf, None, "-r", "2", "-n", "20", "--seed", "3", "--deterministic", "-e", "20"]
    real = walks.generate_paths
    seen = []

    def spy(g, L, reps, **kw):
        out = real(g, L, reps, **kw)
        seen.append((g, L, reps, kw, out))
        return out

    files, logs = {}, {}
    for name, extra in (("off", []), ("one", ["--walk-q", "1"]), ("half", ["--walk-q", "0.5"])):
        prefix = str(tmp_path / name)
        del seen[:]
        monkeypatch.setattr(walks, "generate_paths", spy)
        cli.main([prefix if a is None else a for a in base] + extra)
        monkeypatch.setattr(walks, "generate_paths", real)
        logs[name] = capsys.readouterr().out
        files[name] = [open(prefix + s, "rb").read() for s in ("_vectors.txt", "_lgroups.txt", "_biomarkers.txt")]
        if name == "half":
            assert len(seen) == 2
            for g, L, reps, kw, (rows, lens, key) in seen:
                assert kw["q"] == 0.5 and kw["canonical"]
                rp, col, qw = (t.cpu().numpy() for t in (g.rowptr, g.col, g.qw))
                want, wl = wbo.walks(rp, col, qw.view(np.uint32), L, 3, kw["group"], 0, reps * g.V, 1, 128, 256)
                assert (lens.cpu().numpy() == wl).all()
                assert (rows.cpu().numpy() == np.sort(np.where(want < 0, weg.PAD, want), axis=1)).all()
    assert files["one"] == files["off"]
    assert "walk q" not in logs["off"] and "walk q" not in logs["one"]
    assert "effective q = 0.5" in logs["half"]
    assert all(len(f) > 0 for f in files["half"]) and files["half"][0] != files["off"][0]
    with pytest.raises(SystemExit) as e:
        cli.main([str(tmp_path / "bad") if a is None else a for a in base] + ["--walk-q=0"])
    assert e.value.code == 2 and "--walk-q" in capsys.readouterr().err
