"""Spearman and biweight-midcorrelation edge weights on the GPU (g2v_corr_transform, csrc/g2v_corr.cu; DESIGN.md
§4.22) against the float64 oracle (tests/corr_oracle.py), their refusals, bit-reproducibility and invariances,
`pearson` as the unchanged path, the --min-corr cutoff through the walks, and the command line end to end."""
import os

import numpy as np
import pytest

from tests import corr_oracle as co
from tests import helpers
from tests.test_correlation_host import cohort

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

METHODS = ("spearman", "bicor")
CODE = {"spearman": 1, "bicor": 2}
# every padding step and block size the launch picks (32 .. 1024 threads) and the cap
SIZES = (1, 2, 3, 31, 32, 33, 255, 256, 257, 1000, 4096, 4097, 32768)


@pytest.fixture(scope="module")
def lib():
    from g2vec_b200 import _capi
    return _capi.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


def transform_gpu(lib, X, method):
    """g2v_corr_transform on X [S, V] -> z [S, V] (the kernel's gene-major z, transposed back)."""
    x = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).cuda()
    S, V = X.shape
    z = torch.full((V, S), float("nan"), dtype=torch.float32, device="cuda")
    assert lib.g2v_corr_transform(x.data_ptr(), S, V, CODE[method], z.data_ptr(), _st()) == 0
    torch.cuda.synchronize()
    return z.cpu().numpy().T.copy()


def zscore_gpu(lib, X):
    x = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).cuda()
    S, V = X.shape
    z = torch.empty((V, S), dtype=torch.float32, device="cuda")
    assert lib.g2v_pcc_zscore(x.data_ptr(), S, V, z.data_ptr(), _st()) == 0
    torch.cuda.synchronize()
    return z.cpu().numpy().T.copy()


def weights_gpu(lib, Z, src, dst):
    """g2v_pcc_edge_weights on z [S, V] (float32) -> w [E]."""
    S, V = Z.shape
    z = torch.from_numpy(np.ascontiguousarray(Z.T, dtype=np.float32)).cuda()
    s = torch.from_numpy(np.ascontiguousarray(src, dtype=np.int32)).cuda()
    d = torch.from_numpy(np.ascontiguousarray(dst, dtype=np.int32)).cuda()
    w = torch.empty(len(src), dtype=torch.float32, device="cuda")
    assert lib.g2v_pcc_edge_weights(z.data_ptr(), S, V, s.data_ptr(), d.data_ptr(), len(src), w.data_ptr(), _st()) == 0
    torch.cuda.synchronize()
    return w.cpu().numpy()


def _pairs(V):
    a, b = np.triu_indices(V, 1)
    return a.astype(np.int32), b.astype(np.int32)


def check_against_oracle(lib, X, method, src, dst, T=0.5):
    Z = transform_gpu(lib, X, method)
    want = co.transform(X, method)
    if method == "spearman":                   # exact sums: the oracle's z rounded once, and the host path's bits
        from g2vec_b200 import graph
        assert (Z == want.astype(np.float32)).all()
        assert (Z == graph.corr_transform(X, method)).all()
    else:
        assert (np.abs(Z.astype(np.float64) - want) <= 4 * co.U * np.maximum(1.0, np.abs(want))).all()
    w = weights_gpu(lib, Z, src, dst)
    ref = co.edge_weights(want, src, dst)
    assert np.abs(w - ref).max() <= co.EDGE_TOL
    differ = (w > T) != (ref > T)              # kept sets equal except edges within the bound of the cutoff
    assert (np.abs(ref[differ] - T) <= co.EDGE_TOL).all()
    return Z, w


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("S", SIZES)
def test_transform_random_cohorts(lib, method, S):
    V = 24 if S <= 1000 else (10 if S <= 4097 else 5)
    a, b = _pairs(V)
    for kind in ("heavy", "pairs"):
        check_against_oracle(lib, cohort(S, V, S + (kind == "pairs"), kind), method, a, b)


@pytest.mark.parametrize("method", METHODS)
def test_transform_goldens(lib, golden_dir, method):
    z = np.load(os.path.join(golden_dir, "pcc_small.npz"))
    e = np.load(os.path.join(golden_dir, "ex_expr.npz"))
    label = np.load(os.path.join(golden_dir, "ex_graph.npz"))["label"]
    for expr, lab, src, dst in ((z["expr"], z["label"], z["src"], z["dst"]), (e["expr"], label, e["src"], e["dst"])):
        for g in (0, 1):
            check_against_oracle(lib, expr[lab == g], method, src.astype(np.int32), dst.astype(np.int32))


def test_refusals_launch_nothing(lib):
    from g2vec_b200 import _capi
    x = torch.zeros(64, dtype=torch.float32, device="cuda")
    z = torch.zeros(64, dtype=torch.float32, device="cuda")
    n0 = _capi.launch_count()
    bad = [(x.data_ptr(), 32769, 1, 1, z.data_ptr()), (x.data_ptr(), 0, 1, 2, z.data_ptr()),
           (x.data_ptr(), -3, 1, 1, z.data_ptr()), (x.data_ptr(), 4, 0, 1, z.data_ptr()),
           (x.data_ptr(), 4, 4, 0, z.data_ptr()), (x.data_ptr(), 4, 4, 3, z.data_ptr()),
           (x.data_ptr(), 4, 4, -1, z.data_ptr()), (None, 4, 4, 1, z.data_ptr()), (x.data_ptr(), 4, 4, 2, None)]
    for args in bad:
        assert lib.g2v_corr_transform(*args, _st()) != 0
        assert len(lib.g2v_last_error()) > 0
    assert _capi.launch_count() == n0
    assert lib.g2v_corr_transform(x.data_ptr(), 4, 4, 1, z.data_ptr(), _st()) == 0
    assert _capi.launch_count() == n0 + 2


@pytest.mark.parametrize("S", (8, 33, 1000, 4097))
def test_bicor_mad_zero_rows_are_pcc_zscore(lib, S):
    rs = np.random.RandomState(S)
    X = rs.randn(S, 16).astype(np.float32) * 3
    for v in range(10):                          # more than half the samples at one value, the rest spread
        X[rs.permutation(S)[:S // 2 + 1 + v % 3], v] = np.float32(v - 4)
    X[:, 10] = 2.5                               # constant
    zb, zp = transform_gpu(lib, X, "bicor"), zscore_gpu(lib, X)
    flat = [v for v in range(16) if co.mad(X[:, v]) == 0]
    assert len(flat) == 11
    for v in flat:
        assert (zb[:, v].view(np.uint32) == zp[:, v].view(np.uint32)).all(), v
    for v in set(range(16)) - set(flat):
        assert not (zb[:, v] == zp[:, v]).all()


@pytest.mark.parametrize("S", (33, 1000, 4097))
def test_invariances_are_bit_exact(lib, S):
    rs = np.random.RandomState(S + 1)
    X = cohort(S, 8, S, "heavy")
    a, b = _pairs(8)
    w = {m: weights_gpu(lib, transform_gpu(lib, X, m), a, b) for m in METHODS}
    Y = X.copy()
    for v in range(8):                           # per-gene order-preserving relabelling of the values
        u, inv = np.unique(Y[:, v], return_inverse=True)
        Y[:, v] = np.sort(rs.uniform(-50, 50, size=len(u))).astype(np.float32)[inv.ravel()]
        assert len(np.unique(Y[:, v])) == len(u)
    assert (weights_gpu(lib, transform_gpu(lib, Y, "spearman"), a, b) == w["spearman"]).all()
    for m in METHODS:
        assert (weights_gpu(lib, transform_gpu(lib, -X, m), a, b) == w[m]).all()
    for k in (3, -5):
        assert (weights_gpu(lib, transform_gpu(lib, X * np.float32(2.0 ** k), "bicor"), a, b) == w["bicor"]).all()


@pytest.mark.parametrize("method", METHODS)
def test_two_runs_bit_identical(lib, method):
    X = cohort(4097, 40, 3, "heavy")
    assert (transform_gpu(lib, X, method).view(np.uint32) == transform_gpu(lib, X, method).view(np.uint32)).all()


def test_outlier_gadget():
    """One sample at 1e6 in two independent genes makes their |PCC| ~ 1; the robust coefficients stay low."""
    from g2vec_b200 import graph
    rs = np.random.RandomState(2)
    X = rs.randn(40, 2).astype(np.float32)
    assert co.weights(X, [0], [1], "pearson")[0] < 0.2
    X[0, :] = 1e6
    lab = np.zeros(40, np.int64)
    kept = {}
    for m in ("pearson", "spearman", "bicor"):
        rp, col, w = graph.group_csr_gpu(X, lab, 0, np.array([0], np.int32), np.array([1], np.int32), method=m)
        kept[m] = int(col.shape[0])
        if m != "pearson":
            assert co.weights(X, [0], [1], m)[0] < 0.3
    assert kept == {"pearson": 1, "spearman": 0, "bicor": 0}


# Profiled in a child process: CUDA activity tracing then starts and ends with that process, so the profiler
# sessions of later tests in this one are not affected by these.
_PROFILE = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
from g2vec_b200 import _capi, graph
z = np.load(sys.argv[2])
args = (z["expr"], z["label"], 0, z["src"], z["dst"])
graph.group_csr_gpu(*args)                       # load and warm up outside the profile
out = {}
for m in ("default", "pearson", "spearman", "bicor"):
    n0 = _capi.launch_count()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        graph.group_csr_gpu(*args, **({} if m == "default" else {"method": m}))
        torch.cuda.synchronize()
    names = {e.name.split("g2v::")[1].split("(")[0] for e in prof.events() if "g2v::" in e.name}
    out[m] = [sorted(names), _capi.launch_count() - n0]
print(json.dumps(out))
"""


def test_pearson_runs_only_the_pcc_kernels(golden_dir):
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-c", _PROFILE, root, os.path.join(golden_dir, "pcc_small.npz")],
                         capture_output=True, text=True, timeout=600, cwd=root)
    assert res.returncode == 0, res.stderr[-2000:]
    got = json.loads(res.stdout.strip().splitlines()[-1])
    # launches counted by the library itself: z-score + edges, or transpose + rank pass + edges
    assert {m: n for m, (_, n) in got.items()} == {"default": 2, "pearson": 2, "spearman": 3, "bicor": 3}
    if not any(names for names, _ in got.values()):
        pytest.skip("torch.profiler recorded no CUDA kernels on this device")
    pcc = ["pcc_edge_kernel", "pcc_zscore_kernel"]
    assert got["default"][0] == pcc and got["pearson"][0] == pcc
    assert got["spearman"][0] == ["corr_rank_kernel<1>", "corr_transpose_kernel", "pcc_edge_kernel"]
    assert got["bicor"][0] == ["corr_rank_kernel<2>", "corr_transpose_kernel", "pcc_edge_kernel"]


def _edge_dict(rp, col, w):
    rp, col, w = (np.asarray(t.cpu().numpy() if hasattr(t, "cpu") else t) for t in (rp, col, w))
    return {(int(s), int(d)): float(x) for s, d, x in zip(np.repeat(np.arange(len(rp) - 1), np.diff(rp)), col, w)}


@pytest.mark.parametrize("method", ("pearson",) + METHODS)
@pytest.mark.parametrize("T", (0.0, 0.3, 0.5, 0.9))
def test_min_corr_gpu_equals_host(golden_dir, method, T):
    import oracle
    from g2vec_b200 import graph, walks
    e = np.load(os.path.join(golden_dir, "ex_expr.npz"))
    label = np.load(os.path.join(golden_dir, "ex_graph.npz"))["label"]
    src, dst = e["src"].astype(np.int32), e["dst"].astype(np.int32)
    g = 1
    rp, col, w = graph.group_csr_gpu(e["expr"], label, g, src, dst, threshold=T, method=method)
    got = _edge_dict(rp, col, w)
    ref = _edge_dict(*graph.group_csr(e["expr"], label, g, src, dst, threshold=T, method=method))
    tol = 2e-6 if method == "pearson" else co.EDGE_TOL        # pearson: the host's float32 sums (test_gpu_pcc_cli)
    both = set(got) & set(ref)
    assert len(both) > 100 and max(abs(got[k] - ref[k]) for k in both) <= tol
    for k in set(got) ^ set(ref):
        assert abs((got.get(k) or ref.get(k)) - T) <= tol, k
    assert min(got.values()) > T
    if T == 0.3 and method != "pearson":
        wg = walks.WalkGraph(rp, col, weights=w)
        assert wg.layout == 1                                   # weights below 0.5: the {col, qw} pair layout
        V = len(rp) - 1
        nodes, lens = walks.generate_paths(wg, 80, 1, seed=5, group=g)
        want, wl = oracle.walks(rp.cpu().numpy(), col.cpu().numpy(), graph.quantise_weights(w.cpu().numpy()), 80, 5,
                                g, 0, V)
        assert (lens.cpu().numpy() == wl).all() and (nodes.cpu().numpy() == want).all()


def test_command_line(tmp_path, capsys, monkeypatch):
    from g2vec_b200 import cli, graph, walks
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    base = [ef, cf, nf, None, "-r", "2", "-e", "5", "-n", "20", "--seed", "3"]
    real_csr, real_walk = graph.group_csr_gpu, walks.generate_paths
    seen = {}

    def spy_csr(*a, **k):
        out = real_csr(*a, **k)
        seen.setdefault("csr", []).append((k["method"], k["threshold"]) + tuple(t.cpu().numpy() for t in out))
        return out

    def spy_walk(*a, **k):
        out = real_walk(*a, **k)
        seen.setdefault("walk", []).append(tuple(t.cpu().numpy() for t in out))
        return out

    monkeypatch.setattr(graph, "group_csr_gpu", spy_csr)
    monkeypatch.setattr(walks, "generate_paths", spy_walk)
    runs = {}
    for name, extra, line in (("sp", ["--correlation", "spearman", "--min-corr", "0.6"], "spearman (|r| > 0.6)"),
                              ("bi", ["--correlation", "bicor"], "bicor (|r| > 0.5)")):
        for run in range(2):
            prefix = str(tmp_path / ("%s%d" % (name, run)))
            seen.clear()
            cli.main([prefix if a is None else a for a in base] + extra)
            log = capsys.readouterr().out
            banner = ">>> 3. Generate random paths from each group\n    *** most time consuming step ***\n"
            assert banner + "    correlation: %s\n" % line in log
            vec = open(prefix + "_vectors.txt").read().splitlines()
            assert vec[0] == "GeneSymbol\t" + "\t".join("V%d" % i for i in range(128)) and len(vec) == 7524
            assert vec[1].split("\t")[0] == genes[0] and len(vec[1].split("\t")) == 129
            lg = open(prefix + "_lgroups.txt").read().splitlines()
            assert lg[0] == "GeneSymbol\tLgroup(0:good,1:poor,2:other)" and len(lg) == 7524
            assert {l.split("\t")[1] for l in lg[1:]} <= {"0", "1", "2"}
            bm = open(prefix + "_biomarkers.txt").read().splitlines()
            assert bm[0] == "GeneSymbol" and len(bm) > 1 and bm[1:] == sorted(bm[1:])
            assert [c[:2] for c in seen["csr"]] == [(extra[1], float(extra[3]) if len(extra) > 2 else 0.5)] * 2
            runs[name, run] = (dict(seen), np.array([[float(x) for x in l.split("\t")[1:]] for l in vec[1:]]))
        (s0, v0), (s1, v1) = runs[name, 0], runs[name, 1]
        for a, b in zip(s0["csr"], s1["csr"]):               # the same graphs, bit for bit
            for x, y in zip(a[2:], b[2:]):
                assert x.dtype == y.dtype and (x.view(np.uint8) == y.view(np.uint8)).all()
        for a, b in zip(s0["walk"], s1["walk"]):             # the same walks
            for x, y in zip(a, b):
                assert (x == y).all()
        assert np.abs(v0 - v1).max() < 1e-4
    # the two coefficients give different graphs from pearson's (the golden ex_* graph)
    gr = np.load(os.path.join(helpers.GOLDEN, "ex_graph.npz"))
    assert len(runs["bi", 0][0]["csr"][0][3]) != len(gr["col0"])
