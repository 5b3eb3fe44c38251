"""HOT PATH 1, host side: the walk sampler behind the reference's call
``generate_pathSet(adjMat, args.lenPath, args.numRepetition)`` (/root/reference/G2Vec.py:62,
324-352).  The work is done by ``g2v_walk_launch`` (csrc/g2v_walk.cu) on the current CUDA
device; this module only owns buffers (torch tensors) and the walker-range bookkeeping.
"""
import math

import numpy as np
import torch

from . import _capi, graph as _graph


def _dev(device=None):
    if not torch.cuda.is_available():
        raise RuntimeError("g2vec_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)


def _to_dev(a, dtype, device):
    if isinstance(a, torch.Tensor):
        return a.to(device=device, dtype=dtype).contiguous()
    a = np.ascontiguousarray(a)
    if dtype == torch.int32 and a.dtype == np.uint32:
        a = a.view(np.int32)           # same bits; the kernel reads uint32
    return torch.from_numpy(a).to(device=device, dtype=dtype, non_blocking=True)


class WalkGraph:
    """One group's directed weighted graph resident in HBM as CSR
    (rowptr int32 [V+1], col int32 [E] ascending per row, qw uint32 [E] stored as int32 bits)."""

    def __init__(self, rowptr, col, weights=None, qw=None, device=None):
        device = _dev(device)
        if qw is None:
            if weights is None:
                raise ValueError("need weights or qw")
            if isinstance(weights, torch.Tensor) and weights.is_cuda:
                # same rule as graph.quantise_weights (rint = round-half-even), kept on the device
                wd = weights.to(torch.float32).double()
                if wd.numel() and (not bool(torch.isfinite(wd).all()) or bool((wd < 0).any())):
                    raise ValueError("edge weights must be finite and non-negative")
                q = torch.round(wd * _graph.Q_ONE)
                q = torch.where((wd > 0) & (q < 1), torch.ones_like(q), q)
                if q.numel() and float(q.max()) > _graph.Q_MAX:
                    raise ValueError("edge weight too large to quantise")
                qw = q.to(torch.int32)
            else:
                qw = _graph.quantise_weights(np.asarray(weights.cpu() if isinstance(weights, torch.Tensor) else weights))
        self.rowptr = _to_dev(rowptr, torch.int32, device)
        self.col = _to_dev(col, torch.int32, device)
        self.qw = _to_dev(qw, torch.int32, device)
        self.V = int(self.rowptr.shape[0]) - 1
        self.E = int(self.col.shape[0])
        if self.qw.shape[0] != self.E:
            raise ValueError("col / weight length mismatch")
        self.device = device
        lib = _capi.load()
        self._ws = torch.zeros(max(int(lib.g2v_walk_workspace_bytes()), 64), dtype=torch.uint8, device=device)
        # packed layouts, built once per graph by g2v_walk_prepare: rows = {begin, end} pairs, edges = {col, qw}
        # pairs (layout 1) or 16+16-bit words, two neighbours per 8-byte load (layout 2: V <= 65535, so that node
        # ids and the sentinel id V fit 16 bits, and weights in the |PCC| range [0.5, 1])
        import ctypes
        rb, eb = ctypes.c_size_t(0), ctypes.c_size_t(0)
        _capi.check(lib.g2v_walk_packed_bytes(self.V, self.E, ctypes.byref(rb), ctypes.byref(eb)), "g2v_walk_packed_bytes")
        self.rows = torch.empty(max(rb.value, 8), dtype=torch.uint8, device=device)
        self.edges = torch.empty(max(eb.value, 8), dtype=torch.uint8, device=device)
        lay = ctypes.c_int32(0)
        with torch.cuda.device(device):
            st = torch.cuda.current_stream().cuda_stream
            _capi.check(lib.g2v_walk_prepare(self.rowptr.data_ptr(), self.col.data_ptr(), self.qw.data_ptr(), self.V,
                                             self.E, self.rows.data_ptr(), self.edges.data_ptr(), ctypes.byref(lay),
                                             self._ws.data_ptr(), st), "g2v_walk_prepare")
        self.layout = int(lay.value)

    @classmethod
    def from_dense(cls, adjMat, device=None):
        rp, col, w = _graph.csr_from_dense(adjMat)
        return cls(rp, col, weights=w, device=device)

    def nbytes(self):
        return 4 * (self.V + 1) + 8 * self.E


Q_MIN, Q_MAX = 1.0 / 256.0, 256.0          # node2vec in-out parameter q: the multipliers are integers in [1, 256]


def walk_bias(q):
    """node2vec's in-out parameter ``q`` (Grover & Leskovec 2016) -> the integer multipliers ``(a_near, a_far)``.

    A candidate that is also an out-neighbour of the previous node (distance 1) weighs ``qw * a_near``, any other
    candidate ``qw * a_far``: ``(256, rint(256 / q))`` for q >= 1 (BFS-like, stay near), ``(rint(256 q), 256)``
    below (DFS-like, move away).  Powers of two are exact; otherwise a_near / a_far is within 0.5 / min(a) of 1/q
    in relative terms.  There is no return parameter p: the walks are self-avoiding, so the move back to the
    previous node always has weight 0 and p could not change anything.  Raises ValueError unless q is finite
    and in [1/256, 256]."""
    try:
        qf = float(q)
    except (TypeError, ValueError):
        raise ValueError("q must be a number in [1/256, 256] (got %r)" % (q,))
    if not (math.isfinite(qf) and Q_MIN <= qf <= Q_MAX):
        raise ValueError("q must be finite and in [1/256, 256] (got %r)" % (q,))
    if qf >= 1.0:
        return 256, int(np.rint(256.0 / qf))
    return int(np.rint(256.0 * qf)), 256


def effective_q(q):
    """the q the integer multipliers realise: a_near / a_far"""
    a_near, a_far = walk_bias(q)
    return a_near / a_far


def num_walkers(V, reps, begin=0, end=None, stride=1):
    end = V * reps if end is None else end
    return max(0, (end - begin + stride - 1) // stride)


def generate_paths(g, len_path, reps, seed=0, group=0, walker_begin=0, walker_end=None, walker_stride=1,
                   out=None, canonical=False, plain_csr=False, q=1.0):
    """Run walkers w = walker_begin + i*walker_stride < walker_end (w = rep*V + src) of graph ``g``.

    Returns (nodes int32 [n, len_path] in VISIT order padded with -1, lens int32 [n]) as device
    tensors; asynchronous on the current stream.

    ``canonical=True`` fuses ``path = tuple(sorted(path))`` (G2Vec.py:345) into the sampler: the rows come back
    sorted ascending and padded with INT32_MAX, and a third tensor holds their 64-bit keys (what
    ``paths.canonical_rows`` would otherwise compute from the visit-order rows in a second kernel).
    ``plain_csr=True`` runs the kernel on the unpacked CSR arrays through ``g2v_walk_launch``.
    ``q`` is node2vec's in-out parameter (see ``walk_bias``); ``q == 1`` is the first-order walk and makes exactly
    the launches of the plain entry points, any other q calls the ``_biased`` ones."""
    bias = None if float(q) == 1.0 else walk_bias(q)
    lib = _capi.load()
    end = g.V * reps if walker_end is None else walker_end
    n = num_walkers(g.V, reps, walker_begin, end, walker_stride)
    if out is None:
        nodes = torch.empty((n, len_path), dtype=torch.int32, device=g.device)
        lens = torch.empty((n,), dtype=torch.int32, device=g.device)
        key = torch.empty((n,), dtype=torch.int64, device=g.device) if canonical else None
    else:
        nodes, lens = out[0], out[1]
        key = out[2] if canonical else None
        assert nodes.shape == (n, len_path) and lens.shape == (n,) and nodes.is_contiguous()
    with torch.cuda.device(g.device):
        st = torch.cuda.current_stream().cuda_stream
        if plain_csr:
            if canonical:
                raise ValueError("canonical rows need the packed graph")
            args = (g.rowptr.data_ptr(), g.col.data_ptr(), g.qw.data_ptr(), g.V, g.E, int(len_path),
                    int(seed) & (2**64 - 1), int(group), int(walker_begin), int(end), int(walker_stride),
                    nodes.data_ptr(), lens.data_ptr())
            if bias is None:
                rc = lib.g2v_walk_launch(*args, g._ws.data_ptr(), st)
            else:
                rc = lib.g2v_walk_launch_biased(*args, *bias, g._ws.data_ptr(), st)
        else:
            args = (g.rows.data_ptr(), g.edges.data_ptr(), g.layout, g.V, g.E, int(len_path), int(seed) & (2**64 - 1),
                    int(group), int(walker_begin), int(end), int(walker_stride), nodes.data_ptr(), lens.data_ptr(),
                    0 if key is None else key.data_ptr())
            if bias is None:
                rc = lib.g2v_walk_launch_packed(*args, g._ws.data_ptr(), st)
            else:
                rc = lib.g2v_walk_launch_packed_biased(*args, *bias, g._ws.data_ptr(), st)
    _capi.check(rc, "g2v_walk_launch")
    if canonical:
        return nodes, lens, key
    return nodes, lens


def generate_paths_host(rowptr, col, qw, len_path, reps, seed=0, group=0, walker_begin=0, walker_end=None,
                        walker_stride=1, q=1.0):
    """Same through ``g2v_walk_host`` (``g2v_walk_host_biased`` for q != 1): NumPy arrays in, NumPy arrays out (the
    C ABI does the copies)."""
    bias = None if float(q) == 1.0 else walk_bias(q)
    lib = _capi.load()
    rowptr = np.ascontiguousarray(rowptr, dtype=np.int32); col = np.ascontiguousarray(col, dtype=np.int32)
    qw = np.ascontiguousarray(qw, dtype=np.uint32)
    V = rowptr.shape[0] - 1
    end = V * reps if walker_end is None else walker_end
    n = num_walkers(V, reps, walker_begin, end, walker_stride)
    # page-locked result buffers: the device->host copy of the rows then runs at PCIe speed
    nodes = torch.empty((n, len_path), dtype=torch.int32, pin_memory=True).numpy()
    lens = torch.empty((n,), dtype=torch.int32, pin_memory=True).numpy()
    args = (rowptr.ctypes.data, col.ctypes.data, qw.ctypes.data, V, col.shape[0], int(len_path),
            int(seed) & (2**64 - 1), int(group), int(walker_begin), int(end), int(walker_stride),
            nodes.ctypes.data, lens.ctypes.data)
    rc = lib.g2v_walk_host(*args) if bias is None else lib.g2v_walk_host_biased(*args, *bias)
    _capi.check(rc, "g2v_walk_host")
    return nodes, lens


def generate_pathSet(adjMat, maximumLength, iterations, seed=0, group=0, q=1.0):
    """Drop-in for the reference's ``generate_pathSet(adjMat, maximumLength, iterations)``
    (G2Vec.py:324): dense adjacency (or a WalkGraph) in, ``set`` of sorted int tuples out.  ``q``: node2vec's
    in-out parameter (``walk_bias``)."""
    g = adjMat if isinstance(adjMat, WalkGraph) else WalkGraph.from_dense(adjMat)
    nodes, lens = generate_paths(g, maximumLength, iterations, seed=seed, group=group, q=q)
    nodes = nodes.cpu().numpy(); lens = lens.cpu().numpy()
    return {tuple(sorted(int(x) for x in row[:n])) for row, n in zip(nodes, lens)}
