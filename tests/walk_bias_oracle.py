"""Oracles of the walk sampler with node2vec's in-out bias (``q``, ``a_near`` / ``a_far``).

* ``walks`` -- tests/walk_bias_oracle.c through ctypes, compiled with gcc into a temporary directory on first use
  (the repository tree stays untouched).  Same call and output as ``oracle.walks`` plus the two multipliers.
* ``walks_py`` -- a pure-Python restatement, to cross-check the C on small cases.
* ``step_probs`` -- the exact float64 probabilities of one biased step under the integer rule, by enumeration.
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "walk_bias_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        so = os.path.join(tempfile.gettempdir(), "g2v_walk_bias_oracle_%d_%s.so"
                          % (os.getuid(), hashlib.sha1(src).hexdigest()[:12]))
        if not os.path.exists(so):
            tmp = "%s.%d" % (so, os.getpid())
            subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-Wall", "-o", tmp, _SRC])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        i32p, u32p = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_uint32)
        L.walk_bias_oracle_walks.argtypes = [i32p, i32p, u32p, ctypes.c_int32, ctypes.c_int32, ctypes.c_uint64,
                                             ctypes.c_uint32, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                             ctypes.c_uint32, ctypes.c_uint32, i32p, i32p]
        L.walk_bias_oracle_walks.restype = ctypes.c_int
        _lib = L
    return _lib


def _p(a, ct):
    return a.ctypes.data_as(ctypes.POINTER(ct))


def walks(rowptr, col, qw, L, seed, group, walker_begin, walker_end, walker_stride, a_near, a_far):
    """C oracle. Returns (nodes int32 [n, L] in visit order padded with -1, lengths int32 [n])."""
    rowptr = np.ascontiguousarray(rowptr, np.int32)
    col = np.ascontiguousarray(col, np.int32)
    qw = np.ascontiguousarray(qw, np.uint32)
    V = rowptr.shape[0] - 1
    n = max(0, (walker_end - walker_begin + walker_stride - 1) // walker_stride)
    nodes = np.empty((n, L), np.int32)
    lens = np.empty(n, np.int32)
    rc = lib().walk_bias_oracle_walks(_p(rowptr, ctypes.c_int32), _p(col, ctypes.c_int32), _p(qw, ctypes.c_uint32),
                                      V, L, seed, group, walker_begin, walker_end, walker_stride, a_near, a_far,
                                      _p(nodes, ctypes.c_int32), _p(lens, ctypes.c_int32))
    if rc != 0:
        raise ValueError("walk_bias_oracle_walks: bad arguments")
    return nodes, lens


def candidates(rowptr, col, qw, path, a_near, a_far):
    """[(node, effective weight)] of the walker whose visited nodes are ``path`` (in visit order)"""
    cur = path[-1]
    prev_row = set(int(c) for c in col[rowptr[path[-2]]:rowptr[path[-2] + 1]]) if len(path) > 1 else None
    seen = set(path)
    out = []
    for j in range(rowptr[cur], rowptr[cur + 1]):
        c = int(col[j])
        if c in seen:
            continue
        m = 1 if prev_row is None else (a_near if c in prev_row else a_far)
        out.append((c, int(qw[j]) * m))
    return out


def walks_py(rowptr, col, qw, L, seed, group, walker_ids, a_near, a_far):
    """Pure-Python restatement (lists of visit-order paths)."""
    V = len(rowptr) - 1
    out = []
    for w in walker_ids:
        cur = int(w % V)
        subseq = (group << 40) + int(w)
        path = []
        for s in range(L):
            path.append(cur)
            if s == L - 1:
                break
            nb = candidates(rowptr, col, qw, path, a_near, a_far)
            T = sum(q for _, q in nb)
            if T == 0:
                break
            r = (oracle.draw64_py(seed, subseq, s) * T) >> 64
            acc = 0
            for c, q in nb:
                acc += q
                if acc > r:
                    cur = c
                    break
        out.append(path)
    return out


def step_probs(rowptr, col, qw, path, a_near, a_far):
    """{next node: probability} of the step after ``path``: P(x) = |{draws d : r(d) in [P_{x-1}, P_x)}| / 2^64 with
    r(d) = floor(d T / 2^64), counted exactly (d ranges over [ceil(P_{x-1} 2^64 / T), ceil(P_x 2^64 / T)))."""
    nb = candidates(rowptr, col, qw, path, a_near, a_far)
    T = sum(q for _, q in nb)
    out = {}
    acc = 0
    for c, q in nb:
        lo = -((-acc << 64) // T)
        acc += q
        hi = -((-acc << 64) // T)
        out[c] = (hi - lo) / float(1 << 64)
    return out
