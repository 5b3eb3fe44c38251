"""Best-of-R k-means (k = 3) restarts of the L-groups on the GPU, with each gene's L-group agreement across the restarts
(DESIGN.md §4.26).

Contract (the result is bit-identical to tests/kmeans_oracle.py whatever the grid or the chunking of the restarts).
Rows x_i = float64(W_i); dist(i, c) is the float64 chain acc = acc + t*t, t = x_id - c_d, over d ascending from +0, each
operation rounded separately.  Restart r draws u_t = draw64(seed, 2^62 + r, t), t = 0, 1, 2:
* seeding (k-means++ by an integer inverse CDF): centre 0 is row floor(u_0 n / 2^64); centre t is row floor(u_t n / 2^64)
  if max D = 0, else the smallest i whose inclusive prefix sum of q exceeds floor(u_t Q / 2^64), where D_i is the min of
  dist over the centres so far, q_i = floor(2^32 fl(D_i / max D)) and Q = sum q_i;
* Lloyd, it = 1 .. max_iter: a_i = argmin_c dist(i, C_c) (ties: the lower c), m_i its distance; stop if it > 1, the
  assignment is the previous one and no cluster is empty; else C = the cluster means, each sum a chain inside blocks of
  BLOCK consecutive rows and then over the block partials in ascending order, divided by the count once, and each empty
  cluster, in ascending c, moved to a distinct row of largest m_i (ties: the lowest i).  At it = max_iter the restart
  stops without an update.  Its result is the last assignment, the centres it was measured against, n_iter = it and
  inertia = sum m_i in the same blocked order;
* the best restart r* has the lowest inertia (ties: the lowest r).  Each restart's labels are matched to r*'s by the
  permutation of {0, 1, 2} with the most agreeing genes (ties: the first in itertools.permutations order); a gene's
  agreement is the share of restarts whose matched label equals r*'s.  r*'s clusters are named by name_lgroups.

Device side (csrc/g2v_km.cu): per chunk of restarts g2v_km_seed and g2v_km_assign for the seeding, then per iteration
g2v_km_assign, g2v_km_blocks and g2v_km_update over the restarts still running (one synchronisation per iteration reads
which are done); then g2v_km_contingency and g2v_km_agree for the agreement.
"""
import itertools
from collections import namedtuple

import numpy as np

MAX_GENES = 1 << 30          # G2V_KM_MAX_GENES
MAX_RESTARTS = 1024          # G2V_KM_MAX_RESTARTS
BLOCK = 256                  # G2V_KM_BLOCK: rows per block of the blocked sums
MAX_ITER = 300               # scikit-learn's KMeans default
PERMUTATIONS = list(itertools.permutations((0, 1, 2)))

KMeansResult = namedtuple("KMeansResult", "labels centres inertia n_iter seeds best agreement lgroups reach")
KMeansResult.__doc__ = """kmeans_lgroups' result, R restarts over n genes of dimension D:
labels     int8 [R, n]: each restart's last assignment;
centres    float64 [R, 3, D]: the centres that assignment was measured against;
inertia    float64 [R]; n_iter: int32 [R], the iteration at which each restart stopped;
seeds      int32 [R, 3]: the rows k-means++ picked, in seeding order (= cluster index);
best       r*, the restart of lowest inertia (ties: the lowest r);
agreement  float64 [n]: the share of restarts that put the gene in r*'s cluster after matching;
lgroups    int32 [n]: r*'s clusters named 0 (good), 1 (poor), 2 (other) by name_lgroups;
reach      the number of restarts whose matched partition is r*'s for every gene."""


def check_inputs(W, restarts):
    """ValueError unless the restarts can run: W 2-D [n, D] with 3 <= n <= 2^30 and D >= 1, every value finite in
    float32, and restarts an integer in [1, 1024].  Returns W as a C-contiguous float32 array.  Needs no GPU."""
    W = np.asarray(W)
    if W.ndim != 2:
        raise ValueError("k-means: W must be a 2-D array [genes, dimensions], got shape %s" % (W.shape,))
    n, D = W.shape
    if not 3 <= n <= MAX_GENES:
        raise ValueError("k-means: n = %d genes, must be in [3, %d]" % (n, MAX_GENES))
    if D < 1:
        raise ValueError("k-means: W has no dimensions")
    with np.errstate(over="ignore", invalid="ignore"):
        W = np.ascontiguousarray(W, dtype=np.float32)
    if not np.isfinite(W).all():
        raise ValueError("k-means: every value of W must be finite in float32")
    R = int(restarts) if isinstance(restarts, (int, np.integer)) else None
    if R is None or not 1 <= R <= MAX_RESTARTS:
        raise ValueError("k-means: restarts must be an integer in [1, %d], got %r" % (MAX_RESTARTS, restarts))
    return W


def name_lgroups(labels):
    """L-groups from k = 3 cluster labels, the rule of G2Vec.py:167-200 as reproduced: the largest cluster (ties: the
    lower index) becomes 2 (other); of the other two, in ascending index, the first becomes 1 (poor) and the second 0
    (good).  The reference's good/poor vote compares a list with 0 and so never decides (DESIGN.md §1)."""
    labels = np.asarray(labels)
    sizes = [int(np.count_nonzero(labels == k)) for k in range(3)]
    largest = 0
    for k in (1, 2):
        if sizes[k] > sizes[largest]:
            largest = k
    rest = [k for k in (0, 1, 2) if k != largest]
    poor_c, good_c = rest[0], rest[1]
    out = np.zeros(labels.shape[0], dtype=np.int32)
    out[labels == good_c] = 0
    out[labels == poor_c] = 1
    out[labels == largest] = 2
    return out


def match(table):
    """The permutation p of {0, 1, 2} that maximises sum_c table[c, p[c]] (ties: the first in PERMUTATIONS order) and
    that sum.  table[a, b] = #{i : a_i = a, best_i = b}."""
    table = np.asarray(table)
    best, hits = None, -1
    for p in PERMUTATIONS:
        h = int(table[0, p[0]] + table[1, p[1]] + table[2, p[2]])
        if h > hits:
            best, hits = p, h
    return best, hits


def chunk_restarts(n, D, restarts, max_chunk_bytes):
    """Restarts per chunk: each needs its labels, distances, centres and block partials within max_chunk_bytes."""
    nb = -(-n // BLOCK)
    per = 9 * n + 24 * D + nb * (24 * D + 20) + 64
    return int(max(1, min(int(restarts), int(max_chunk_bytes) // per)))


def summary(res):
    """The k-means line of the command line (without its indentation)."""
    R = res.labels.shape[0]
    return ("k-means: best of %d restarts on the GPU: inertia %.6g (restart %d, %d iterations); %d of %d restarts "
            "reach its partition; %.1f %% of the genes agree in every restart"
            % (R, res.inertia[res.best], res.best, res.n_iter[res.best], res.reach, R,
               100.0 * float((res.agreement == 1.0).mean())))


def kmeans_lgroups(W, restarts, seed=0, max_iter=MAX_ITER, max_chunk_bytes=None):
    """R k-means (k = 3) restarts of the rows of W on the GPU, the best of them and each gene's agreement.

    W: host float32 array [n, D]; restarts: 1 <= R <= 1024; seed: the Philox key (--seed); max_iter >= 1 Lloyd
    iterations at most; max_chunk_bytes: bound on the device memory of one chunk of restarts (default: half the free
    device memory).  Returns a KMeansResult (see the module docstring for the exact contract); ValueError (before
    anything is uploaded) on inputs check_inputs refuses; RuntimeError without a CUDA device."""
    W = check_inputs(W, restarts)
    R = int(restarts)
    if not isinstance(max_iter, (int, np.integer)) or max_iter < 1:
        raise ValueError("k-means: max_iter must be an integer >= 1, got %r" % (max_iter,))
    max_iter = int(max_iter)
    import torch
    from . import _capi
    lib = _capi.load()
    if not torch.cuda.is_available():
        raise RuntimeError("g2vec_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    dev = torch.device("cuda", torch.cuda.current_device())
    n, D = W.shape
    nb = -(-n // BLOCK)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    if max_chunk_bytes is None:
        max_chunk_bytes = torch.cuda.mem_get_info(dev)[0] // 2
    Rc = chunk_restarts(n, D, R, max_chunk_bytes)
    st = torch.cuda.current_stream(dev).cuda_stream
    Wd = torch.from_numpy(W).to(dev)
    labels_d = torch.empty((Rc, n), dtype=torch.int8, device=dev)
    mind = torch.empty((Rc, n), dtype=torch.float64, device=dev)
    centres_d = torch.empty((Rc, 3, D), dtype=torch.float64, device=dev)
    psum = torch.empty((Rc, nb, 3, D), dtype=torch.float64, device=dev)
    pcnt = torch.empty((Rc, nb, 3), dtype=torch.int32, device=dev)
    pin = torch.empty((Rc, nb), dtype=torch.float64, device=dev)
    flags = torch.empty(Rc, dtype=torch.int32, device=dev)
    state = torch.empty(Rc, dtype=torch.int32, device=dev)
    inertia_d = torch.empty(Rc, dtype=torch.float64, device=dev)
    n_iter_d = torch.empty(Rc, dtype=torch.int32, device=dev)
    seeds_d = torch.empty((Rc, 3), dtype=torch.int32, device=dev)
    labels = np.empty((R, n), dtype=np.int8)
    centres = np.empty((R, 3, D), dtype=np.float64)
    inertia = np.empty(R, dtype=np.float64)
    n_iter = np.empty(R, dtype=np.int32)
    seeds = np.empty((R, 3), dtype=np.int32)
    p = lambda t: t.data_ptr()
    for r0 in range(0, R, Rc):
        k = min(Rc, R - r0)
        labels_d.fill_(-1)
        centres_d.zero_()
        flags.zero_()
        state.zero_()
        active = torch.arange(k, dtype=torch.int32, device=dev)
        _capi.check(lib.g2v_km_seed(p(Wd), n, D, None, seed, r0, 0, k, p(centres_d), p(seeds_d), st), "g2v_km_seed")
        for t in (1, 2):
            _capi.check(lib.g2v_km_assign(p(Wd), n, D, p(centres_d), t, p(active), k, None, p(mind), None, st),
                        "g2v_km_assign")
            _capi.check(lib.g2v_km_seed(p(Wd), n, D, p(mind), seed, r0, t, k, p(centres_d), p(seeds_d), st),
                        "g2v_km_seed")
        n_active = k
        for it in range(1, max_iter + 1):
            _capi.check(lib.g2v_km_assign(p(Wd), n, D, p(centres_d), 3, p(active), n_active, p(labels_d), p(mind),
                                          p(flags), st), "g2v_km_assign")
            _capi.check(lib.g2v_km_blocks(p(Wd), p(labels_d), p(mind), n, D, p(active), n_active, p(psum), p(pcnt),
                                          p(pin), st), "g2v_km_blocks")
            _capi.check(lib.g2v_km_update(p(Wd), p(mind), p(psum), p(pcnt), p(pin), n, D, p(active), n_active, it,
                                          max_iter, p(flags), p(centres_d), p(state), p(inertia_d), p(n_iter_d), st),
                        "g2v_km_update")
            running = np.flatnonzero(state[:k].cpu().numpy() == 0).astype(np.int32)   # the one sync per iteration
            if running.size == 0:
                break
            n_active = int(running.size)
            active = torch.from_numpy(running).to(dev)
        labels[r0:r0 + k] = labels_d[:k].cpu().numpy()
        centres[r0:r0 + k] = centres_d[:k].cpu().numpy()
        inertia[r0:r0 + k] = inertia_d[:k].cpu().numpy()
        n_iter[r0:r0 + k] = n_iter_d[:k].cpu().numpy()
        seeds[r0:r0 + k] = seeds_d[:k].cpu().numpy()
    del psum, pcnt, pin, mind

    best = int(np.argmin(inertia))                     # the first of equal values
    best_d = torch.from_numpy(labels[best]).to(dev)
    count = torch.zeros(n, dtype=torch.int32, device=dev)
    table = torch.empty((Rc, 9), dtype=torch.int64, device=dev)
    perm = np.empty((Rc, 3), dtype=np.int8)
    reach = 0
    for r0 in range(0, R, Rc):
        k = min(Rc, R - r0)
        labels_d[:k].copy_(torch.from_numpy(labels[r0:r0 + k]))
        table.zero_()
        _capi.check(lib.g2v_km_contingency(p(labels_d), p(best_d), n, k, p(table), st), "g2v_km_contingency")
        for s, tab in enumerate(table[:k].cpu().numpy().reshape(k, 3, 3)):
            perm[s], hits = match(tab)
            reach += hits == n
        perm_d = torch.from_numpy(perm[:k].copy()).to(dev)
        _capi.check(lib.g2v_km_agree(p(labels_d), p(best_d), p(perm_d), n, k, p(count), st), "g2v_km_agree")
    agreement = count.cpu().numpy().astype(np.float64) / R
    return KMeansResult(labels=labels, centres=centres, inertia=inertia, n_iter=n_iter, seeds=seeds, best=best,
                        agreement=agreement, lgroups=name_lgroups(labels[best]), reach=int(reach))
