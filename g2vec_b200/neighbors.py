"""Exact cosine K nearest genes of every gene in the learned embedding (DESIGN.md §4.25).

Contract, in IEEE float64 (the result is bit-exact and reproducible): dot_ij is the chain
((0 + W_i0 W_j0) + W_i1 W_j1) + ... in ascending d (a float32 product is exact in float64, so the GPU's fma chain gives
NumPy's acc + a*b bits); n_i = dot_ii; inv_i = 1 / sqrt(n_i), 0 when n_i = 0; s_ij = (dot_ij inv_i) inv_j, +0 when
either norm is 0.  The neighbours of gene i are the K genes j != i with the largest s_ij, ordered by s_ij descending and
equal values by j ascending.  s_ij may differ from s_ji in the last bit; each row uses its own.

Device side (csrc/g2v_nbr.cu): g2v_nbr_norms (inv), g2v_nbr_partial (FP64 FMA tiles with the top-K fused into the
epilogue, the column range split over CTAs when m is small) and, with more than one split, g2v_nbr_merge.
"""
import numpy as np

MAX_K = 64                   # G2V_NBR_MAX_K
MAX_GENES = 1 << 30          # G2V_NBR_MAX_GENES


def check_inputs(W, k):
    """ValueError unless the search can run: W 2-D [m, D] with 2 <= m <= 2^30 and D >= 1, every value finite in
    float32, and k an integer in [1, min(64, m - 1)].  Returns W as a C-contiguous float32 array.  Needs no GPU."""
    W = np.asarray(W)
    if W.ndim != 2:
        raise ValueError("nearest genes: W must be a 2-D array [genes, dimensions], got shape %s" % (W.shape,))
    m, D = W.shape
    if not 2 <= m <= MAX_GENES:
        raise ValueError("nearest genes: m = %d genes, must be in [2, %d]" % (m, MAX_GENES))
    if D < 1:
        raise ValueError("nearest genes: W has no dimensions")
    with np.errstate(over="ignore", invalid="ignore"):
        W = np.ascontiguousarray(W, dtype=np.float32)
    if not np.isfinite(W).all():
        raise ValueError("nearest genes: every value of W must be finite in float32")
    K = int(k) if isinstance(k, (int, np.integer)) else None
    if K is None or not 1 <= K <= min(MAX_K, m - 1):
        raise ValueError("nearest genes: k must be an integer in [1, min(%d, m - 1 = %d)], got %r"
                         % (MAX_K, m - 1, k))
    return W


def nearest_genes(W, k):
    """The k nearest genes of every row of W by cosine, on the GPU.

    W: host float32 array [m, D]; k: 1 <= k <= min(64, m - 1).  Returns (idx int32 [m, k], sim float64 [m, k]): row i
    lists the genes j != i with the largest cosine, descending, ties by j ascending (see the module docstring for the
    exact float64 contract).  ValueError (before anything is uploaded) on inputs check_inputs refuses; RuntimeError
    without a CUDA device."""
    W = check_inputs(W, k)
    K = int(k)
    import torch
    from . import _capi
    lib = _capi.load()
    if not torch.cuda.is_available():
        raise RuntimeError("g2vec_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    dev = torch.device("cuda", torch.cuda.current_device())
    m, D = W.shape
    splits = int(lib.g2v_nbr_splits(m))
    if splits < 1:
        _capi.check(1, "g2v_nbr_splits")
    Wd = torch.from_numpy(W).to(dev)
    inv = torch.empty(m, dtype=torch.float64, device=dev)
    idx = torch.empty((m, K), dtype=torch.int32, device=dev)
    sim = torch.empty((m, K), dtype=torch.float64, device=dev)
    if splits > 1:
        pidx = torch.empty((splits, m, K), dtype=torch.int32, device=dev)
        psim = torch.empty((splits, m, K), dtype=torch.float64, device=dev)
    else:
        pidx, psim = idx, sim
    st = torch.cuda.current_stream(dev).cuda_stream
    _capi.check(lib.g2v_nbr_norms(Wd.data_ptr(), m, D, inv.data_ptr(), st), "g2v_nbr_norms")
    _capi.check(lib.g2v_nbr_partial(Wd.data_ptr(), inv.data_ptr(), m, D, K, pidx.data_ptr(), psim.data_ptr(), st),
                "g2v_nbr_partial")
    if splits > 1:
        _capi.check(lib.g2v_nbr_merge(pidx.data_ptr(), psim.data_ptr(), splits, m, K, idx.data_ptr(), sim.data_ptr(),
                                      st), "g2v_nbr_merge")
    return idx.cpu().numpy(), sim.cpu().numpy()


# ------------------------------------------------------------------------------------------ command-line helpers
def genes_in_paths(code):
    """The search universe of ``--neighbors``: indices (ascending) of the genes that occur in at least one window,
    code >= 0 in paths.build_windows' per-gene code."""
    code = code.cpu().numpy() if hasattr(code, "cpu") else np.asarray(code)
    return np.flatnonzero(code.astype(np.int64) >= 0)


def same_lgroup_share(lgroup, nbr):
    """Fraction of the (gene, neighbour) pairs whose two genes are in the same L-group.  lgroup: per searched gene;
    nbr [m, K]: neighbour positions among the searched genes."""
    lgroup = np.asarray(lgroup)
    return float((lgroup[nbr] == lgroup[:, None]).mean())
