"""Exact 2-D t-SNE map of the gene vectors on the GPU, with float64 affinities and gradient (DESIGN.md §4.27).

Contract: scikit-learn's exact t-SNE (``TSNE(method="exact")``) with the differences DESIGN.md §4.27 lists.  x_i =
float64(W_i); d_ij is the chain acc = acc + t*t, t = x_id - x_jd, over d ascending from +0, each operation rounded
separately.  Per row, scikit-learn's perplexity bisection on d in float64 gives beta_i, the 0-based evaluation s_i
that met the tolerance (100 if none did) and c_ij = exp(-d_ij beta_i) / S_i; P_ij = (c_ij + c_ji) / (2m).  exp and log
are CUDA's, so beta and s, not the bits of P, are the contract of that part.  Given P and Y0 the iteration is +, -, *, /
only and bit-identical to tests/tsne_oracle.py: per row i and column block of BLOCK columns the chains over j != i
(ascending) of w = 1 / (1 + ((y_i0 - y_j0)^2 + (y_i1 - y_j1)^2)), p_ij w t_c and w^2 t_c; the block partials chained in
ascending order; Z = the chain of the Z_i in blocks of BLOCK rows, then over the blocks; g = 4 ((alpha A) - (R / Z));
scikit-learn's gains, momentum and step with eta = max(m / 12 / 4, 50); alpha = 12 and momentum 0.5 for iterations
0 .. 249, then 1 and 0.8, u and the gains starting over at 250.  Every run takes exactly n_iter iterations.

Device side (csrc/g2v_tsne.cu): g2v_tsne_dist, g2v_tsne_affinity and g2v_tsne_symmetrize build P in one m x m float64
buffer; per iteration g2v_tsne_grad and g2v_tsne_update, with no synchronisation; g2v_tsne_kl at the end.
"""
from collections import namedtuple
from numbers import Real

import numpy as np

MAX_GENES = 32768            # G2V_TSNE_MAX_GENES: P alone is 8 GiB there
BLOCK = 256                  # G2V_TSNE_BLOCK: columns per block of the gradient chains, rows per block of Z
EXPLORATION = 250            # iterations with early exaggeration (scikit-learn's _EXPLORATION_MAX_ITER)
EXAGGERATION = 12.0
MAX_STEPS = 100              # perplexity bisection evaluations per row
TOLERANCE = float(np.float32(1e-5))
N_ITER = 1000

TsneResult = namedtuple("TsneResult", "Y beta steps kl learning_rate")
TsneResult.__doc__ = """tsne_map's result for m genes:
Y              float64 [m, 2]: the map after n_iter iterations;
beta           float64 [m]: each row's precision from the perplexity bisection;
steps          int32 [m]: the 0-based bisection evaluation that met the tolerance, 100 if none did;
kl             the KL divergence of P and Q at Y;
learning_rate  eta = max(m / 12 / 4, 50), scikit-learn's learning_rate="auto"."""


def check_inputs(W, perplexity, n_iter=N_ITER, init="pca"):
    """ValueError unless the map can run: W 2-D [m, D] with 2 <= m <= 32768 and D >= 1, every value finite in float32;
    perplexity a finite number with 1 <= perplexity < m; n_iter an integer >= 1; init "pca" or a finite array [m, 2].
    Returns (W as a C-contiguous float32 array, init as "pca" or a C-contiguous float64 array).  Needs no GPU."""
    W = np.asarray(W)
    if W.ndim != 2:
        raise ValueError("t-SNE: W must be a 2-D array [genes, dimensions], got shape %s" % (W.shape,))
    m, D = W.shape
    if not 2 <= m <= MAX_GENES:
        raise ValueError("t-SNE: m = %d genes, must be in [2, %d]" % (m, MAX_GENES))
    if D < 1:
        raise ValueError("t-SNE: W has no dimensions")
    with np.errstate(over="ignore", invalid="ignore"):
        W = np.ascontiguousarray(W, dtype=np.float32)
    if not np.isfinite(W).all():
        raise ValueError("t-SNE: every value of W must be finite in float32")
    if isinstance(perplexity, (bool, np.bool_)) or not isinstance(perplexity, Real) \
            or not (np.isfinite(perplexity) and 1 <= perplexity < m):
        raise ValueError("t-SNE: perplexity must be a finite number with 1 <= perplexity < m = %d, got %r"
                         % (m, perplexity))
    if isinstance(n_iter, (bool, np.bool_)) or not isinstance(n_iter, (int, np.integer)) or n_iter < 1:
        raise ValueError("t-SNE: n_iter must be an integer >= 1, got %r" % (n_iter,))
    if isinstance(init, str):
        if init != "pca":
            raise ValueError("t-SNE: init must be 'pca' or an array [m, 2], got %r" % (init,))
        return W, init
    return W, _check_y0(init, m)


def _check_y0(Y0, m):
    Y0 = np.asarray(Y0)
    if Y0.shape != (m, 2) or not np.issubdtype(Y0.dtype, np.number):
        raise ValueError("t-SNE: init must be 'pca' or an array [m = %d, 2], got shape %s" % (m, Y0.shape))
    Y0 = np.ascontiguousarray(Y0, dtype=np.float64)
    if not np.isfinite(Y0).all():
        raise ValueError("t-SNE: every value of init must be finite")
    return Y0


def learning_rate(m):
    """scikit-learn's learning_rate="auto": max(m / early_exaggeration / 4, 50), in float64."""
    return float(max(m / EXAGGERATION / 4, 50.0))


def pca_init(W, seed=0):
    """Y0 [m, 2] float64: the centred rows projected on the first two right singular vectors of np.linalg.svd, each
    flipped so that its largest-|.| entry is positive, scaled so that column 0 has standard deviation 1e-4.  With
    D < 2, or when that standard deviation is 0 (all rows equal), np.random.default_rng(seed).standard_normal((m, 2))
    * 1e-4 instead."""
    X = np.asarray(W, dtype=np.float64)
    m = X.shape[0]
    if X.shape[1] >= 2:
        Xc = X - X.mean(axis=0)
        _, _, Vt = np.linalg.svd(Xc, full_matrices=False)
        comps = Vt[:2]
        top = np.argmax(np.abs(comps), axis=1)
        comps = comps * np.sign(comps[np.arange(2), top])[:, None]
        Y = Xc @ comps.T
        sd = np.std(Y[:, 0])
        if sd > 0:
            return np.ascontiguousarray(Y / sd * 1e-4)
    return np.random.default_rng(seed).standard_normal((m, 2)) * 1e-4


def summary(n, perplexity, n_iter, kl):
    """The t-SNE line of the command line (without its indentation)."""
    return ("t-SNE: 2-D map of %d genes in paths, perplexity %g, %d iterations: KL divergence %.6f"
            % (n, perplexity, n_iter, kl))


def _device():
    import torch
    from . import _capi
    lib = _capi.load()
    if not torch.cuda.is_available():
        raise RuntimeError("g2vec_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    dev = torch.device("cuda", torch.cuda.current_device())
    return lib, dev, torch.cuda.current_stream(dev).cuda_stream


def _affinities(lib, dev, st, W, perplexity):
    """P (device, [m, m] float64), beta and steps (device)."""
    import torch
    from . import _capi
    m, D = W.shape
    Wd = torch.from_numpy(W).to(dev)
    P = torch.empty((m, m), dtype=torch.float64, device=dev)
    beta = torch.empty(m, dtype=torch.float64, device=dev)
    steps = torch.empty(m, dtype=torch.int32, device=dev)
    _capi.check(lib.g2v_tsne_dist(Wd.data_ptr(), m, D, P.data_ptr(), st), "g2v_tsne_dist")
    _capi.check(lib.g2v_tsne_affinity(P.data_ptr(), m, float(perplexity), beta.data_ptr(), steps.data_ptr(), st),
                "g2v_tsne_affinity")
    _capi.check(lib.g2v_tsne_symmetrize(P.data_ptr(), m, st), "g2v_tsne_symmetrize")
    return P, beta, steps


def _optimize(lib, dev, st, P, Y0, n_iter):
    """n_iter iterations from Y0 on the device P; (Y, kl) on the host."""
    import torch
    from . import _capi
    m = Y0.shape[0]
    eta = learning_rate(m)
    Y = torch.from_numpy(Y0).to(dev)
    u = torch.empty((m, 2), dtype=torch.float64, device=dev)        # set at iteration 0
    gains = torch.empty((m, 2), dtype=torch.float64, device=dev)
    ws = torch.empty(int(lib.g2v_tsne_workspace_bytes(m)) // 8, dtype=torch.float64, device=dev)
    kl = torch.empty(1, dtype=torch.float64, device=dev)
    p, y, w = P.data_ptr(), Y.data_ptr(), ws.data_ptr()
    for it in range(n_iter):
        _capi.check(lib.g2v_tsne_grad(p, y, m, w, st), "g2v_tsne_grad")
        _capi.check(lib.g2v_tsne_update(w, m, it, eta, y, u.data_ptr(), gains.data_ptr(), st), "g2v_tsne_update")
    _capi.check(lib.g2v_tsne_kl(p, y, m, w, kl.data_ptr(), st), "g2v_tsne_kl")
    return Y.cpu().numpy(), float(kl.item())


def affinities(W, perplexity):
    """(P host float64 [m, m], beta float64 [m], steps int32 [m]) of the rows of W: the distances, the perplexity
    bisection and the symmetrisation on the GPU.  For tests at small m (P is m^2 doubles).  ValueError before anything
    is uploaded on inputs check_inputs refuses; RuntimeError without a CUDA device."""
    W, _ = check_inputs(W, perplexity)
    lib, dev, st = _device()
    P, beta, steps = _affinities(lib, dev, st, W, perplexity)
    return P.cpu().numpy(), beta.cpu().numpy(), steps.cpu().numpy()


def optimize(P, Y0, n_iter=N_ITER):
    """(Y float64 [m, 2], kl) after n_iter iterations from Y0 [m, 2] on the joint affinities P [m, m] (host float64,
    symmetric), on the GPU.  ValueError before anything is uploaded on bad shapes or values; RuntimeError without a CUDA
    device."""
    P = np.asarray(P)
    if P.ndim != 2 or P.shape[0] != P.shape[1] or not 2 <= P.shape[0] <= MAX_GENES:
        raise ValueError("t-SNE: P must be a square array [m, m] with 2 <= m <= %d, got shape %s"
                         % (MAX_GENES, P.shape))
    P = np.ascontiguousarray(P, dtype=np.float64)
    if not np.isfinite(P).all():
        raise ValueError("t-SNE: every value of P must be finite")
    Y0 = _check_y0(Y0, P.shape[0])
    if isinstance(n_iter, (bool, np.bool_)) or not isinstance(n_iter, (int, np.integer)) or n_iter < 1:
        raise ValueError("t-SNE: n_iter must be an integer >= 1, got %r" % (n_iter,))
    import torch
    lib, dev, st = _device()
    return _optimize(lib, dev, st, torch.from_numpy(P).to(dev), Y0, int(n_iter))


def tsne_map(W, perplexity=30.0, n_iter=N_ITER, seed=0, init="pca"):
    """The exact 2-D t-SNE map of the rows of W on the GPU; P stays on the device.

    W: host float32 array [m, D], 2 <= m <= 32768; perplexity: 1 <= perplexity < m; n_iter >= 1 iterations, all of
    them run; seed: the random initialisation when PCA cannot give one (see pca_init); init: "pca" or Y0 [m, 2].
    Returns a TsneResult (see the module docstring for the contract); ValueError (before anything is uploaded) on
    inputs check_inputs refuses; RuntimeError without a CUDA device."""
    W, init = check_inputs(W, perplexity, n_iter, init)
    Y0 = pca_init(W, seed) if isinstance(init, str) else init
    lib, dev, st = _device()
    P, beta, steps = _affinities(lib, dev, st, W, perplexity)
    Y, kl = _optimize(lib, dev, st, P, Y0, int(n_iter))
    return TsneResult(Y=Y, beta=beta.cpu().numpy(), steps=steps.cpu().numpy(), kl=kl,
                      learning_rate=learning_rate(W.shape[0]))
