"""Float64 NumPy restatement of the lasso / elastic-net logistic path (DESIGN.md §4.37): glmnet-style proximal Newton
with cyclic coordinate descent over every gene (no screening), the same lambda sequence and stop rules.  It shares no
code with g2vec_b200/lasso.py or the kernels; the tests compare solutions, not bits."""
import numpy as np

N_LAMBDA, MAX_ACTIVE = 100, 512


def standardise(x):
    """(z, mu, sd) with the population SD; a constant gene gets z = 0 (mu = its value, sd = 1)."""
    mn, mx = x.min(axis=0), x.max(axis=0)
    const = mn == mx
    mu = np.where(const, mn, x.mean(axis=0))
    sd = np.where(const, 1.0, np.sqrt(((x - mu) ** 2).mean(axis=0)))
    z = np.where(const, 0.0, (x - mu) / sd)
    return z, mu, sd, const


def lambdas(z, y, alpha):
    n, G = z.shape
    lam_max = np.abs(z.T @ (y - y.mean())).max() / (n * max(alpha, 1e-3))
    ratio = 0.01 if n < G else 1e-4
    return lam_max * ratio ** (np.arange(N_LAMBDA) / (N_LAMBDA - 1.0))


def objective(z, y, b0, beta, lam, alpha):
    eta = b0 + z @ beta
    nll = np.mean(np.logaddexp(0.0, eta) - y * eta)
    return nll + lam * (alpha * np.abs(beta).sum() + 0.5 * (1 - alpha) * (beta ** 2).sum())


def gradient(z, y, b0, beta, lam, alpha):
    """(g0, g) of the smooth part."""
    n = len(y)
    r = y - 1.0 / (1.0 + np.exp(-(b0 + z @ beta)))
    return -r.sum() / n, -(z.T @ r) / n + lam * (1 - alpha) * beta


def kkt(z, y, b0, beta, lam, alpha, const=None):
    g0, g = gradient(z, y, b0, beta, lam, alpha)
    l1 = lam * alpha
    v = np.where(beta == 0, np.maximum(np.abs(g) - l1, 0.0), np.abs(g + l1 * np.sign(beta)))
    if const is not None:
        v[const] = 0.0
    return max(abs(g0), v.max() if v.size else 0.0)


def sweep(z, w, r, beta, genes, l1, l2, n):
    dlx = 0.0
    for j in genes:
        zj = z[:, j]
        wz = w * zj
        v = wz @ zj / n
        if v == 0.0:
            continue
        u = wz @ r / n + v * beta[j]
        bn = np.sign(u) * max(abs(u) - l1, 0.0) / (v + l2)
        d = bn - beta[j]
        if d != 0.0:
            r -= d * zj
            beta[j] = bn
            dlx = max(dlx, v * d * d)
    return dlx


def solve(z, y, b0, beta, lam, alpha, tol=1e-22, max_newton=200):
    n, G = z.shape
    beta = beta.copy()
    l1, l2 = lam * alpha, lam * (1 - alpha)
    for _ in range(max_newton):
        eta = b0 + z @ beta
        p = 1.0 / (1.0 + np.exp(-eta))
        w = np.maximum(p * (1 - p), 1e-5 * (1 - 1e-5))
        r = (y - p) / w
        sw = w.sum()
        first = None
        genes = np.arange(G)
        while True:
            dlx = sweep(z, w, r, beta, genes, l1, l2, n)
            d0 = (w * r).sum() / sw
            r -= d0
            b0 += d0
            dlx = max(dlx, sw / n * d0 * d0)
            if first is None:
                first = dlx
            if dlx < tol:
                break
            act = np.nonzero(beta)[0]                  # cycle over the nonzero genes until they settle
            while True:
                dlx = sweep(z, w, r, beta, act, l1, l2, n)
                d0 = (w * r).sum() / sw
                r -= d0
                b0 += d0
                if max(dlx, sw / n * d0 * d0) < tol:
                    break
        if first < tol:
            break
    return b0, beta


def path(x, y, alpha, lams=None):
    """The path of one fit on samples x [n, G], y [n]: dict with lambdas, b0 [L], beta [L, G], dev_ratio [L], entry [G],
    entry_abs [G], L (the path length by the stop rules), z, mu, sd."""
    y = np.asarray(y, dtype=np.float64)
    z, mu, sd, const = standardise(np.asarray(x, dtype=np.float64))
    n, G = z.shape
    if lams is None:
        lams = lambdas(z, y, alpha)
    ybar = y.mean()
    b0 = np.log(ybar / (1 - ybar))
    beta = np.zeros(G)
    dev_null = 2 * np.sum(np.logaddexp(0.0, b0) - y * b0)
    entry = np.full(G, -1, dtype=np.int64)
    entry_abs = np.zeros(G)
    B0, B, DR = [], [], []
    prev, L = 0.0, len(lams)
    for k, lam in enumerate(lams):
        nb0, nbeta = solve(z, y, b0, beta, lam, alpha)
        new = (nbeta != 0) & (entry < 0)
        if (entry >= 0).sum() + new.sum() > MAX_ACTIVE:
            L = k
            break
        b0, beta = nb0, nbeta
        entry[new] = k
        entry_abs[new] = np.abs(beta[new])
        eta = b0 + z @ beta
        dr = 1 - 2 * np.sum(np.logaddexp(0.0, eta) - y * eta) / dev_null
        B0.append(b0); B.append(beta.copy()); DR.append(dr)
        if dr > 0.999 or (k >= 4 and dr - prev < 1e-5 * dr):
            L = k + 1
            break
        prev = dr
    return dict(lambdas=np.asarray(lams), b0=np.asarray(B0), beta=np.asarray(B), dev_ratio=np.asarray(DR),
                entry=entry, entry_abs=entry_abs, L=L, z=z, mu=mu, sd=sd, const=const)


def predict(fit, x_test, k):
    """The linear predictor of x_test at lambda index k (the last solution when the path stopped before k)."""
    k = min(k, len(fit["b0"]) - 1)
    zt = np.where(fit["const"], 0.0, (x_test - fit["mu"]) / fit["sd"])
    return fit["b0"][k] + zt @ fit["beta"][k]


P_MIN = 1e-5                                           # glmnet's clamp of a held-out probability


def heldout_deviance(eta, y):
    """Each sample's binomial deviance -2 log p (y = 1) or -2 log(1 - p) (y = 0), p = sigmoid(eta) clamped to
    [1e-5, 1 - 1e-5]."""
    eta, y = np.asarray(eta, dtype=np.float64), np.asarray(y)
    p = np.clip(1.0 / (1.0 + np.exp(-eta)), P_MIN, 1.0 - P_MIN)
    return np.where(y == 1, -2.0 * np.log(p), -2.0 * np.log(1.0 - p))


def cv_glmnet(dev, folds, F):
    """cv.glmnet's grouped rule over the K F folds as one set (DESIGN.md §4.37), from the held-out deviances dev
    [L, K, n] and the folds [K, n]: (cvm, cvsd, i_min, i_1se).  cvm is the fold-size-weighted mean of the fold means,
    which is the plain mean over every held-out (repeat, sample); cvsd = sqrt(sum_f N_f (m_f - cvm)^2 / N / (K F - 1));
    i_min the first argmin of cvm; i_1se the first (largest-lambda) index with cvm <= cvm[i_min] + cvsd[i_min]."""
    dev = np.asarray(dev, dtype=np.float64)
    L, K, n = dev.shape
    group = (np.arange(K)[:, None] * F + np.asarray(folds, dtype=np.int64)).ravel()     # fold id of (k, i)
    N = np.bincount(group, minlength=K * F).astype(np.float64)
    cvm = np.empty(L)
    cvsd = np.empty(L)
    for li in range(L):
        d = dev[li].ravel()
        cvm[li] = d.mean()
        m = np.bincount(group, weights=d, minlength=K * F) / N
        cvsd[li] = np.sqrt((N * (m - cvm[li]) ** 2).sum() / N.sum() / (K * F - 1))
    best = cvm.min()
    i_min = next(li for li in range(L) if cvm[li] == best)
    i_1se = next(li for li in range(L) if cvm[li] <= cvm[i_min] + cvsd[i_min])
    return cvm, cvsd, i_min, i_1se
