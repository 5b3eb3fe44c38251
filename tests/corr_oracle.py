"""Float64 restatements of the Spearman and biweight-midcorrelation edge weights (DESIGN.md §4.22), written from the
definitions and independent of g2vec_b200.graph: Spearman through scipy.stats.rankdata (checked against
scipy.stats.spearmanr by the tests), bicor as WGCNA defines it (maxPOutliers = 1, pearsonFallback = "individual").

Error bound per edge: the kernels store z in float32, so each z_i carries a relative error <= u = 2^-24; with
mean z^2 = 1 for both genes, Cauchy-Schwarz bounds the weight's error by 2u plus the double dot product's own error,
far below EDGE_TOL."""
import numpy as np
from scipy import stats

U = 2.0 ** -24
EDGE_TOL = 1e-6


def pearson_z(x):
    """Pearson z-score of one gene's values: population std, 0 when all values are equal."""
    x = np.asarray(x, dtype=np.float64)
    sd = x.std()
    return (x - x.mean()) / sd if sd > 0 else np.zeros_like(x)


def spearman_z(x):
    """z-score of the average ranks (ties share the mean of their positions; -0.0 ties with +0.0)."""
    return pearson_z(stats.rankdata(np.asarray(x, dtype=np.float64), method="average"))


def _median(v):
    v = np.sort(v)
    n = v.shape[0]
    return v[n // 2] if n % 2 else (v[n // 2 - 1] + v[n // 2]) / 2.0


def bicor_z(x):
    """Tukey's biweight transform scaled to sum z^2 = S; the Pearson z-score when the MAD is 0."""
    x = np.asarray(x, dtype=np.float64)
    S = x.shape[0]
    med = _median(x)
    mad = _median(np.abs(x - med))
    if mad == 0:
        return pearson_z(x)
    u = (x - med) / (9.0 * mad)
    a = np.where(np.abs(u) < 1.0, (1.0 - u * u) ** 2, 0.0)
    t = (x - med) * a
    return t * np.sqrt(S) / np.sqrt((t * t).sum())


def mad(x):
    x = np.asarray(x, dtype=np.float64)
    return _median(np.abs(x - _median(x)))


TRANSFORMS = {"pearson": pearson_z, "spearman": spearman_z, "bicor": bicor_z}


def transform(X, method):
    """X [S, V] (one group's samples) -> z [S, V] float64, column by column."""
    X = np.asarray(X)
    f = TRANSFORMS[method]
    Z = np.zeros(X.shape, dtype=np.float64)
    for v in range(X.shape[1]):
        Z[:, v] = f(X[:, v])
    return Z


def edge_weights(Z, src, dst):
    """|mean_s z[s, src] z[s, dst]| in float64 from z [S, V]."""
    S = Z.shape[0]
    return np.abs((Z[:, np.asarray(src)] * Z[:, np.asarray(dst)]).sum(axis=0) / S)


def weights(X, src, dst, method):
    return edge_weights(transform(X, method), src, dst)
