"""Seeded synthetic cohorts for the nested cross-validation tests: genes in correlated modules joined by a module
network, with labels independent of expression (null) or one module whose expression shifts with the label
(planted)."""
import numpy as np

N_SAMPLES, N_GENES, MODULE = 120, 400, 10
PLANTED = np.arange(10)            # the planted genes: the first module


def module_cohort(seed, planted=False, n=N_SAMPLES, G=N_GENES, module=MODULE, shift=2.5):
    """(expr float32 [n, G], label int [n] with n / 2 of each, genes, edges as (src, dst) int32).

    Every module of `module` consecutive genes shares one factor per sample: x = 0.85 f + 0.5 e, so two genes of a
    module correlate at about 0.74 (above the default --min-corr 0.5).  The network joins each gene to 4 random genes
    of its module and adds G / 10 random edges across modules.  With planted=False every module is co-expressed in
    both groups, so the labels are independent of the expression.  planted=True makes the cohort G2Vec's model: module
    m with m % 4 == 1 is co-expressed in the good samples only and m % 4 == 2 in the poor samples only (x = e in the
    other group), so the good-only, poor-only and shared genes fall into three L-groups; and the genes of PLANTED (the
    first module) become a poor-only module whose level also shifts: x = e on the good samples, shift + 0.85 f + 0.5 e
    on the poor ones."""
    rs = np.random.RandomState(seed)
    label = np.array([0] * (n // 2) + [1] * (n - n // 2))
    rs.shuffle(label)
    x = np.empty((n, G))
    src, dst = [], []
    for m0 in range(0, G, module):
        m = np.arange(m0, min(m0 + module, G))
        f = rs.standard_normal((n, 1))
        x[:, m] = 0.85 * f + 0.5 * rs.standard_normal((n, m.size))
        only = (m0 // module) % 4                     # with planted: 1 good-only, 2 poor-only
        if planted and only in (1, 2):
            off = (label != only - 1)[:, None]
            x[:, m] = np.where(off, rs.standard_normal((n, m.size)), x[:, m])
        for g in m:
            for h in rs.choice(m[m != g], size=min(4, m.size - 1), replace=False):
                src.append(g); dst.append(h)
    for _ in range(G // 10):
        a, b = rs.randint(0, G, 2)
        if a != b:
            src.append(a); dst.append(b)
    if planted:
        f = rs.standard_normal((n, 1))
        e = rs.standard_normal((n, PLANTED.size))
        poor = (label == 1)[:, None]
        x[:, PLANTED] = np.where(poor, shift + 0.85 * f + 0.5 * e, e)
        keep = [(a, b) for a, b in zip(src, dst) if (a in PLANTED) == (b in PLANTED)]
        src, dst = [a for a, _ in keep], [b for _, b in keep]
        for g in PLANTED:
            for h in rs.choice(PLANTED[PLANTED != g], size=4, replace=False):
                src.append(g); dst.append(h)
    genes = np.array(["G%03d" % i for i in range(G)])
    return x.astype(np.float32), label, genes, (np.array(src, np.int32), np.array(dst, np.int32))
