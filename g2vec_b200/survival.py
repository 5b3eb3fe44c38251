"""Permutation Cox score test of every gene against patient survival (DESIGN.md §4.31): per gene the Cox
partial-likelihood score test at beta = 0 with Breslow ties (survival::coxph(ties="breslow")'s score test; for a 0/1
covariate without tied event times, the log-rank test), a raw permutation p-value, the Westfall & Young step-down maxT
adjusted p-value and the Benjamini & Hochberg q-value.

Host side (NumPy): the survival file, the samples with a record, each gene quantised to integers q with |q| <= 2^16
(perm.quantise(x, bits=16)), the time order, the flags and the per-group factors a = 1 / S0 and c = d / S0^2 (S0 and d
do not change under permutation: only the expression moves).
Device side (csrc/g2v_surv.cu, csrc/g2v_dcx.cu): one g2v_surv_scores launch on the time order itself for the observed
T, U and V; then per chunk of permutations g2v_surv_rows (Fisher-Yates with the draws of --permutations' rows for the
same seed), g2v_surv_scores and g2v_dcx_tally over the genes in rank order.

For a time group k (the distinct times, descending) with d_k events and risk set {time >= t_k}: S0, S1, S2 are the
count, sum q and sum q^2 over the risk set and E1 the sum of q over the group's events; num_u = S0 E1 - d S1 and
num_v = S0 S2 - S1^2 are exact int64, U = sum of num_u / S0 and V = sum of d num_v / S0^2 in descending time, and
T = U^2 / V (0 when V = 0).  The counts are integers, so P, P_maxT and Q depend only on the expression, the records,
the seed and B.
"""
import math
from collections import namedtuple

import numpy as np

from . import perm

MAX_SAMPLES = 32768          # G2V_SURV_MAX_SAMPLES
MAX_GENES = 1 << 20          # G2V_SURV_MAX_GENES
MAX_PERMUTATIONS = 1 << 20   # G2V_SURV_MAX_PERMUTATIONS
MIN_SAMPLES = 3
Q_BITS = 16                  # |q| <= 2^16

SurvivalResult = namedtuple("SurvivalResult", "Z T P_score P P_maxT Q count count_maxt order n_perm n n_events")
SurvivalResult.__doc__ = """survival_test's result, every array over the genes in their input order except `order`:
Z       U / sqrt(V), signed: > 0 when higher expression goes with higher hazard; 0 when V = 0;
T       the observed statistic U^2 / V (the squared Z), 0 when V = 0;
P_score erfc(|Z| / sqrt(2)), the score test's asymptotic two-sided p-value;
P       (1 + count) / (B + 1);
P_maxT  step-down maxT adjusted p-values, (1 + count_maxt) / (B + 1) made non-decreasing along the ranks;
Q       Benjamini-Hochberg q-values of P;
count   #{b : T_b >= T_obs};  count_maxt: #{b : max of T_b over the ranks >= this one's >= T_obs} (before the running
        max);
order   the genes by T descending, ties by gene index (rank j -> gene order[j]);
n_perm  B;  n, n_events: the samples and the events of the test."""


def _value(text):
    """A field of the survival file -> float, or None for NA / empty; ValueError on anything else."""
    t = text.strip()
    if t == "" or t.upper() == "NA":
        return None
    return float(t)


def read_survival(path):
    """Tab-delimited SAMPLE, TIME, EVENT (header skipped, further columns ignored) -> {sample: (time, event)}, with
    (None, None) for a row whose TIME or EVENT is NA or empty.  ValueError on a duplicated sample, a short row, or a
    TIME that is not a finite number >= 0 or an EVENT that is not 0 or 1."""
    out = {}
    with open(path) as f:
        lines = f.read().splitlines()
    for ln, line in enumerate(lines[1:], start=2):
        if line.strip() == "":
            continue
        cols = line.split("\t")
        if len(cols) < 3:
            raise ValueError("%s line %d: expected SAMPLE, TIME and EVENT, got %d column(s)" % (path, ln, len(cols)))
        s = cols[0].strip()
        if s in out:
            raise ValueError("%s line %d: sample %s appears twice" % (path, ln, s))
        try:
            t, e = _value(cols[1]), _value(cols[2])
        except ValueError:
            raise ValueError("%s line %d: TIME and EVENT must be numbers or NA, got %r and %r"
                             % (path, ln, cols[1], cols[2])) from None
        if t is None or e is None:
            out[s] = (None, None)
            continue
        if not (math.isfinite(t) and t >= 0.0):
            raise ValueError("%s line %d: TIME must be a finite number >= 0, got %r" % (path, ln, cols[1]))
        if e not in (0.0, 1.0):
            raise ValueError("%s line %d: EVENT must be 0 or 1, got %r" % (path, ln, cols[2]))
        out[s] = (t, int(e))
    return out


def match_survival(records, samples):
    """The records of the expression samples -> (time float64 [N], event int64 [N], used bool [N]); time and event are
    NaN and 0 where the record is NA.  ValueError if a sample has no row."""
    missing = [s for s in samples if s not in records]
    if missing:
        raise ValueError("%d expression sample(s) have no row, the first is %s" % (len(missing), missing[0]))
    N = len(samples)
    time = np.full(N, np.nan)
    event = np.zeros(N, dtype=np.int64)
    used = np.zeros(N, dtype=bool)
    for i, s in enumerate(samples):
        t, e = records[s]
        if t is not None:
            time[i], event[i], used[i] = t, e, True
    return time, event, used


def check_inputs(expr, time, event, n_perm):
    """ValueError unless the test can run: expression [n, G] with one time and event per sample, 3 <= n <= 32768,
    1 <= G <= 2^20, every time finite and >= 0, every event 0 or 1 and at least one of them 1, every expression value
    finite, and 1 <= n_perm <= 2^20.  Returns (x float64 [n, G], time float64 [n], event int64 [n]).  Needs no GPU."""
    x = np.asarray(expr)
    t = np.asarray(time, dtype=np.float64).reshape(-1)
    e = np.asarray(event).reshape(-1)
    if x.ndim != 2 or x.shape[0] != t.shape[0] or e.shape != t.shape:
        raise ValueError("expression must be [samples, genes] with one time and one event per sample, got %s, %d "
                         "times and %d events" % (x.shape, t.shape[0], e.shape[0]))
    n, G = x.shape
    B = int(n_perm)
    if B != n_perm or not 1 <= B <= MAX_PERMUTATIONS:
        raise ValueError("the number of permutations must be an integer in [1, %d], got %r" % (MAX_PERMUTATIONS, n_perm))
    if n < MIN_SAMPLES:
        raise ValueError("%d samples used, at least %d are needed" % (n, MIN_SAMPLES))
    if n > MAX_SAMPLES:
        raise ValueError("%d samples used, at most %d are allowed" % (n, MAX_SAMPLES))
    if not 1 <= G <= MAX_GENES:
        raise ValueError("%d genes, must be in [1, %d]" % (G, MAX_GENES))
    if not (np.isfinite(t).all() and (t >= 0).all()):
        raise ValueError("every time must be a finite number >= 0")
    if not np.isin(e, (0, 1)).all():
        raise ValueError("every event must be 0 or 1")
    if not (e == 1).any():
        raise ValueError("no events among the %d samples used" % n)
    x = x.astype(np.float64)
    if not np.isfinite(x).all():
        raise ValueError("expression values must be finite")
    return x, t, e.astype(np.int64)


def time_groups(time, event):
    """The scan's layout: order (time position -> sample: time descending, ties by sample index), slot (its inverse,
    int32), flags uint8 [n] (bit 0 event, bit 1 last position of its time group) and a, c float64 [n] at the group
    ends (a = 1 / S0, c = d / (S0 S0), S0 = position + 1, d = the group's events; 0 elsewhere)."""
    time = np.asarray(time, dtype=np.float64)
    ev = np.asarray(event).astype(np.int64)
    n = time.shape[0]
    order = np.argsort(-time, kind="stable")
    slot = np.empty(n, dtype=np.int32)
    slot[order] = np.arange(n, dtype=np.int32)
    ts, es = time[order], ev[order]
    end = np.ones(n, dtype=bool)
    end[:-1] = ts[1:] != ts[:-1]
    flags = (es | (end.astype(np.int64) << 1)).astype(np.uint8)
    grp = np.cumsum(np.r_[0, end[:-1]])                # group number of every position
    d = np.bincount(grp, weights=es).astype(np.int64)
    a = np.zeros(n)
    c = np.zeros(n)
    S0 = np.nonzero(end)[0].astype(np.float64) + 1.0
    a[end] = 1.0 / S0
    c[end] = d.astype(np.float64) / (S0 * S0)           # S0 S0 <= 2^30: exact
    return order, slot, flags, a, c


def prepare(expr, time, event, n_perm=1):
    """Host side up to the upload: a dict with n, n_events, q (int64 [n, G], |q| <= 2^16) and the layout of
    time_groups (order, slot, flags, a, c)."""
    x, t, e = check_inputs(expr, time, event, n_perm)
    order, slot, flags, a, c = time_groups(t, e)
    return {"n": x.shape[0], "n_events": int(e.sum()), "q": perm.quantise(x, bits=Q_BITS), "order": order,
            "slot": slot, "flags": flags, "a": a, "c": c}


def cox_score(x, time, event):
    """The Breslow score test at beta = 0 in plain float64, for covariates x [n] or [n, G]: returns (Z, U, V) with
    U = sum_k (E1_k - d_k S1_k / S0_k), V = sum_k d_k (S2_k / S0_k - (S1_k / S0_k)^2) and Z = U / sqrt(V) (0 when
    V = 0)."""
    x = np.asarray(x, dtype=np.float64)
    one = x.ndim == 1
    x = x.reshape(x.shape[0], -1)
    order, _, flags, _, _ = time_groups(time, event)
    xs = x[order]
    ev = (flags & 1).astype(bool)
    end = (flags & 2).astype(bool)
    S1, S2 = np.cumsum(xs, axis=0)[end], np.cumsum(xs * xs, axis=0)[end]
    S0 = (np.nonzero(end)[0] + 1.0)[:, None]
    grp = np.cumsum(np.r_[0, end[:-1]])
    E1 = np.zeros_like(S1)
    np.add.at(E1, grp[ev], xs[ev])
    d = np.bincount(grp, weights=ev.astype(np.float64))[:, None]
    m = S1 / S0
    U = (E1 - d * m).sum(axis=0)
    V = (d * (S2 / S0 - m * m)).sum(axis=0)
    V = np.maximum(V, 0.0)
    Z = np.zeros_like(U)
    np.divide(U, np.sqrt(V), out=Z, where=V > 0)
    if one:
        return float(Z[0]), float(U[0]), float(V[0])
    return Z, U, V


def z_of(U, V):
    """Z = U / sqrt(V), 0 where V = 0."""
    U = np.asarray(U, np.float64); V = np.asarray(V, np.float64)
    Z = np.zeros(np.broadcast(U, V).shape)
    np.divide(U, np.sqrt(V), out=Z, where=V > 0)
    return Z


def p_score(Z):
    """erfc(|Z| / sqrt(2)) per element."""
    return np.array([math.erfc(abs(z) / math.sqrt(2.0)) for z in np.asarray(Z, np.float64).reshape(-1)])


def finish(prep, T_obs, U, V, order, count_rank, count_maxt_rank, n_perm):
    """Counts in rank order -> SurvivalResult."""
    B, G = int(n_perm), order.shape[0]
    count = np.empty(G, dtype=np.int64); count[order] = count_rank
    count_maxt = np.empty(G, dtype=np.int64); count_maxt[order] = count_maxt_rank
    P = (1.0 + count) / (B + 1.0)
    pm = np.empty(G); pm[order] = np.maximum.accumulate((1.0 + np.asarray(count_maxt_rank)) / (B + 1.0))
    Z = z_of(U, V)
    return SurvivalResult(Z=Z, T=np.asarray(T_obs, np.float64), P_score=p_score(Z), P=P, P_maxT=pm, Q=perm.bh(P),
                          count=count, count_maxt=count_maxt, order=order, n_perm=B, n=prep["n"],
                          n_events=prep["n_events"])


def chunk_rows(n, G, n_perm, max_chunk_bytes):
    """Permutations per chunk: idx (2 n bytes) and T (8 G bytes) of every row within max_chunk_bytes, at least 1."""
    return int(max(1, min(int(n_perm), int(max_chunk_bytes) // (2 * n + 8 * G))))


def _device():
    """The torch device and stream of a run, and the upload helper; RuntimeError without a GPU."""
    import torch
    from . import _capi
    lib = _capi.load()
    if not torch.cuda.is_available():
        raise RuntimeError("g2vec_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    dev = torch.device("cuda", torch.cuda.current_device())
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return lib, dev, torch.cuda.current_stream(dev).cuda_stream, up


def _observed(prep, lib, dev, st, up):
    """One g2v_surv_scores launch on the time order itself: (T_obs, U, V float64 [G], order, (flags_d, a_d, c_d)),
    with order the genes by T descending, ties by gene index."""
    import torch
    from . import _capi
    n, q = prep["n"], prep["q"]
    G = q.shape[1]
    q_d = up(q.astype(np.int32))
    flags_d, a_d, c_d = up(prep["flags"]), up(prep["a"]), up(prep["c"])
    ident_d = up(prep["order"].astype(np.uint16))
    T1 = torch.empty((1, G), dtype=torch.float64, device=dev)
    UV = torch.empty((2, 1, G), dtype=torch.float64, device=dev)
    _capi.check(lib.g2v_surv_scores(q_d.data_ptr(), n, G, ident_d.data_ptr(), 1, flags_d.data_ptr(), a_d.data_ptr(),
                                    c_d.data_ptr(), T1.data_ptr(), UV.data_ptr(), st), "g2v_surv_scores")
    T_obs, UVh = T1[0].cpu().numpy(), UV.cpu().numpy()
    return T_obs, UVh[0, 0], UVh[1, 0], np.argsort(-T_obs, kind="stable"), (flags_d, a_d, c_d)


def rank_genes(expr, time, event):
    """The genes by their observed Cox score statistic T, descending, ties by gene index: survival_test's `order`,
    from the same device scan (one launch).  ValueError on inputs check_inputs refuses, RuntimeError without a GPU."""
    prep = prepare(expr, time, event)
    return _observed(prep, *_device())[3]


def survival_test(expr, time, event, n_perm, seed=0, max_chunk_bytes=None):
    """Permutation Cox score test of every gene against survival on the GPU.

    expr: host float array [samples, genes]; time: one finite time >= 0 per sample (any unit); event: 1 for an event
    (death or relapse), 0 for censored.  n_perm: B, 1 <= B <= 2^20 permutations of the expression against the
    records (the observed pairing is not among them), with the Fisher-Yates draws of perm.perm_test's rows for the
    same seed and sample count; seed: the Philox key (--seed).  max_chunk_bytes: bound on the device memory of one
    chunk's rows and statistics (default: half the free device memory).  Makes 1 launch, then 3 per chunk.  Returns a
    SurvivalResult; ValueError (before anything is uploaded) on inputs check_inputs refuses."""
    prep = prepare(expr, time, event, n_perm)
    import torch
    from . import _capi
    lib, dev, st, up = _device()
    n, B, q = prep["n"], int(n_perm), prep["q"]
    G = q.shape[1]
    T_obs, U, V, order, (flags_d, a_d, c_d) = _observed(prep, lib, dev, st, up)
    slot_d = up(prep["slot"])
    # the permutations run over the genes in rank order, so the tally reads every row of T front to back
    qr_d = up(q[:, order].astype(np.int32))
    Tobs_d = up(T_obs[order])
    cnt = torch.zeros(G, dtype=torch.int64, device=dev)
    cmax = torch.zeros(G, dtype=torch.int64, device=dev)
    if max_chunk_bytes is None:
        max_chunk_bytes = torch.cuda.mem_get_info(dev)[0] // 2
    rows = chunk_rows(n, G, B, max_chunk_bytes)
    idx = torch.empty((rows, n), dtype=torch.uint16, device=dev)
    T = torch.empty((rows, G), dtype=torch.float64, device=dev)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    for b0 in range(0, B, rows):
        nb = min(rows, B - b0)
        _capi.check(lib.g2v_surv_rows(slot_d.data_ptr(), n, seed, b0, nb, idx.data_ptr(), st), "g2v_surv_rows")
        _capi.check(lib.g2v_surv_scores(qr_d.data_ptr(), n, G, idx.data_ptr(), nb, flags_d.data_ptr(),
                                        a_d.data_ptr(), c_d.data_ptr(), T.data_ptr(), None, st), "g2v_surv_scores")
        _capi.check(lib.g2v_dcx_tally(T.data_ptr(), nb, G, Tobs_d.data_ptr(), cnt.data_ptr(), cmax.data_ptr(), st),
                    "g2v_dcx_tally")
    return finish(prep, T_obs, U, V, order, cnt.cpu().numpy(), cmax.cpu().numpy(), B)


def label_score(label, time, event):
    """Cox score test of the good / poor label (1 = poor) over the samples with label 0 or 1: (Z, P_score) from
    cox_score; (0, 1) when fewer than 2 such samples or no event among them."""
    lab = np.asarray(label).reshape(-1)
    keep = (lab == 0) | (lab == 1)
    ev = np.asarray(event)[keep]
    if keep.sum() < 2 or not (ev == 1).any():
        return 0.0, 1.0
    z = cox_score(lab[keep].astype(np.float64), np.asarray(time)[keep], ev)[0]
    return z, math.erfc(abs(z) / math.sqrt(2.0))


def summary(res, is_biomarker, label_z, label_p):
    """The command line's line: is_biomarker (0/1 per gene), and the label's Z and P_score from label_score."""
    sig = res.P_maxT <= 0.05
    return ("survival: %d permutations of %d samples (%d events): %d genes with P_maxT <= 0.05 (%d of the biomarkers), "
            "%d with Q <= 0.05; Cox score test of the good / poor label: Z = %.4f, P_score = %.4g"
            % (res.n_perm, res.n, res.n_events, int(sig.sum()), int((sig & (np.asarray(is_biomarker) > 0)).sum()),
               int((res.Q <= 0.05).sum()), label_z, label_p))
