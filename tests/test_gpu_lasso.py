"""The lasso / elastic-net path on the GPU (DESIGN.md §4.37) against the float64 oracle in tests/lasso_oracle.py: the
host recomputes every certified solution's KKT conditions, objectives match the oracle's, coefficients and held-out
scores match at G < n, and the results are bit-identical across calls and chunkings."""
import numpy as np
import pytest

from tests import lasso_oracle as orc

pytestmark = pytest.mark.gpu


def cohort(n, G, seed, planted=4, const=True):
    rs = np.random.RandomState(seed)
    x = rs.randn(n, G) * rs.uniform(0.5, 2.0, G) + rs.uniform(-1, 3, G)
    lab = (rs.rand(n) < 0.5).astype(np.int64)
    lab[:2] = [0, 1]
    x[:, :planted] += 0.8 * lab[:, None]
    if const:
        x[:, G - 1] = 1.25
    return x, lab


def run(x, lab, **kw):
    from g2vec_b200 import lasso
    return lasso.lasso_cv(x, lab, **kw)


def check_fit(res, x, lab, alpha, L):
    z, mu, sd, const = orc.standardise(x)
    y = lab.astype(np.float64)
    ref = orc.path(x, y, alpha, lams=res.lambdas)
    for k in range(L):
        if res.kkt[0, k] <= 1e-7:                     # the host's own standardisation moves g by ~1e-14 only
            assert orc.kkt(z, y, res.a0[k], res.beta[k], res.lambdas[k], alpha, const) <= 1e-7 + 1e-12
        assert not res.beta[k][const].any()
        if k < len(ref["b0"]):
            o_dev = orc.objective(z, y, res.a0[k], res.beta[k], res.lambdas[k], alpha)
            o_ref = orc.objective(z, y, ref["b0"][k], ref["beta"][k], res.lambdas[k], alpha)
            assert o_dev <= o_ref + 1e-9 * abs(o_ref), (k, o_dev, o_ref)
    return ref


@pytest.mark.parametrize("n,G,alpha", [(31, 12, 1.0), (32, 13, 0.5), (33, 20, 1.0), (40, 70, 1.0)])
def test_fit0_and_folds_against_oracle(n, G, alpha):
    x, lab = cohort(n, G, n * 7 + G)
    F = 3
    res = run(x, lab, folds=F, repeats=1, alpha=alpha, seed=5)
    L = res.n_lambda
    assert 2 <= L <= 100 and res.beta.shape == (L, G)
    ref = check_fit(res, x, lab, alpha, L)
    assert ref["L"] == L
    if G < n:
        np.testing.assert_allclose(res.beta, ref["beta"][:L], atol=1e-6)
        want = np.where(ref["entry"] < L, ref["entry"], -1)
        # a gene whose coefficient is within the tolerance of 0 when it enters may enter one lambda apart
        differ = np.nonzero(res.entry[0] != want)[0]
        assert all(min(res.entry_abs[0][j], ref["entry_abs"][j]) < 1e-5 or abs(int(res.entry[0][j]) - want[j]) <= 1
                   for j in differ), differ
    assert res.entry[0][G - 1] == -1 and (res.entry[:, G - 1] == -1).all()
    # every fold fit against the oracle on its own training samples, with the shared lambdas
    y = lab.astype(np.float64)
    if G < n:
        for f in range(F):
            te = res.folds[0] == f
            fit = orc.path(x[~te], y[~te], alpha, lams=res.lambdas)
            for li in range(L):
                np.testing.assert_allclose(res.scores[li, 0, te], orc.predict(fit, x[te], li), atol=1e-5)
    assert (res.kkt <= 1e-7).sum() == res.converged
    assert res.converged == res.fits * L


def test_lambda_max_is_null_and_certified():
    x, lab = cohort(50, 30, 3)
    res = run(x, lab, folds=5)
    assert not res.beta[0].any() and res.df[0] == 0 and res.kkt[0, 0] <= 1e-7
    z, mu, sd, const = orc.standardise(x)
    ref = orc.lambdas(z, lab.astype(np.float64), 1.0)
    np.testing.assert_allclose(res.lambdas, ref[:res.n_lambda], rtol=1e-12)


def test_determinism_and_chunking():
    x, lab = cohort(45, 90, 11)
    a = run(x, lab, folds=4, repeats=2, alpha=0.5)
    b = run(x, lab, folds=4, repeats=2, alpha=0.5)
    c = run(x, lab, folds=4, repeats=2, alpha=0.5, max_chunk_bytes=1)
    for r in (b, c):
        for name in ("lambdas", "a0", "beta", "df", "dev_ratio", "cvm", "cvsd", "auc", "entry", "entry_abs", "kkt",
                     "scores"):
            assert np.array_equal(getattr(a, name), getattr(r, name)), name
        assert a.n_lambda == r.n_lambda and a.i_min == r.i_min and a.i_1se == r.i_1se


def test_separable_stops_by_deviance_and_carries_folds():
    rs = np.random.RandomState(4)
    n, G = 40, 10
    x = rs.randn(n, G)
    lab = (np.arange(n) % 2).astype(np.int64)
    x[:, 0] += 6.0 * lab                               # separable on one gene
    res = run(x, lab, folds=3)
    assert res.n_lambda < 100
    assert res.dev_ratio[-1] > 0.999 or res.dev_ratio[-1] - res.dev_ratio[-2] < 1e-5 * res.dev_ratio[-1]
    check_fit(res, x, lab, 1.0, res.n_lambda)
    check_carry(res)


def check_carry(res):
    """A fold fit that stopped (no Newton steps from some lambda on) reports its last solution: its held-out scores
    repeat bit for bit.  Returns how many fold fits carried."""
    K, F = res.auc.shape[1:]
    carried = 0
    for k in range(K):
        for f in range(F):
            it = res.n_iter[1 + k * F + f]
            s = len(it)
            while s > 1 and it[s - 1] == 0:
                s -= 1
            te = res.folds[k] == f
            for li in range(s, res.n_lambda):
                assert np.array_equal(res.scores[li, k, te], res.scores[s - 1, k, te]), (k, f, li)
            carried += s < res.n_lambda
    return carried


def test_active_cap_ends_the_path_and_folds_carry():
    rs = np.random.RandomState(8)
    n, G = 2000, 1200
    x = rs.randn(n, G)
    eta = x @ (rs.randn(G) * 0.08)
    lab = (rs.rand(n) < 1 / (1 + np.exp(-eta))).astype(np.int64)
    res = run(x, lab, folds=3)
    L = res.n_lambda
    entered = int((res.entry[0] >= 0).sum())
    assert L < 100 and entered <= 512 and res.dev_ratio[-1] < 0.999, (L, entered)
    assert (res.entry[1:] >= 0).sum(axis=1).max() <= 512
    # the path ended at the cap, not by the deviance rules
    assert not (L >= 5 and res.dev_ratio[-1] - res.dev_ratio[-2] < 1e-5 * res.dev_ratio[-1])
    z, mu, sd, const = orc.standardise(x)
    y = lab.astype(np.float64)
    for k in (L // 2, L - 1):
        assert res.kkt[0, k] <= 1e-7
        assert orc.kkt(z, y, res.a0[k], res.beta[k], res.lambdas[k], 1.0, const) <= 1e-7 + 1e-12
    check_carry(res)


def test_auc_equals_sig_auc_on_oracle_scores():
    import torch
    from g2vec_b200 import _capi
    x, lab = cohort(40, 25, 9)
    F, K = 4, 2
    res = run(x, lab, folds=F, repeats=K)
    L = res.n_lambda
    y = lab.astype(np.float64)
    sc = np.zeros((L, K, len(lab)))
    for k in range(K):
        for f in range(F):
            te = res.folds[k] == f
            fit = orc.path(x[~te], y[~te], 1.0, lams=res.lambdas)
            for li in range(L):
                sc[li, k, te] = orc.predict(fit, x[te], li)
    lib = _capi.load()
    d = torch.device("cuda")
    s_d = torch.from_numpy(sc).to(d)
    y_d = torch.from_numpy(lab.astype(np.uint8)).to(d)
    f_d = torch.from_numpy(res.folds).to(d)
    auc = torch.empty((L, K, F), dtype=torch.float64, device=d)
    acc = torch.empty_like(auc)
    n0, n1 = int((lab == 0).sum()), int((lab == 1).sum())
    cap = -(-n0 // F) + -(-n1 // F)
    _capi.check(lib.g2v_sig_auc(s_d.data_ptr(), y_d.data_ptr(), f_d.data_ptr(), len(lab), K, F, L, cap,
                                auc.data_ptr(), acc.data_ptr(), torch.cuda.current_stream().cuda_stream), "auc")
    np.testing.assert_array_equal(auc.cpu().numpy(), res.auc)


# ------------------------------------------------------------------------------------------------------- CLI
def test_command_line_writes_both_files_and_leaves_the_other_files_alone(tmp_path, capsys):
    import os
    import re
    from g2vec_b200 import cli, lasso, nested
    from tests import helpers
    ef, cf, nf, genes = helpers.write_ex_tsv(tmp_path)
    base = ["-r", "2", "-e", "5", "--deterministic", "--signature-cv", "10", "--signature-folds", "5",
            "--signature-repeats", "1", "--nested-cv", "5"]
    a, b = str(tmp_path / "plain"), str(tmp_path / "lasso")
    cli.main([ef, cf, nf, a] + base)
    log_a = capsys.readouterr().out
    cli.main([ef, cf, nf, b] + base + ["--lasso", "5"])
    log_b = capsys.readouterr().out
    for suffix in ("_biomarkers.txt", "_lgroups.txt", "_vectors.txt", "_signature.txt", "_nested_cv.txt",
                   "_nested_selection.txt"):
        assert open(a + suffix, "rb").read() == open(b + suffix, "rb").read(), suffix
    assert not os.path.exists(a + "_lasso.txt") and not os.path.exists(a + "_lasso_path.txt")
    untimed = lambda log, prefix: [re.sub(r" \([0-9.]+ sec\)$", "", l).replace(prefix, "RES")
                                   for l in log.splitlines()]
    extra = [l for l in untimed(log_b, b) if l not in untimed(log_a, a)]
    assert len(extra) == 4 and extra[0].startswith("Namespace(") and "lasso=5, lasso_repeats=1, lasso_alpha=1.0" \
        in extra[0]
    assert extra[1].startswith("    lasso: alpha 1, 5-fold x 1 repeats, ") and "top_lasso AUC" in extra[1]
    assert "nested_lasso AUC" in extra[1]
    assert extra[2:] == ["    RES_lasso.txt", "    RES_lasso_path.txt"]
    # the same numbers from the library: lasso_cv, then nested_lasso = score_fit of each fold fit's top_lasso list
    data = cli.load_data(ef)
    data["label"] = cli.match_labels(cli.load_clinical(cf), data["sample"])
    data, net = cli.restrict(data, cli.load_network(nf))
    res = lasso.lasso_cv(data["expr"], data["label"], folds=5, seed=0)
    x, lab = lasso.check_inputs(data["expr"], data["label"], 5, 1, 1.0)
    rows = open(b + "_nested_cv.txt").read().splitlines()[1:6]
    gi = {g: i for i, g in enumerate(data["gene"])}
    lists = [[[gi[g] for g in r.split("\t")[-1].split(",")] for r in rows]]
    want = np.array([[nested.score_fit(x, lab, res.folds, 0, f, lasso.fold_top(res, 0, f, len(lists[0][f]))[None, :])
                      [0][0] for f in range(5)]])
    assert np.array_equal(lasso.nested_lasso(x, lab, res, lists, 0), want)
    assert ("nested_lasso AUC %.3f" % want.mean()) in extra[1]
    out = open(b + "_lasso.txt").read().splitlines()
    assert out[0] == "GeneSymbol\tLgroup(0:good,1:poor,2:other)\tEntry\tBeta_min\tBeta_1se\tFold_entered\tBiomarker"
    assert len(out) == len(data["gene"]) + 2 and out[-1] == extra[1].strip()
    for j in range(0, len(data["gene"]), 101):
        assert out[1 + j].split("\t")[:3] == [data["gene"][j], out[1 + j].split("\t")[1], str(res.entry[0][j])]
    path = open(b + "_lasso_path.txt").read().splitlines()
    assert len(path) == res.n_lambda + 1 and path[1 + res.i_min].split("\t")[-1] in ("min", "min,1se")
