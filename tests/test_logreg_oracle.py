"""CPU checks of the big_univLogReg restatement (tests/logreg_ref.py): convergence to the maximum-likelihood fit, invariance
to the covariate basis, repeated rows, the refit path, the normal p-values of MHTest, and two anchors from the
reference's own tests (test-6-PRS.R's pval.rds and test-1-readBed.R's plink --assoc check)."""
import os

import numpy as np
import pytest
from scipy import stats

from tests import gwas_ref as G
from tests import logreg_ref as L

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
N, M = 517, 4542


@pytest.fixture(scope="module")
def codes():
    return G.read_bed_codes(os.path.join(GOLDEN, "example.bed"), N, M)


@pytest.fixture(scope="module")
def y01():
    return L.read_fam_affection(os.path.join(GOLDEN, "example.fam")).astype(np.float64) - 1


def _dense(codes, rows, cols):
    X = codes[np.ix_(rows, cols)].astype(np.float64)
    X[X == 3] = np.nan
    return X


def _ok(X, lo=0.05):
    m = np.nanmean(X, axis=0) / 2
    return ~np.isnan(X).any(axis=0) & (np.minimum(m, 1 - m) > lo)


def test_fixture_is_case_control(y01):
    assert int(y01.sum()) == 157 and int((1 - y01).sum()) == 360


def test_reaches_the_mle(codes, y01):
    rng = np.random.default_rng(1)
    cols = rng.choice(M, 200, replace=False)
    X = _dense(codes, np.arange(N), cols)
    covar = rng.normal(size=(N, 3))
    res = L.univlogreg(X, y01, covar)
    assert res["U"].shape[1] == 4
    conv = res["converged"] & _ok(X)
    assert conv.sum() > 150 and res["niter"][conv].max() <= 8
    C = np.column_stack([np.ones(N), covar])
    for j in np.flatnonzero(conv)[:60]:
        b, se = L.newton_mle(np.column_stack([C, X[:, j]]), y01)
        assert abs(res["estim"][j] - b[-1]) <= 1e-6 * abs(b[-1]) + 1e-12
        assert abs(res["std_err"][j] - se[-1]) <= 1e-6 * se[-1]


def test_null_model_is_glm(y01):
    rng = np.random.default_rng(2)
    covar = rng.normal(size=(N, 2))
    C = np.column_stack([np.ones(N), covar])
    coef, se, it, conv = L.glm_fit(C, y01)
    b, se0 = L.newton_mle(C, y01)
    assert conv and 3 <= it <= 8
    np.testing.assert_allclose(coef, b, rtol=1e-7, atol=1e-9)
    np.testing.assert_allclose(se, se0, rtol=1e-6)
    # the package's host copy is the same algorithm
    from bigsnpr_b200.api import logit_glm_fit

    c2, s2, it2, conv2 = logit_glm_fit(C, y01)
    np.testing.assert_allclose(c2, coef, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(s2, se, rtol=1e-12)
    assert (it2, conv2) == (it, conv)


def test_basis_invariance(codes, y01):
    """U from the SVD against the raw cbind(1, covar): the same span, so the same estimate of x to rounding.  std.err
    comes from the last H solved, evaluated at the previous iterate, which lies within about one step (< tol) of the
    optimum along a path that depends on the basis: it agrees to tol, not to rounding."""
    rng = np.random.default_rng(3)
    cols = rng.choice(M, 150, replace=False)
    X = _dense(codes, np.arange(N), cols)
    covar = rng.normal(size=(N, 4)) * [1, 10, 0.1, 3] + 2
    C = np.column_stack([np.ones(N), covar])
    a = L.univlogreg(X, y01, covar)
    b = L.irls(X, y01, C, L.glm_fit(C, y01)[0])
    ok = a["converged"] & b["converged"] & _ok(X)
    assert ok.sum() > 120
    np.testing.assert_allclose(a["estim"][ok], b["estim"][ok], rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(a["std_err"][ok], b["std_err"][ok], rtol=1e-8)


def test_repeated_rows_are_observations(codes, y01):
    """Rows given twice weigh twice: the fit equals the frequency-weighted MLE."""
    rng = np.random.default_rng(4)
    rows = np.concatenate([np.arange(N), rng.choice(N, 120, replace=False)])
    cols = rng.choice(M, 40, replace=False)
    X = _dense(codes, rows, cols)
    res = L.univlogreg(X, y01[rows])
    wts = np.bincount(rows, minlength=N).astype(np.float64)
    for j in np.flatnonzero(res["converged"] & _ok(X))[:20]:
        A = np.column_stack([np.ones(N), _dense(codes, np.arange(N), cols[j:j + 1])[:, 0]])
        beta = np.zeros(2)
        for _ in range(50):
            p = 1 / (1 + np.exp(-(A @ beta)))
            H = (A * (wts * p * (1 - p))[:, None]).T @ A
            step = np.linalg.solve(H, A.T @ (wts * (y01 - p)))
            beta += step
            if np.max(np.abs(step)) < 1e-14:
                break
        assert abs(res["estim"][j] - beta[1]) <= 1e-6 * abs(beta[1])


def test_separated_snp_is_refitted(codes, y01):
    X = _dense(codes, np.arange(N), np.arange(20))
    X[:, 5] = 2 * y01  # perfect separation: the IRLS diverges
    res = L.univlogreg(X, y01, maxiter=20)
    assert res["refitted"][5] and not res["converged"][5] and res["niter"][5] >= 1
    assert np.isfinite(res["estim"][5]) and res["estim"][5] > 5
    assert res["refitted"].sum() == 1


def test_nan_semantics(codes, y01):
    X = _dense(codes, np.arange(N), np.arange(10))
    X[:, 2] = 1.0
    X[7, 4] = np.nan
    res = L.univlogreg(X, y01)
    for j in (2, 4):
        assert np.isnan(res["estim"][j]) and np.isnan(res["std_err"][j]) and res["niter"][j] == 0
        assert not res["refitted"][j]


def test_mhtest_normal_pvalues():
    from bigsnpr_b200.api import MHTest

    rng = np.random.default_rng(5)
    e, s = rng.normal(size=50), rng.uniform(0.1, 1, size=50)
    r = MHTest(e, s, e / s, None)
    p = 2 * stats.norm.sf(np.abs(e / s))
    np.testing.assert_allclose(10 ** r.predict(), p, rtol=1e-12)
    np.testing.assert_allclose(r.predict(log10=False), p, rtol=1e-12)
    # a t-test result keeps the t distribution
    t = MHTest(e, s, e / s, 30)
    np.testing.assert_allclose(t.predict(log10=False), 2 * stats.t.sf(np.abs(e / s), 30), rtol=1e-12)


def reference_pcs(codes, oracle):
    """snp_autoSVD's first iteration on example.bed as test-6-PRS.R runs it: the MAF / MAC filter, clumping at r2 0.2
    over 500 kb, then the top 10 left singular vectors of the snp_scaleBinom-scaled kept columns (dense SVD).  Returns
    (u, kept columns, outliers the reference's detector flags)."""
    from bigsnpr_b200.outliers import autosvd_outlier_fun

    af = codes.astype(np.float64).sum(axis=0) / (2 * N)
    maf = np.minimum(af, 1 - af)
    nok = maf < max(0.02, 10 / (2 * N))
    bim = np.loadtxt(os.path.join(GOLDEN, "example.bim"), dtype=str)
    chrs, pos = bim[:, 0].astype(int), bim[:, 3].astype(float)
    F = oracle.OracleFBM(codes)
    keep = oracle.snp_clumping(F, chrs, thr_r2=0.2, size=500, infos_pos=pos, exclude=np.flatnonzero(nok) + 1)
    Xk = codes[:, keep - 1].astype(np.float64)
    p = Xk.mean(axis=0) / 2
    Z = (Xk - 2 * p) / np.sqrt(2 * p * (1 - p))
    u, d, vt = np.linalg.svd(Z, full_matrices=False)
    out = autosvd_outlier_fun()(vt[:10].T, chrs[keep - 1])
    return u[:, :10], keep, out


def test_reference_pvalues(codes, y01, oracle):
    """test-6-PRS.R:15-22: big_univLogReg(G, y01, covar.train = svd$u) against the reference's pval.rds, < 1e-4 mean
    relative difference (R's expect_equal tolerance)."""
    u, keep, out = reference_pcs(codes, oracle)
    assert keep.size == 4270 and out.size == 0
    X = codes.astype(np.float64)
    res = L.univlogreg(X, y01, u)
    pv = 2 * stats.norm.sf(np.abs(res["score"]))
    ref = np.load(os.path.join(GOLDEN, "prs_clumping.npz"))["pval"]
    ok = ~np.isnan(ref)
    assert np.array_equal(ok, ~np.isnan(pv))
    rel = np.mean(np.abs(pv[ok] - ref[ok])) / np.mean(np.abs(ref[ok]))
    assert rel < 1e-4, rel
    assert res["niter"][ok].min() >= 2 and res["niter"][ok].max() <= 6
    assert not res["refitted"].any()


def test_plink_assoc_stand_in(codes, y01):
    """test-1-readBed.R:65: without covariates the log odds ratios follow plink --assoc's allelic odds ratios
    (computed here from the case / control allele counts), correlation > 0.99."""
    X = codes.astype(np.float64)
    res = L.univlogreg(X, y01)
    a1 = X[y01 == 1].sum(axis=0)
    n1 = 2 * (y01 == 1).sum()
    a0 = X[y01 == 0].sum(axis=0)
    n0 = 2 * (y01 == 0).sum()
    with np.errstate(divide="ignore", invalid="ignore"):
        lor = np.log(a1 / (n1 - a1)) - np.log(a0 / (n0 - a0))
    ok = np.isfinite(lor) & np.isfinite(res["estim"])
    assert ok.sum() > 4000
    assert np.corrcoef(res["estim"][ok], lor[ok])[0, 1] > 0.99
