"""CPU checks of the big_univLinReg restatements (tests/gwas_ref.py): the literal fp64 statistic against per-SNP least
squares, the covariate glue, and the exact model of the device arithmetic against its stated bound."""
import os

import numpy as np
import pytest
from scipy import stats

from tests import gwas_ref as G

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def codes():
    return G.read_bed_codes(os.path.join(GOLDEN, "example.bed"), 517, 4542)


def _dense(codes, rows, cols):
    X = codes[np.ix_(rows, cols)].astype(np.float64)
    X[X == 3] = np.nan
    return X


def _ok_cols(X, lo=0.05):
    m = np.nanmean(X, axis=0) / 2
    return np.where(~np.isnan(X).any(axis=0) & (np.minimum(m, 1 - m) > lo))[0]


def test_fp64_matches_lstsq(codes):
    rng = np.random.default_rng(1)
    rows = np.arange(517)
    cols = rng.choice(4542, 300, replace=False)
    X = _dense(codes, rows, cols)
    covar = rng.normal(size=(517, 3))
    y = rng.normal(size=517) + 0.3 * np.nan_to_num(X[:, 7])
    U = G.covar_basis(covar, 517)
    assert U.shape[1] == 4
    est, se, score = G.univlinreg_fp64(X, y, U)
    C = np.column_stack([np.ones(517), covar])
    for j in _ok_cols(X)[:80]:
        A = np.column_stack([C, X[:, j]])
        coef, rss, *_ = np.linalg.lstsq(A, y, rcond=None)
        df = 517 - A.shape[1]
        s2 = rss[0] / df
        se_j = np.sqrt(s2 * np.linalg.inv(A.T @ A)[-1, -1])
        assert abs(est[j] - coef[-1]) <= 1e-10 * abs(coef[-1]) + 1e-14
        assert abs(se[j] - se_j) <= 1e-10 * se_j
    from bigsnpr_b200.api import MHTest

    res = MHTest(est, se, score, 517 - 4 - 1)
    ok = _ok_cols(X)
    p = 2 * stats.t.sf(np.abs(score[ok]), 512)
    np.testing.assert_allclose(10 ** res.predict()[ok], p, rtol=1e-10)
    np.testing.assert_allclose(res.predict(log10=False)[ok], p, rtol=1e-10)


def test_duplicated_covariates_dropped(codes):
    rng = np.random.default_rng(2)
    cov = rng.normal(size=(517, 2))
    U0 = G.covar_basis(cov, 517)
    U1 = G.covar_basis(np.column_stack([cov, cov[:, 1], np.ones(517)]), 517)
    assert U0.shape[1] == U1.shape[1] == 3
    X = _dense(codes, np.arange(517), np.arange(200))
    y = rng.normal(size=517)
    a = G.univlinreg_fp64(X, y, U0)
    b = G.univlinreg_fp64(X, y, U1)
    ok = _ok_cols(X)
    np.testing.assert_allclose(b[0][ok], a[0][ok], rtol=1e-10)
    np.testing.assert_allclose(b[1][ok], a[1][ok], rtol=1e-10)


def test_no_covariates_is_simple_regression(codes):
    rng = np.random.default_rng(3)
    X = _dense(codes, np.arange(517), np.arange(300))
    y = rng.normal(size=517)
    U = G.covar_basis(None, 517)
    assert U.shape[1] == 1
    est, se, _ = G.univlinreg_fp64(X, y, U)
    for j in _ok_cols(X)[:50]:
        x = X[:, j]
        xc, yc = x - x.mean(), y - y.mean()
        b = xc @ yc / (xc @ xc)
        rss = np.sum((yc - b * xc) ** 2)
        assert abs(est[j] - b) <= 1e-10 * abs(b) + 1e-14
        assert abs(se[j] - np.sqrt(rss / 515 / (xc @ xc))) <= 1e-10 * se[j]


def test_repeated_rows_count(codes):
    rng = np.random.default_rng(4)
    rows = np.concatenate([np.arange(517), rng.choice(517, 60)])
    X = _dense(codes, rows, np.arange(100))
    y = rng.normal(size=rows.size)
    cov = rng.normal(size=(rows.size, 2))
    U = G.covar_basis(cov, rows.size)
    est, se, _ = G.univlinreg_fp64(X, y, U)
    C = np.column_stack([np.ones(rows.size), cov])
    for j in _ok_cols(X)[:30]:
        A = np.column_stack([C, X[:, j]])
        coef, rss, *_ = np.linalg.lstsq(A, y, rcond=None)
        se_j = np.sqrt(rss[0] / (rows.size - 4) * np.linalg.inv(A.T @ A)[-1, -1])
        assert abs(est[j] - coef[-1]) <= 1e-10 * abs(coef[-1]) + 1e-14
        assert abs(se[j] - se_j) <= 1e-10 * se_j


def _check_model(vals, na, rows, cols, U, y, D=1, informative=1e-6):
    est, se, parts = G.univlinreg_model(vals, na, rows, cols, U, y, D=D, with_parts=True)
    X = vals[np.ix_(rows, cols)].astype(np.float64) / D
    X[na[np.ix_(rows, cols)]] = np.nan
    e0, s0, _ = G.univlinreg_fp64(X, y, U)
    assert np.array_equal(np.isnan(est), np.isnan(e0))
    be, bs = G.model_bound(parts, est, se)
    ok = ~np.isnan(est)
    assert ok.sum() > 0
    assert np.all(np.abs(est - e0)[ok] <= be[ok]), np.max((np.abs(est - e0) / be)[ok])
    assert np.all(np.abs(se - s0)[ok] <= bs[ok]), np.max((np.abs(se - s0) / bs)[ok])
    # the bound is informative: well below the statistics themselves (a nearly collinear column loses 1 / (1 - r^2))
    assert np.median((be / np.abs(est))[ok]) < informative
    return est, se


def test_model_within_bound_example(codes):
    rng = np.random.default_rng(5)
    rows = np.sort(np.concatenate([rng.choice(517, 400, replace=False), rng.choice(517, 30)]))
    cols = rng.choice(4542, 500)
    cov = rng.normal(size=(rows.size, 5)) + 3.0
    U = G.covar_basis(cov, rows.size)
    y = 170 + 10 * rng.normal(size=rows.size)
    _check_model(codes, codes == 3, rows, cols, U, y)


def test_model_within_bound_ld_slice():
    from tests.synth_ref import synth_matrix_ld

    A = synth_matrix_ld(3000, 300, seed=7, rho=0.9, ld_block=30)
    vals = np.ascontiguousarray(A)
    rng = np.random.default_rng(6)
    cov = rng.normal(size=(3000, 10))
    U = G.covar_basis(cov, 3000)
    y = vals[:, 10].astype(float) * 0.5 + rng.normal(size=3000)
    _check_model(vals, vals == 3, np.arange(3000), np.arange(300), U, y)


def test_model_within_bound_collinear_snp(codes):
    rng = np.random.default_rng(8)
    X = _dense(codes, np.arange(517), np.arange(4542))
    j = _ok_cols(X, 0.2)[0]
    x = X[:, j]
    xc = (x - x.mean()) / x.std()
    noise = rng.normal(size=517)
    noise -= noise.mean() + (noise @ xc) / 517 * xc
    noise /= noise.std()
    cov = xc * np.sqrt(0.999) + noise * np.sqrt(0.001)  # r^2(x, covariate) = 0.999
    assert abs(np.corrcoef(cov, x)[0, 1] ** 2 - 0.999) < 1e-9
    U = G.covar_basis(cov, 517)
    y = rng.normal(size=517) + 0.2 * cov
    est, se = _check_model(codes, codes == 3, np.arange(517), np.array([j, j + 1]), U, y, informative=1e-4)
    assert np.all(np.isfinite(est))


def test_model_dosage_within_bound():
    rng = np.random.default_rng(9)
    D = 100
    vals = rng.integers(0, 201, size=(800, 60)).astype(np.uint8)
    na = rng.random((800, 60)) < 0.002
    U = G.covar_basis(rng.normal(size=(800, 3)), 800)
    y = rng.normal(size=800)
    _check_model(vals, na, np.arange(800), np.arange(60), U, y, D=D)
