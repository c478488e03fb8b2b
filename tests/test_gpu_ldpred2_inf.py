"""sp_solve_sym / snp_ldpred2_inf on the device against the CPU oracle (tests/spsolve_oracle.c): x, iters and error
byte-identical, in both SFBM storage forms; snp_ldsc2 on an SFBM against snp_ldsc; the ABI errors."""
import warnings

import numpy as np
import pytest

import bigsnpr_b200 as B
from bigsnpr_b200 import _lib, api
from tests import spsolve_ref as S
from tests.test_gpu_lassosum2 import bed_fixture
from tests.test_lassosum2_oracle import sumstats
from tests.test_spsolve_oracle import zero_storage

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def example():
    return bed_fixture("example.bed", 1)


@pytest.fixture(scope="module")
def example_missing():
    return bed_fixture("example-missing.bed", 2)


@pytest.fixture(scope="module")
def synth():
    """bsg_open_synth_ld, 2,000 samples x 20,000 SNPs, 100-SNP window (the matrix of test_gpu_lassosum2)."""
    g = B.Bed.synthetic(2000, 20000, seed=11, ld_rho=0.9, ld_block=50)
    G = B.read_bed(g, g.rows_along(), g.cols_along(), na_val=3)
    keep = (np.flatnonzero(G.std(0) > 0) + 1).astype(np.int32)
    corr = B.bed_cor(g, ind_col=keep, size=100)
    g.close()
    df = sumstats(G[:, keep - 1], 5)
    return corr, df


def same(got, want):
    """x, iters and error byte for byte (NaN entries only as NaN: their sign and payload are not defined by IEEE)."""
    (x, it, err), (x0, it0, err0) = got, want[:3]
    assert it == it0
    nan = np.isnan(x0)
    assert np.array_equal(np.isnan(x), nan) and x[~nan].tobytes() == x0[~nan].tobytes()
    assert (np.isnan(err) and np.isnan(err0)) or np.float64(err).tobytes() == np.float64(err0).tobytes()


def check(storage, b, d, tol=1e-10, maxiter=None):
    n, p, data, first_i = storage
    sf = api.SFBM(n, n, p, data, first_i)
    try:
        got = api._sp_solve(sf, b, d, tol, maxiter)
    finally:
        sf.close()
    want = S.solve(storage, b, d, tol, maxiter)
    same(got, want)
    return got


def ldpred2_inputs(df, n, h2):
    N = df["n_eff"]
    scale = np.sqrt(N * df["beta_se"] ** 2 + df["beta"] ** 2)
    return df["beta"] / scale, scale, n / (h2 * N)


@pytest.mark.parametrize("compact", [False, True])
@pytest.mark.parametrize("which", ["example", "example_missing"])
def test_bed_cor_several_h2(which, compact, request):
    g, poly, corr, df = request.getfixturevalue(which)
    st = api.sfbm_storage(corr, compact=compact)
    for h2 in (0.05, 0.3, 1.0):
        bh, sc, d = ldpred2_inputs(df, poly.size, h2)
        x, it, err = check(st, bh, d)
        assert it > 0 and err < 1e-10
    x, it, err = check(st, bh, np.array([2.5]))  # one value added to every diagonal entry
    assert it > 0


@pytest.mark.parametrize("compact", [False, True])
def test_synth_ld_matrix(synth, compact):
    corr, df = synth
    n = len(corr[0]) - 1
    st = api.sfbm_storage(corr, compact=compact)
    bh, sc, d = ldpred2_inputs(df, n, 0.3)
    x, it, err = check(st, bh, d)
    assert it > 5 and err < 1e-10
    check(st, bh, np.array([0.8]), tol=1e-8, maxiter=40)


@pytest.mark.parametrize("compact", [False, True])
def test_every_exit(example, compact):
    g, poly, corr, df = example
    st = api.sfbm_storage(corr, compact=compact)
    n = poly.size
    bh, sc, d = ldpred2_inputs(df, n, 0.3)
    x, it, err = check(st, np.zeros(n), d)  # b = 0
    assert it == 0 and err == 0 and not x.any()
    x, it, err = check(st, bh, d, tol=2.0)  # no iteration: x = 0
    assert it == 0 and err == 1.0 and not x.any()
    x, it, err = check(st, bh, d, maxiter=0)
    assert it == 0 and err == 1.0
    x, it, err = check(st, bh, d, tol=1e-14, maxiter=3)  # maxiter reached
    assert it == 3 and err > 1e-14
    x, it, err = check(st, bh, 0.5, tol=1e-12, maxiter=130)  # more iterations than one block of the host loop
    x, it, err = check(zero_storage(n, compact), bh, 0.0, maxiter=5)  # zero matrix and diagonal: NaN
    assert np.isnan(err) and it == 5


def test_ldpred2_inf(example):
    """snp_ldpred2_inf = scale x the oracle's solve; two calls identical (test-8-LDpred2.R:166-168); cor(G beta_inf, y) >
    0.2 (:48-49) with the phenotype the sumstats come from."""
    g, poly, corr, df = example
    sf = B.as_SFBM(corr)
    h2 = B.snp_ldsc2(sf, df)[1]
    assert h2 > 0
    a = B.snp_ldpred2_inf(sf, df, h2=h2)
    b = B.snp_ldpred2_inf(sf, df, h2=h2)
    assert a.tobytes() == b.tobytes()
    bh, sc, d = ldpred2_inputs(df, poly.size, h2)
    x, it, err = S.solve(api.sfbm_storage(corr), bh, d, 1e-10)
    assert a.tobytes() == (x * sc).tobytes()
    sf.close()
    # the phenotype of sumstats(G, 1), regenerated
    G = B.read_bed(g, g.rows_along(), poly, na_val=3)
    rng = np.random.default_rng(1)
    n, m = G.shape
    X = G.astype(np.float64)
    X[G == 3] = np.nan
    mu = np.nanmean(X, 0)
    X = np.where(np.isnan(X), mu, X) - mu
    bt = np.zeros(m)
    causal = rng.choice(m, max(m // 20, 1), replace=False)
    bt[causal] = rng.normal(size=causal.size)
    y = X @ bt
    y = y / y.std() * np.sqrt(0.4) + rng.normal(size=n) * np.sqrt(0.6)
    assert np.allclose(X.T @ (y - y.mean()) / (X ** 2).sum(0), df["beta"], rtol=1e-10, atol=1e-12)
    assert np.corrcoef(X @ a, y)[0, 1] > 0.2


def test_sp_solve_sym_messages():
    n = 50
    st = zero_storage(n, False)
    sf = api.SFBM(n, n, st[1], st[2])
    with pytest.raises(RuntimeError, match="^Solver failed.$"):
        B.sp_solve_sym(sf, np.ones(n), 0.0, maxiter=3)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        x = B.sp_solve_sym(sf, np.ones(n), 2.0, tol=0.0, maxiter=1)
    assert np.array_equal(x, np.full(n, 0.5))  # (0 + 2 I) x = 1 in one step; the error is 0, not above tol = 0
    assert not w
    sf.close()


@pytest.mark.parametrize("intercept", [1, None])
def test_ldsc2_equals_ldsc(example, intercept):
    """snp_ldsc2(SFBM) = snp_ldsc(ld_scores_sfbm) exactly, and snp_ldsc(bed_ld_scores) to 1e-10 (test-8-LDpred2.R:41-44)."""
    g, poly, _, df = example
    corr = B.bed_cor(g, ind_col=poly, size=300, fill_diag=True)
    sf = B.as_SFBM(corr)
    chi2 = (df["beta"] / df["beta_se"]) ** 2
    for blocks in (None, 20):
        got = B.snp_ldsc2(sf, df, blocks=blocks, intercept=intercept)
        want = B.snp_ldsc(B.ld_scores_sfbm(sf), poly.size, chi2, df["n_eff"], blocks=blocks, intercept=intercept)
        assert got.tobytes() == want.tobytes()
        ld = B.bed_ld_scores(g, ind_col=poly, size=300)
        alt = B.snp_ldsc(ld, poly.size, chi2, df["n_eff"], blocks=blocks, intercept=intercept)
        assert np.max(np.abs(got - alt)) < 1e-10
    sub = np.arange(2, poly.size, 3) + 1  # ind_beta: LD scores over all columns, regression on a subset
    d2 = {k: v[sub - 1] for k, v in df.items()}
    got = B.snp_ldsc2(sf, d2, ind_beta=sub, intercept=intercept)
    want = B.snp_ldsc(B.ld_scores_sfbm(sf)[sub - 1], poly.size, (d2["beta"] / d2["beta_se"]) ** 2, d2["n_eff"], blocks=None,
                      intercept=intercept)
    assert got.tobytes() == want.tobytes()
    sf.close()


def test_errors():
    L_ = _lib.lib()
    C = _lib.C

    def solve(h, b, d, dlen, tol, maxiter, x):
        it, err = C.c_int(), C.c_double()
        return L_.bsg_sfbm_solve(h, api._pd(b), api._pd(d), dlen, tol, maxiter, api._pd(x), C.byref(it), C.byref(err))

    b, d, x = np.ones(3), np.ones(3), np.empty(3)
    h = _lib.vp()
    p = np.array([0, 1, 2, 3], dtype=np.float64)
    _lib.check(L_.bsg_sfbm_open(4, 3, api._pd(p), api._pd(np.array([0, 1.0, 1, 1.0, 3, 1.0])), None, 0, C.byref(h)))
    assert solve(h, b, d, 3, 1e-10, 10, x) == 1  # non-square
    L_.bsg_sfbm_close(h)
    _lib.check(L_.bsg_sfbm_open(3, 3, api._pd(p), api._pd(np.array([0, 1.0, 1, 1.0, 2, 1.0])), None, 0, C.byref(h)))
    assert solve(h, b, d, 2, 1e-10, 10, x) == 1 and "Incompatibility" in L_.bsg_last_error().decode()
    assert solve(h, b, d, 0, 1e-10, 10, x) == 1
    assert solve(h, b, d, 3, -1e-3, 10, x) == 9
    assert solve(h, b, d, 3, float("nan"), 10, x) == 9
    assert solve(h, b, d, 3, 1e-10, -1, x) == 9
    assert solve(None, b, d, 3, 1e-10, 10, x) == 9
    assert solve(h, None, d, 3, 1e-10, 10, x) == 9
    assert solve(h, b, None, 3, 1e-10, 10, x) == 9
    assert solve(h, b, d, 3, 1e-10, 10, None) == 9
    it, err = C.c_int(), C.c_double()
    assert L_.bsg_sfbm_solve(h, api._pd(b), api._pd(d), 3, 1e-10, 10, api._pd(x), None, C.byref(err)) == 9
    assert L_.bsg_sfbm_solve(h, api._pd(b), api._pd(d), 3, 1e-10, 10, api._pd(x), C.byref(it), None) == 9
    assert solve(h, b, d, 3, 1e-10, 10, x) == 0 and np.array_equal(x, np.full(3, 0.5))
    assert L_.bsg_sfbm_last_solve_ms(h) > 0
    L_.bsg_sfbm_close(h)

