"""snp_lassosum2 and ld_scores_sfbm on the device against the CPU oracle (tests/lassosum2_oracle.c): beta_est and num_iter
bit-identical, in both SFBM storage forms."""
import os

import numpy as np
import pytest

import bigsnpr_b200 as B
from bigsnpr_b200 import _lib, api
from tests import lassosum2_ref as L
from tests.test_lassosum2_oracle import exit_kinds, sumstats

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def bed_fixture(name, seed):
    g = B.Bed(os.path.join(GOLD, name), device=0)
    G = B.read_bed(g, g.rows_along(), g.cols_along(), na_val=3)
    poly = (np.flatnonzero(np.nanstd(np.where(G == 3, np.nan, G), 0) > 0) + 1).astype(np.int32)
    corr = B.bed_cor(g, ind_col=poly, size=500)
    return g, poly, corr, sumstats(G[:, poly - 1], seed)


@pytest.fixture(scope="module")
def example():
    return bed_fixture("example.bed", 1)


@pytest.fixture(scope="module")
def example_missing():
    return bed_fixture("example-missing.bed", 2)


def check_grid(corr, df, compact, ind_corr=None, **kw):
    """snp_lassosum2 on the device == the oracle's grid on the same storage, bit for bit; returns the result."""
    sf = B.as_SFBM(corr, compact=compact)
    try:
        got = B.snp_lassosum2(sf, df, ind_corr=ind_corr, **kw)
    finally:
        sf.close()
    st = api.sfbm_storage(corr, compact=compact)
    keys = ("delta", "nlambda", "lambda_min_ratio")
    bh, sc, lam, dp1, gl, gd = L.grid_inputs(df, **{k: kw[k] for k in keys if k in kw})
    ind = np.arange(bh.size) if ind_corr is None else np.asarray(ind_corr) - 1
    want, it = L.lassosum2(st, bh, ind, lam, dp1, kw.get("dfmax", 200e3), kw.get("maxiter", 1000), kw.get("tol", 1e-5))
    gp = got.grid_param
    assert np.array_equal(np.asarray(got), want * sc[:, None], equal_nan=True)
    assert np.array_equal(gp["num_iter"], it)
    assert np.array_equal(gp["lambda"], gl) and np.array_equal(gp["delta"], gd)
    assert np.all(gp["time"] > 0)
    return got, want, it


@pytest.mark.parametrize("compact", [False, True])
def test_example_default_grid(example, compact):
    g, poly, corr, df = example
    got, want, it = check_grid(corr, df, compact)
    assert got.shape == (poly.size, 120)
    assert {"converged", "diverged"} <= exit_kinds(want, it, 1000, 200e3)


@pytest.mark.parametrize("compact", [False, True])
def test_example_missing_default_grid(example_missing, compact):
    g, poly, corr, df = example_missing
    check_grid(corr, df, compact)


@pytest.mark.parametrize("compact", [False, True])
def test_every_exit(example, compact):
    g, poly, corr, df = example
    seen = set()
    for dfmax, maxiter in ((200e3, 4), (20, 1000)):
        got, want, it = check_grid(corr, df, compact, dfmax=dfmax, maxiter=maxiter)
        seen |= exit_kinds(want, it, maxiter, dfmax)
    assert {"maxiter", "dfmax"} <= seen


@pytest.mark.parametrize("compact", [False, True])
def test_synth_ld_matrix(compact):
    """bsg_open_synth_ld, 2,000 samples x 20,000 SNPs, 100-SNP window."""
    n, m = 2000, 20000
    g = B.Bed.synthetic(n, m, seed=11, ld_rho=0.9, ld_block=50)
    G = B.read_bed(g, g.rows_along(), g.cols_along(), na_val=3)
    keep = (np.flatnonzero(G.std(0) > 0) + 1).astype(np.int32)
    corr = B.bed_cor(g, ind_col=keep, size=100)
    g.close()
    df = sumstats(G[:, keep - 1], 5)
    del G
    check_grid(corr, df, compact, nlambda=10, maxiter=200)


def test_more_points_than_sms(example):
    g, poly, corr, df = example
    got, _, _ = check_grid(corr, df, False, nlambda=60, maxiter=200)
    assert got.shape[1] == 240


def test_subset_unsorted_with_repeat_and_one_point(example):
    """The C ABI: ngrid = 1, and an unsorted ind_sub with a repeated column (two coordinates on one column)."""
    g, poly, corr, df = example
    rng = np.random.default_rng(3)
    n = poly.size
    sub = rng.choice(n, 800, replace=False).astype(np.int32)
    sub[5] = sub[700]
    bh, sc, lam, dp1, gl, gd = L.grid_inputs({k: v[sub] for k, v in df.items()}, nlambda=10)
    for compact in (False, True):
        sf = B.as_SFBM(corr, compact=compact)
        st = api.sfbm_storage(corr, compact=compact)
        for cols in (slice(0, lam.shape[1]), slice(12, 13)):
            la, dp = np.asfortranarray(lam[:, cols]), np.asfortranarray(dp1[:, cols])
            ng = la.shape[1]
            beta, it, secs = np.empty((sub.size, ng), order="F"), np.empty(ng, dtype=np.int32), np.empty(ng)
            _lib.check(_lib.lib().bsg_lassosum2(sf._h, api._pd(bh), sub.size, api._pi(sub), ng, api._pd(la), api._pd(dp),
                                                200e3, 300, 1e-5, api._pd(beta), api._pi(it), api._pd(secs)))
            want, it0 = L.lassosum2(st, bh, sub, la, dp, 200e3, 300, 1e-5)
            assert np.array_equal(beta, want, equal_nan=True) and np.array_equal(it, it0)
        sf.close()


def test_two_calls_identical(example):
    """tests/testthat/test-9-lassosum2.R:49-51: no sampling, so reproducible."""
    g, poly, corr, df = example
    sf = B.as_SFBM(corr)
    a = B.snp_lassosum2(sf, df, nlambda=12, maxiter=100)
    b = B.snp_lassosum2(sf, df, nlambda=12, maxiter=100)
    sf.close()
    assert np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)
    assert np.array_equal(a.grid_param["num_iter"], b.grid_param["num_iter"])
    assert np.array_equal(a.grid_param["sparsity"], b.grid_param["sparsity"], equal_nan=True)


@pytest.mark.parametrize("compact", [False, True])
def test_ld_scores_sfbm(example, compact):
    g, poly, corr, df = example
    sf = B.as_SFBM(corr, compact=compact)
    st = api.sfbm_storage(corr, compact=compact)
    rng = np.random.default_rng(8)
    for sub in (np.arange(poly.size), rng.choice(poly.size, 900, replace=False)):
        got = B.ld_scores_sfbm(sf, sub + 1)  # 1-based, like ind_corr
        want = L.ld_scores(st, sub)
        assert np.allclose(got, want, rtol=1e-12, atol=0)
    sf.close()


def test_ld_scores_sfbm_equals_bed_ld_scores(example):
    """test-2-ld-scores.R:24-27 on the sparse side, on the polymorphic SNPs of example.bed."""
    g, poly, _, _ = example
    corr = B.bed_cor(g, ind_col=poly, size=300, fill_diag=True)
    sf = B.as_SFBM(corr)
    got = B.ld_scores_sfbm(sf)
    sf.close()
    want = B.bed_ld_scores(g, ind_col=poly, size=300)
    assert np.max(np.abs(got - want)) < 1e-10


def test_errors():
    L_ = _lib.lib()

    def open_(nrow, ncol, p, data, first_i=None):
        h = _lib.vp()
        p, data = np.asarray(p, dtype=np.float64), np.asarray(data, dtype=np.float64)
        fi = None if first_i is None else np.asarray(first_i, dtype=np.int32)
        rc = L_.bsg_sfbm_open(nrow, ncol, api._pd(p), api._pd(data), api._pi(fi), 0, _lib.C.byref(h))
        return rc, h

    # malformed p / rows / compact spans
    assert open_(3, 3, [1, 1, 1, 1], [0, 1.0])[0] == 9
    assert open_(3, 3, [0, 2, 1, 2], [0, 1.0, 1, 0.5, 2, 1.0, 2, 1.0])[0] == 9
    assert open_(3, 3, [0, 1.5, 2, 3], [0, 1.0, 1, 1.0, 2, 1.0])[0] == 9
    assert open_(3, 3, [0, 1, 2, 3], [0, 1.0, 3, 1.0, 2, 1.0])[0] == 9
    assert open_(3, 3, [0, 1, 2, 3], [0, 1.0, 0.5, 1.0, 2, 1.0])[0] == 9
    assert open_(3, 3, [0, 2, 3, 4], [1, 1.0, 1, 1.0, 1, 1.0, 2, 1.0])[0] == 9  # a row stored twice in one column
    assert open_(3, 3, [0, 1, 2, 4], [1.0, 1.0, 1.0, 1.0], [0, 1, 2])[0] == 9
    # non-square: lassosum2 refuses it, ld_scores reads it
    rc, h = open_(4, 3, [0, 1, 2, 3], [0, 1.0, 1, 1.0, 3, 1.0])
    assert rc == 0 and L_.bsg_sfbm_nrow(h) == 4 and L_.bsg_sfbm_ncol(h) == 3
    one = np.ones(3)
    sub = np.arange(3, dtype=np.int32)
    beta, it = np.empty(3), np.empty(1, dtype=np.int32)
    rc = L_.bsg_lassosum2(h, api._pd(one), 3, api._pi(sub), 1, api._pd(one), api._pd(one), 10.0, 10, 1e-5, api._pd(beta),
                          api._pi(it), None)
    assert rc == 1 and "Incompatibility" in L_.bsg_last_error().decode()
    L_.bsg_sfbm_close(h)
    rc, h = open_(3, 3, [0, 1, 2, 3], [0, 1.0, 1, 1.0, 2, 1.0])
    bad = np.array([0, 3, 1], dtype=np.int32)
    rc = L_.bsg_lassosum2(h, api._pd(one), 3, api._pi(bad), 1, api._pd(one), api._pd(one), 10.0, 10, 1e-5, api._pd(beta),
                          api._pi(it), None)
    assert rc == 2
    out = np.empty(3)
    assert L_.bsg_sfbm_ld_scores(h, api._pi(bad), 3, api._pd(out)) == 2
    L_.bsg_sfbm_close(h)
    with pytest.raises(ValueError, match="ind.corr"):
        sf = B.as_SFBM((np.array([0, 1, 2]), np.array([0, 1]), np.ones(2)))
        B.snp_lassosum2(sf, {"beta": np.ones(2), "beta_se": np.ones(2), "n_eff": np.ones(2)}, ind_corr=[1, 3])


@pytest.mark.parametrize("compact", [False, True])
def test_shim_entry_points_equal_the_c_abi(example, compact, tmp_path):
    """_bigsnpr_lassosum2 (8 arguments, one grid point per call) and _bigsnpr_ld_scores_sfbm (3) through the R shim, linked
    against the stand-in for R's C API, on an SFBM environment ($p, $first_i, $nrow, $ncol, $sbk) over a written data
    file: the results equal the C ABI's."""
    from tests.test_abi import build_shim_with_minir
    from tests.test_gpu_shim import MiniR

    g, poly, corr, df = example
    n, p, data, first_i = api.sfbm_storage(corr, compact=compact)
    sbk = tmp_path / "corr.sbk"
    data.tofile(sbk)
    R = MiniR(build_shim_with_minir(tmp_path))
    fields = dict(p=R.reals(p), nrow=R.ints([n]), ncol=R.ints([n]), sbk=R.s(str(sbk)))
    if compact:
        fields["first_i"] = R.ints(first_i)
    env = R.env(**fields)
    sf = api.SFBM(n, n, p, data, first_i)
    rng = np.random.default_rng(12)
    sub = rng.permutation(n)[:1200].astype(np.int32)
    got = R.vec(R.call("_bigsnpr_ld_scores_sfbm", env, R.ints(sub), R.ints([1])))
    want = np.empty(sub.size)
    _lib.check(_lib.lib().bsg_sfbm_ld_scores(sf._h, api._pi(sub), sub.size, api._pd(want)))
    assert np.array_equal(got, want)
    bh, sc, lam, dp1, gl, gd = L.grid_inputs({k: v[sub] for k, v in df.items()}, nlambda=4)
    ng = lam.shape[1]
    beta, it = np.empty((sub.size, ng), order="F"), np.empty(ng, dtype=np.int32)
    _lib.check(_lib.lib().bsg_lassosum2(sf._h, api._pd(bh), sub.size, api._pi(sub), ng, api._pd(lam), api._pd(dp1), 200e3,
                                        100, 1e-5, api._pd(beta), api._pi(it), None))
    for c in range(ng):  # R/lassosum2.R:56-69: one .Call per grid point
        res = R.call("_bigsnpr_lassosum2", env, R.reals(bh), R.reals(lam[:, c]), R.reals(dp1[:, c]), R.ints(sub),
                     R.reals([200e3]), R.ints([100]), R.reals([1e-5]))
        b = R.vec(R.L.minir_list_by_name(res, b"beta_est"))
        k = R.vec(R.L.minir_list_by_name(res, b"num_iter"))
        assert np.array_equal(b, beta[:, c], equal_nan=True) and int(k[0]) == it[c]
    assert R.L.minir_env_get(env, b".bsg_sfbm")  # the staged handle is cached in the environment
    sf.close()
