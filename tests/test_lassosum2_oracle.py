"""CPU checks of the lassosum2 / ld_scores_sfbm oracle (tests/lassosum2_oracle.c) against independent facts, and of the host
mirror of snp_lassosum2 / as_SFBM that runs without a GPU (R/lassosum2.R:25-81, bigsparser's storage)."""
import os

import numpy as np
import pytest

from bigsnpr_b200 import api
from tests import lassosum2_ref as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dense_of(storage):
    """The n x n matrix a storage holds."""
    n, p, data, first_i = storage
    D = np.zeros((n, n))
    p = p.astype(np.int64)
    for j in range(n):
        if first_i is None:
            rows, vals = data[2 * p[j]:2 * p[j + 1]:2].astype(np.int64), data[2 * p[j] + 1:2 * p[j + 1]:2]
        else:
            vals = data[p[j]:p[j + 1]]
            rows = first_i[j] + np.arange(vals.size)
        D[rows, j] = vals
    return D


def sumstats(G, seed):
    """Per-SNP OLS of a seeded phenotype on the genotypes (code 3 = missing, mean-imputed), with varying n_eff."""
    rng = np.random.default_rng(seed)
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
    y = y - y.mean()
    vx = (X ** 2).sum(0)
    beta = X.T @ y / vx
    se = np.sqrt(((y[:, None] - X * beta) ** 2).sum(0) / (n - 2) / vx)
    return {"beta": beta, "beta_se": se, "n_eff": np.round(n * rng.uniform(0.6, 1.0, m))}


@pytest.fixture(scope="module")
def example():
    """example.bed: 1,500 polymorphic SNPs, bed_cor at size = 500 (the oracle's), sumstats by OLS."""
    from oracle import ref

    o = ref.OracleBed(os.path.join(ROOT, "tests", "golden", "example.bed"))
    G = ref.read_bed(o, o.rows_along(), o.cols_along(), na_val=3)
    poly = np.flatnonzero(G.std(0) > 0)[:1500] + 1
    corr = ref.cor0(o, ind_col=poly, size=500)
    return corr, sumstats(G[:, poly - 1], 1)


def pd_fixture(m=200, seed=3):
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(1000, m)) + 0.3 * rng.normal(size=(1000, 1))
    R = np.corrcoef(A, rowvar=False)
    R = (R + R.T) / 2
    np.fill_diagonal(R, 1.0)
    assert np.linalg.eigvalsh(R).min() > 0.1
    import scipy.sparse as sp

    return R, api.sfbm_storage(sp.csc_matrix(R))


def test_solves_the_linear_system():
    """lambda = 0: the fixed point solves (R + diag(pf delta)) beta = beta_hat."""
    R, st = pd_fixture()
    m = R.shape[0]
    rng = np.random.default_rng(4)
    bh = rng.normal(size=m) * 0.05
    pf = np.sqrt(1 / rng.uniform(0.5, 1, m))
    for delta in (0.05, 0.5):
        dp1 = (pf * delta + 1)[:, None]
        b, it = L.lassosum2(st, bh, np.arange(m), np.zeros((m, 1)), dp1, 200e3, 100000, 1e-13)
        want = np.linalg.solve(R + np.diag(pf * delta), bh)
        assert it[0] < 100000
        assert np.max(np.abs(b[:, 0] - want)) < 1e-10


def test_kkt_conditions_at_converged_points(example):
    (p, i, x), df = example
    st = api.sfbm_storage((p, i, x))
    R = dense_of(st)
    bh, sc, lam, dp1, gl, gd = L.grid_inputs(df)
    tol, maxiter = 1e-5, 1000
    b, it = L.lassosum2(st, bh, np.arange(bh.size), lam, dp1, 200e3, maxiter, tol)
    bound = tol * np.abs(R - np.diag(np.diag(R))).sum(0) * 1.01 + 1e-12
    nconv = 0
    for g in range(b.shape[1]):
        if np.isnan(b[:, g]).any() or it[g] > maxiter:
            continue
        nconv += 1
        beta = b[:, g]
        resid = bh - R @ beta  # bh_j - (R beta)_j; R has a unit diagonal
        pen = (dp1[:, g] - 1) * beta
        nz = beta != 0
        assert np.all(np.abs(resid[nz] - pen[nz] - lam[nz, g] * np.sign(beta[nz])) <= bound[nz])
        assert np.all(np.abs(resid[~nz]) <= lam[~nz, g] + bound[~nz])
    assert nconv >= 20


def test_subset_equals_submatrix(example):
    """tests/testthat/test-9-lassosum2.R:53-59, bit for bit, in both storage forms, with an unsorted subset."""
    (p, i, x), df = example
    import scipy.sparse as sp

    st = api.sfbm_storage((p, i, x))
    full = sp.csc_matrix((st[2][1::2], st[2][0::2].astype(np.int64), st[1].astype(np.int64)), shape=(st[0], st[0]))
    rng = np.random.default_rng(9)
    sub = rng.choice(st[0], 600, replace=False)
    dsub = {k: v[sub] for k, v in df.items()}
    bh, sc, lam, dp1, gl, gd = L.grid_inputs(dsub, nlambda=10)
    want, it0 = L.lassosum2(api.sfbm_storage(full[sub][:, sub]), bh, np.arange(sub.size), lam, dp1, 200e3, 50, 1e-5)
    for compact in (False, True):
        got, it = L.lassosum2(api.sfbm_storage((p, i, x), compact=compact), bh, sub, lam, dp1, 200e3, 50, 1e-5)
        assert np.array_equal(got, want, equal_nan=True) and np.array_equal(it, it0)


def exit_kinds(b, it, maxiter, dfmax):
    kinds = set()
    for g in range(b.shape[1]):
        if np.isnan(b[:, g]).all():
            kinds.add("diverged")
        elif it[g] == maxiter + 1:
            kinds.add("maxiter")
        elif np.count_nonzero(b[:, g]) > dfmax:
            kinds.add("dfmax")
        else:
            kinds.add("converged")
    return kinds


def test_every_exit_occurs(example):
    """Convergence and divergence (example.bed's banded matrix is not positive definite) on the default grid, maxiter with
    maxiter = 4, dfmax with dfmax = 20."""
    (p, i, x), df = example
    st = api.sfbm_storage((p, i, x))
    bh, sc, lam, dp1, gl, gd = L.grid_inputs(df)
    seen = set()
    for dfmax, maxiter in ((200e3, 1000), (200e3, 4), (20, 1000)):
        b, it = L.lassosum2(st, bh, np.arange(bh.size), lam, dp1, dfmax, maxiter, 1e-5)
        assert np.all(it <= maxiter + 1)
        k = exit_kinds(b, it, maxiter, dfmax)
        seen |= k
        nan_cols = np.isnan(b).any(0)
        assert np.array_equal(nan_cols, np.isnan(b).all(0))  # a diverged point is NA in its whole column
        nb = b.view(np.uint64)[:, nan_cols]
        assert np.all(nb == np.uint64(0x7FF00000000007A2))  # R's NA_real_
    assert seen == {"converged", "diverged", "maxiter", "dfmax"}


def test_ld_scores_oracle(example):
    (p, i, x), _ = example
    st = api.sfbm_storage((p, i, x))
    R = dense_of(st)
    rng = np.random.default_rng(2)
    sub = rng.choice(st[0], 700, replace=False)
    want = (R[np.ix_(sub, sub)] ** 2).sum(0)
    for compact in (False, True):
        got = L.ld_scores(api.sfbm_storage((p, i, x), compact=compact), sub)
        assert np.allclose(got, want, rtol=1e-12, atol=0)


# ---- host mirror, no GPU ----------------------------------------------------------------------------------------------

def test_storage_both_forms_and_upper_expansion():
    rng = np.random.default_rng(5)
    n = 40
    D = np.zeros((n, n))
    for j in range(n):
        for k in range(max(0, j - 6), j + 1):
            if rng.uniform() < 0.7 or k == j:
                D[k, j] = rng.normal()
    D[3, 9] = 7.0
    import scipy.sparse as sp

    up = sp.csc_matrix(D)
    up.data[up.data == 7.0] = 0.0  # an explicit zero: kept as stored
    D[3, 9] = 0.0
    p, i, x = up.indptr.astype(np.int64), up.indices.astype(np.int32), up.data.copy()
    full = D + D.T - np.diag(np.diag(D))
    for corr, kw in (((p, i, x), {}), (up, {"upper": True}), (sp.csc_matrix(full), {})):
        for compact in (False, True):
            st = api.sfbm_storage(corr, compact=compact, **kw)
            assert st[0] == n and st[1][0] == 0 and np.all(np.diff(st[1]) >= 0)
            assert np.array_equal(dense_of(st), full)
            if compact:
                pp = st[1].astype(np.int64)
                for j in range(n):  # first_i = smallest stored row, values run to the largest one
                    rows = np.flatnonzero(full[:, j])
                    if rows.size:
                        assert st[3][j] <= rows[0] and st[3][j] + pp[j + 1] - pp[j] - 1 >= rows[-1]
            else:
                assert st[3] is None and st[2].size == 2 * st[1][-1]
                pp = st[1].astype(np.int64)
                for j in range(n):
                    r = st[2][2 * pp[j]:2 * pp[j + 1]:2]
                    assert np.all(np.diff(r) > 0)
    # the explicit zero of the upper triangle is stored in both of its columns
    st = api.sfbm_storage((p, i, x))
    pp = st[1].astype(np.int64)
    assert 3 in st[2][2 * pp[9]:2 * pp[10]:2] and 9 in st[2][2 * pp[3]:2 * pp[4]:2]
    with pytest.raises(ValueError, match="below the diagonal"):
        api.sfbm_storage(sp.csc_matrix(full), upper=True)


def test_storage_of_an_unsorted_tuple():
    """A (p, i, x) tuple with rows out of order and a repeated entry is stored like its canonical form."""
    rng = np.random.default_rng(6)
    n = 30
    D = np.triu(rng.normal(size=(n, n)) * (rng.uniform(size=(n, n)) < 0.4)) + np.diag(np.ones(n))
    import scipy.sparse as sp

    up = sp.csc_matrix(D)
    p, i, x = up.indptr.astype(np.int64), up.indices.copy(), up.data.copy()
    for j in range(n):  # reverse the rows of every column, split the diagonal of column 7 into two entries
        i[p[j]:p[j + 1]], x[p[j]:p[j + 1]] = i[p[j]:p[j + 1]][::-1].copy(), x[p[j]:p[j + 1]][::-1].copy()
    k = int(np.flatnonzero(i[p[7]:p[8]] == 7)[0]) + p[7]
    x[k] = x[k] / 2
    i, x = np.insert(i, k, 7), np.insert(x, k, x[k])
    p = p + (np.arange(n + 1) > 7)
    full = D + D.T - np.diag(np.diag(D))
    for compact in (False, True):
        st = api.sfbm_storage((p, i, x), compact=compact)
        assert np.array_equal(dense_of(st), full)
        assert np.array_equal(st[1], api.sfbm_storage((up.indptr, up.indices, up.data), compact=compact)[1])


def test_seq_log_and_grid_order():
    s = api.seq_log(1, 1000, 4)
    assert s[0] == 1 and abs(s[-1] - 1000) < 1e-9 and np.allclose(s, [1, 10, 100, 1000], rtol=1e-13)
    a, b = np.log(0.3), np.log(0.003)
    s = api.seq_log(0.3, 0.003, 31)
    inner = a + np.arange(1, 30) * ((b - a) / 30)  # seq(length.out =): both ends exact, the inner points from + i * by
    assert np.array_equal(np.log(s[1:-1]), np.log(np.exp(inner))) and s[0] == np.exp(a) and s[-1] == np.exp(b)
    rng = np.random.default_rng(1)
    df = {"beta": rng.normal(size=50) * 0.02, "beta_se": rng.uniform(0.01, 0.03, 50), "n_eff": rng.uniform(1e3, 2e3, 50)}
    delta = np.array([0.001, 0.01, 0.1, 1])
    got = api._lassosum2_grid(df["beta"], df["beta_se"], df["n_eff"], delta, 30, 0.01)
    want = L.grid_inputs(df)
    beta_hat, scale, g_lam, g_delta, lam, dp1 = got
    assert np.array_equal(beta_hat, want[0]) and np.array_equal(scale, want[1])
    assert np.array_equal(lam, want[2]) and np.array_equal(dp1, want[3])
    assert np.array_equal(g_lam, want[4]) and np.array_equal(g_delta, want[5])
    assert g_lam.size == 120 and np.array_equal(g_lam[:30], g_lam[30:60]) and np.all(np.diff(g_lam[:30]) < 0)
    assert np.array_equal(g_delta, np.repeat(delta, 30))  # expand.grid: lambda varies fastest
    assert g_lam[0] < np.max(np.abs(beta_hat / np.sqrt(df["n_eff"].max() / df["n_eff"])))  # seq_log(...)[-1]


def test_argument_checks_without_gpu():
    df = {"beta": np.ones(3), "beta_se": np.ones(3), "n_eff": np.ones(3)}
    fake = api.SFBM.__new__(api.SFBM)
    for k in ("beta", "beta_se", "n_eff"):
        with pytest.raises(ValueError, match="'df_beta' should have element '%s'." % k):
            api.snp_lassosum2(fake, {kk: v for kk, v in df.items() if kk != k})
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        api.snp_lassosum2(fake, df, ind_corr=[1, 2])
    with pytest.raises(TypeError, match="'corr' is not of class 'SFBM'."):
        api.snp_lassosum2(object(), df)


def test_oracle_is_uncontracted():
    """The oracle is built without FMA contraction, as the reference is."""
    import subprocess

    L.lib()
    src = open(os.path.join(ROOT, "tests", "lassosum2_ref.py")).read()
    assert "-ffp-contract=off" in src
    so = L.lib()._name
    out = subprocess.run(["objdump", "-d", so], capture_output=True, text=True).stdout
    assert "vfmadd" not in out


def test_lassosum2_kernel_code(tmp_path):
    """The device kernel has no spills, and its PTX no fused multiply-add: every update rounds twice, as the reference's
    (the division stays div.rn.f64, IEEE-rounded)."""
    import re
    import subprocess

    from bigsnpr_b200 import build

    so = build.build()
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    fun = [f for f in sass.split("Function : ") if f.split("\n", 1)[0].find("k_lassosum2") >= 0]
    assert len(fun) == 1 and "STL" not in fun[0] and "LDL" not in fun[0]
    ptx = tmp_path / "sparse.ptx"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-ptx", "-arch=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-I",
                           os.path.join(ROOT, "bigsnpr_b200", "csrc"),
                           os.path.join(ROOT, "bigsnpr_b200", "csrc", "bsg_sparse.cu"), "-o", str(ptx)])
    text = ptx.read_text()
    body = re.search(r"\.entry \w*k_lassosum2\w*\((.*?)\n}\n", text, re.S).group(1)
    assert "fma.rn.f64" not in body and "div.rn.f64" in body and "mul.rn.f64" in body and "add.rn.f64" in body
