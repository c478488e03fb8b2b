"""CPU checks of the sp_solve_sym oracle (tests/spsolve_oracle.c) against independent facts, of the host LD score regression
(snp_ldsc, R/ldsc.R), and of the host side of snp_ldpred2_inf / sp_solve_sym that runs without a GPU."""
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from bigsnpr_b200 import api
from tests import spsolve_ref as S
from tests.test_lassosum2_oracle import dense_of, example, pd_fixture  # noqa: F401  (example: module fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def zero_storage(n, compact):
    """An n x n SFBM that stores its diagonal as zeros."""
    p = np.arange(n + 1, dtype=np.float64)
    if compact:
        return n, p, np.zeros(n), np.arange(n, dtype=np.int32)
    data = np.zeros(2 * n)
    data[0::2] = np.arange(n)
    return n, p, data, None


def test_solves_the_linear_system():
    """||(R + D) x - b|| <= tol ||b|| (SciPy), and x equals numpy.linalg.solve to the condition-scaled tolerance."""
    R, st = pd_fixture()
    m = R.shape[0]
    rng = np.random.default_rng(4)
    b = rng.normal(size=m)
    A = sp.csc_matrix(R)
    for d in (np.array([0.0]), np.array([0.3]), rng.uniform(0.1, 2, m)):
        D = np.diag(np.broadcast_to(d, (m,)))
        for tol in (1e-6, 1e-10):
            x, it, err = S.solve(st, b, d, tol)
            res = A @ x + D @ x - b
            assert np.linalg.norm(res) <= tol * np.linalg.norm(b) * 1.0001
            assert 0 < it < 10 * m and err < tol
            want = np.linalg.solve(R + D, b)
            kappa = np.linalg.cond(R + D)
            assert np.linalg.norm(x - want) <= 2 * kappa * tol * np.linalg.norm(want)


def test_error_is_the_relative_residual():
    R, st = pd_fixture(m=120, seed=5)
    b = np.random.default_rng(6).normal(size=120)
    for maxiter in (1, 3, 7):
        x, it, err = S.solve(st, b, 0.2, 1e-12, maxiter)
        assert it == maxiter
        r = b - (R @ x + 0.2 * x)  # the recursive residual differs from the true one by rounding only
        assert abs(err - np.linalg.norm(r) / np.linalg.norm(b)) < 1e-10


def test_every_exit(example):  # noqa: F811
    """b = 0; tol >= 1 (iters 0); maxiter reached with error > tol; a NaN failure; and the ordinary convergence."""
    R, st = pd_fixture()
    m = R.shape[0]
    b = np.random.default_rng(7).normal(size=m)
    x, it, err = S.solve(st, np.zeros(m), 0.5)
    assert it == 0 and err == 0 and not x.any()
    x, it, err = S.solve(st, b, 0.5, tol=2.0)  # |b|^2 < 4 |b|^2 before the first iteration: x stays 0
    assert it == 0 and err == 1.0 and not x.any()
    x, it, err = S.solve(st, b, 0.5, tol=1.0)  # iterates until |r| < |b| (not always after one step), uncounted
    assert it <= 3 and 0 < err < 1 and x.any()
    x, it, err = S.solve(st, b, 0.5, tol=1e-14, maxiter=5)
    assert it == 5 and err > 1e-14
    x, it, err = S.solve(st, b, 0.5, tol=1e-10)
    assert 0 < it < 10 * m and err < 1e-10
    for compact in (False, True):  # zero matrix, zero diagonal: alpha = |b|^2 / 0
        x, it, err = S.solve(zero_storage(6, compact), np.ones(6), 0.0, maxiter=4)
        assert np.isnan(err) and it == 4
    # maxiter = 0: no iteration, the residual is b
    x, it, err = S.solve(st, b, 0.5, maxiter=0)
    assert it == 0 and err == 1.0 and not x.any()


def test_storage_forms_agree(example):  # noqa: F811
    """Compact and non-compact storage agree to 1e-12 relative; they are not bit-identical in general, because the zeros
    filled into compact columns shift which lane folds which entry."""
    (p, i, x), df = example
    n = len(p) - 1
    rng = np.random.default_rng(8)
    b = rng.normal(size=n) * 0.05
    d = n / (0.3 * df["n_eff"])
    got = [S.solve(api.sfbm_storage((p, i, x), compact=c), b, d, 1e-10) for c in (False, True)]
    assert got[0][1] == got[1][1] or abs(got[0][1] - got[1][1]) <= 1
    assert np.max(np.abs(got[0][0] - got[1][0])) <= 1e-12 * np.max(np.abs(got[0][0]))


def test_thread_count_changes_nothing(example):  # noqa: F811
    (p, i, x), df = example
    st = api.sfbm_storage((p, i, x))
    b = np.random.default_rng(9).normal(size=st[0])
    a = S.solve(st, b, 3.0, 1e-10, nthreads=1)
    c = S.solve(st, b, 3.0, 1e-10, nthreads=4)
    assert a[0].tobytes() == c[0].tobytes() and a[1:] == c[1:]


def test_oracle_is_uncontracted():
    S.lib()
    src = open(os.path.join(ROOT, "tests", "spsolve_ref.py")).read()
    assert "-ffp-contract=off" in src
    out = subprocess.run(["objdump", "-d", S.lib()._name], capture_output=True, text=True).stdout
    assert "vfmadd" not in out


# ---- LD score regression ----------------------------------------------------------------------------------------------

def ldsc_inputs(M=3000, seed=1):
    rng = np.random.default_rng(seed)
    ld = rng.uniform(1, 60, M)
    N = np.round(rng.uniform(5e3, 2e4, M))
    return ld, N


@pytest.mark.parametrize("intercept", [None, 1.07])
def test_ldsc_noise_free(intercept):
    """chi2 = int + N h2 ld / M (the 1e-8 the function adds taken off beforehand) returns int and h2."""
    ld, N = ldsc_inputs()
    M, h2, it = ld.size, 0.35, 1.07
    chi2 = it + N * h2 * ld / M - 1e-8
    got = api.snp_ldsc(ld, M, chi2, N, blocks=None, intercept=intercept)
    assert got.shape == (2,)
    assert abs(got[0] - it) < 1e-10 and abs(got[1] - h2) < 1e-10
    got = api.snp_ldsc(ld, M, chi2 - 1e-8, N, blocks=50, intercept=intercept)  # its fits add 1e-8 a second time
    assert got.shape == (4,)
    assert abs(got[0] - it) < 1e-10 and abs(got[2] - h2) < 1e-10 and got[1] < 1e-8 and got[3] < 1e-8


def test_ldsc_thresholds_and_scalar_sample_size():
    """Variants with chi2 >= chi2_thr2 leave step 2; a scalar sample size stands for all."""
    ld, _ = ldsc_inputs(M=2000, seed=2)
    rng = np.random.default_rng(3)
    M = ld.size
    chi2 = 1.0 + 1e4 * 0.2 * ld / M + rng.normal(size=M) * 0.1
    chi2[:10] = 500.0  # outliers, out of both steps below
    a = api.snp_ldsc(ld, M, chi2, 1e4, blocks=None, chi2_thr2=100)
    b = api.snp_ldsc(ld[10:], M, chi2[10:], np.full(M - 10, 1e4), blocks=None, chi2_thr2=100)
    assert np.array_equal(a, b)


def test_ldsc_jackknife_pseudovalues():
    """The delete-a-block jackknife on a block vector equals its pseudovalue formulas restated directly."""
    ld, N = ldsc_inputs(M=1200, seed=4)
    rng = np.random.default_rng(5)
    M = ld.size
    chi2 = 1.02 + N * 0.3 * ld / M + rng.normal(size=M) * 0.5
    blocks = rng.integers(1, 13, M) * 7  # unsorted labels, uneven sizes
    got = api.snp_ldsc(ld, M, chi2, N, blocks=blocks, intercept=None)
    c = chi2 + 1e-8
    full = api.snp_ldsc(ld, M, c, N, blocks=None)
    labs = np.unique(blocks)
    h = np.array([M / np.sum(blocks == lab) for lab in labs])
    dele = np.array([api.snp_ldsc(ld[blocks != lab], M, c[blocks != lab], N[blocks != lab], blocks=None) for lab in labs])
    ps_int = h * full[0] - (h - 1) * dele[:, 0]
    ps_h2 = h * full[1] - (h - 1) * dele[:, 1]
    int_j, h2_j = np.sum(ps_int / h), np.sum(ps_h2 / h)
    want = [int_j, np.sqrt(np.mean((ps_int - int_j) ** 2 / (h - 1))), h2_j, np.sqrt(np.mean((ps_h2 - h2_j) ** 2 / (h - 1)))]
    assert np.array_equal(got, np.array(want))
    assert 0.2 < got[2] < 0.4 and got[3] > 0


def test_ldsc_block_count_is_consecutive_groups():
    """blocks = K: sort(rep_len(1:K, M)), the first M %% K blocks one variant larger."""
    ld, N = ldsc_inputs(M=1003, seed=6)
    chi2 = 1.0 + N * 0.2 * ld / 1003 + np.random.default_rng(7).normal(size=1003)
    lab = np.sort(np.resize(np.arange(1, 11), 1003))
    assert np.array_equal(np.bincount(lab)[1:], [101, 101, 101, 100, 100, 100, 100, 100, 100, 100])
    assert np.array_equal(api.snp_ldsc(ld, 1003, chi2, N, blocks=10), api.snp_ldsc(ld, 1003, chi2, N, blocks=lab))


# ---- argument checks, kernels, no GPU ---------------------------------------------------------------------------------

class FakeSFBM(api.SFBM):
    """An SFBM of the given shape with no device handle: for the checks that come before any device call."""

    def __init__(self, nrow, ncol):
        self._h, self._shape = None, (nrow, ncol)

    nrow = property(lambda self: self._shape[0])
    ncol = property(lambda self: self._shape[1])


def test_argument_checks():
    """tests/testthat/test-8-LDpred2.R:120 and the checks of R/LDpred2.R:29-32, R/ldsc.R:78-88 and :210-213."""
    df = {"beta": np.ones(3), "beta_se": np.ones(3), "n_eff": np.full(3, 100.0)}
    fake = FakeSFBM(3, 3)
    for k in ("beta", "beta_se", "n_eff"):
        with pytest.raises(ValueError, match="'df_beta' should have element '%s'." % k):
            api.snp_ldpred2_inf(fake, {kk: v for kk, v in df.items() if kk != k}, 0.3)
        with pytest.raises(ValueError, match="'df_beta' should have element '%s'." % k):
            api.snp_ldsc2(fake, {kk: v for kk, v in df.items() if kk != k})
    with pytest.raises(TypeError, match="'corr' is not of class 'SFBM'."):
        api.snp_ldpred2_inf(object(), df, 0.3)
    with pytest.raises(TypeError, match="'corr' is not of class 'SFBM'."):
        api.sp_solve_sym(object(), np.ones(3))
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        api.snp_ldpred2_inf(FakeSFBM(4, 4), df, 0.3)
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        api.snp_ldpred2_inf(FakeSFBM(4, 3), df, 0.3)
    with pytest.raises(ValueError, match="'df_beta\\$beta_se' should have only positive values."):
        api.snp_ldpred2_inf(fake, dict(df, beta_se=np.array([1.0, 0.0, 1.0])), 0.3)
    for h2 in (0, -0.1):
        with pytest.raises(ValueError, match="'h2' should have only positive values."):
            api.snp_ldpred2_inf(fake, df, h2)
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        api.sp_solve_sym(fake, np.ones(4))
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        api.sp_solve_sym(fake, np.ones(3), add_to_diag=np.ones(2))
    with pytest.raises(ValueError, match="all\\(ind.beta %in% cols_along\\(corr\\)\\) is not TRUE"):
        api.snp_ldsc2(fake, df, ind_beta=[1, 2, 4])
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        api.snp_ldsc2(fake, df, ind_beta=[1, 2])
    ld = np.ones(3)
    with pytest.raises(ValueError, match="'chi2' should have only positive values."):
        api.snp_ldsc(ld, 3, np.array([1.0, -1.0, 2.0]), 100)
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        api.snp_ldsc(ld, 3, np.ones(4), 100)
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        api.snp_ldsc(ld, 3, np.ones(3), np.ones(2))
    with pytest.raises(ValueError, match="'ld_size' should contain only integers."):
        api.snp_ldsc(ld, 3.5, np.ones(3), 100)
    with pytest.raises(ValueError, match="'ld_size' should be of length 1."):
        api.snp_ldsc(ld, [3, 3], np.ones(3), 100)


def test_solver_kernel_code(tmp_path):
    """The solver kernels have no spills, and their PTX no fused multiply-add: every product and sum rounds once, as the
    oracle's (the divisions stay div.rn.f64)."""
    from bigsnpr_b200 import build

    so = build.build()
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    funs = [f for f in sass.split("Function : ") if "k_cg_" in f.split("\n", 1)[0]]
    assert len(funs) == 6
    for f in funs:
        assert "STL" not in f and "LDL" not in f
    ptx = tmp_path / "sparse.ptx"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-ptx", "-arch=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-I",
                           os.path.join(ROOT, "bigsnpr_b200", "csrc"),
                           os.path.join(ROOT, "bigsnpr_b200", "csrc", "bsg_sparse.cu"), "-o", str(ptx)])
    bodies = dict(re.findall(r"\.entry \w*?(k_cg_\w+?)E\w*\((.*?)\n}\n", ptx.read_text(), re.S))
    assert set(bodies) == {"k_cg_init", "k_cg_init_fold", "k_cg_matvec", "k_cg_pt", "k_cg_update", "k_cg_direction"}
    for name, body in bodies.items():
        assert "fma.rn.f64" not in body, name
    assert "div.rn.f64" in bodies["k_cg_update"] and "div.rn.f64" in bodies["k_cg_direction"]
    assert "mul.rn.f64" in bodies["k_cg_matvec"] and "add.rn.f64" in bodies["k_cg_matvec"]


def test_no_gpu_fails_loudly():
    """Without a CUDA device the SFBM cannot be staged, and the solver refuses a missing handle: no CPU fallback."""
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    from bigsnpr_b200 import BsgError, _lib

    n, p, data, first_i = zero_storage(4, False)
    with pytest.raises(BsgError, match="no CPU fallback|CUDA"):
        api.SFBM(n, n, p, data, first_i)
    b, d, x = np.ones(4), np.ones(1), np.empty(4)
    it, err = _lib.C.c_int(), _lib.C.c_double()
    rc = _lib.lib().bsg_sfbm_solve(None, api._pd(b), api._pd(d), 1, 1e-10, 10, api._pd(x), _lib.C.byref(it),
                                   _lib.C.byref(err))
    assert rc == 9

