"""big_univLogReg on the device (bsg_univlogreg) against the restatement of tests/logreg_ref.py: equal iteration counts and
refit sets, std.err within 1e-9 relative and estim within 1e-9 of max(|estim|, std.err) on converged SNPs, on both
storage forms, dosages, subsets and multisets, K = 0 / 10 / 20 covariates, an LD-structured 100,000-row matrix;
byte-identical results whatever else the call holds; the error paths; and test-6-PRS.R end to end (autoSVD -> logistic
GWAS -> clumping -> PRS)."""
import os

import numpy as np
import pytest

from tests import gwas_ref as G
from tests import logreg_ref as L

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
N, M = 517, 4542
NM, MM = 200, 500  # example-missing.bed
REL = 1e-9


@pytest.fixture(scope="module")
def B():
    import bigsnpr_b200 as B

    return B


@pytest.fixture(scope="module")
def codes():
    return G.read_bed_codes(os.path.join(GOLDEN, "example.bed"), N, M)


@pytest.fixture(scope="module")
def codes_missing():
    return G.read_bed_codes(os.path.join(GOLDEN, "example-missing.bed"), NM, MM)


@pytest.fixture(scope="module")
def y01():
    return L.read_fam_affection(os.path.join(GOLDEN, "example.fam")).astype(np.float64) - 1


def _same(a, b):
    na, nb = np.isnan(a), np.isnan(b)
    assert np.array_equal(na, nb)
    assert np.array_equal(a[~na].view(np.int64), b[~nb].view(np.int64))


def _same_res(r1, r2):
    _same(r1.estim, r2.estim)
    _same(r1.std_err, r2.std_err)
    assert np.array_equal(r1.niter, r2.niter) and np.array_equal(r1.refitted, r2.refitted)


def _dense(vals, na, rows0, cols0, D=1):
    Xd = vals[np.ix_(rows0, cols0)].astype(np.float64) / D
    Xd[na[np.ix_(rows0, cols0)]] = np.nan
    return Xd


def _check(B, X, vals, na, rows, cols, covar, y, D=1, tol=1e-8, maxiter=20):
    """rows / cols 1-based.  Device against the restatement on the same basis U."""
    res = B.big_univLogReg(X, y, ind_train=rows, ind_col=cols, covar_train=covar, tol=tol, maxiter=maxiter)
    U = B.api.univlinreg_covar_basis(covar, len(rows))
    ref = L.univlogreg(_dense(vals, na, np.asarray(rows) - 1, np.asarray(cols) - 1, D), y, tol=tol, maxiter=maxiter, U=U)
    assert res.df is None
    assert np.array_equal(np.isnan(res.estim), np.isnan(ref["estim"]))
    assert np.array_equal(np.isnan(res.std_err), np.isnan(ref["std_err"]))
    assert np.array_equal(res.refitted, ref["refitted"])
    # a step within 1e-6 relative of tol could fall on either side of it: such SNPs are listed, none expected
    st = ref["steps"]
    border = np.any(np.abs(st - tol) <= 1e-6 * tol, axis=1)
    assert not border.any(), np.flatnonzero(border)
    assert np.array_equal(res.niter, ref["niter"])
    ok = ~np.isnan(ref["estim"]) & ~ref["refitted"]
    if ok.any():
        # an estimate near 0 has no relative precision to speak of: its error is weighed against its standard error
        e_err = np.abs(res.estim[ok] - ref["estim"][ok]) / np.maximum(np.abs(ref["estim"][ok]), ref["std_err"][ok])
        s_rel = np.abs(res.std_err[ok] - ref["std_err"][ok]) / ref["std_err"][ok]
        assert np.all(e_err <= REL), e_err.max()
        assert np.all(s_rel <= REL), s_rel.max()
    rf = ref["refitted"]
    if rf.any():  # the host refit sees the same column; a separated SNP has no MLE, glm.fit stops where 25 steps end
        np.testing.assert_allclose(res.estim[rf], ref["estim"][rf], rtol=1e-6)
    return res, ref


@pytest.mark.parametrize("K", [0, 10, 20])
def test_example_bed(B, codes, y01, K):
    rng = np.random.default_rng(K)
    X = B.Bed(os.path.join(GOLDEN, "example.bed"))
    covar = rng.normal(size=(N, K)) if K else None
    res, ref = _check(B, X, codes, codes == 3, np.arange(1, N + 1), np.arange(1, M + 1), covar, y01)
    assert np.isfinite(res.estim).sum() > 4000
    F = B.Bed.from_fbm(codes)  # the FBM.code256 twin gives the same bytes
    _same_res(B.big_univLogReg(F, y01, covar_train=covar), res)


def test_example_missing_subsets(B, codes_missing):
    rng = np.random.default_rng(11)
    X = B.Bed(os.path.join(GOLDEN, "example-missing.bed"))
    F = B.Bed.from_fbm(codes_missing)
    rows = np.concatenate([rng.choice(NM, 150, replace=False), rng.choice(NM, 30)]) + 1
    cols = np.concatenate([rng.choice(MM, 700) + 1, [5, 5, 1, MM]])
    covar = rng.normal(size=(rows.size, 3))
    y = (rng.random(rows.size) < 0.4).astype(np.float64)
    res, _ = _check(B, X, codes_missing, codes_missing == 3, rows, cols, covar, y)
    assert np.isnan(res.estim).any() and np.isfinite(res.estim).any()
    assert np.all(res.niter[np.isnan(res.estim)] == 0)
    _same_res(B.big_univLogReg(F, y, ind_train=rows, ind_col=cols, covar_train=covar), res)


def test_dosage_fbm(B):
    rng = np.random.default_rng(12)
    code256 = np.full(256, np.nan)
    code256[:201] = np.arange(201) / 100
    D = B.code256_dosage_scale(code256)
    assert D == 100
    byt = rng.integers(0, 201, size=(900, 300)).astype(np.uint8)
    byt[rng.random(byt.shape) < 0.001] = 255
    F = B.Bed.from_fbm(byt, code256)
    vals = np.where(byt == 255, 0, byt)
    rows = np.concatenate([np.arange(1, 901), rng.choice(900, 40) + 1])
    cols = rng.choice(300, 350) + 1
    covar = rng.normal(size=(rows.size, 4))
    g = vals[rows - 1, 7] / 100.0
    y = (rng.random(rows.size) < 1 / (1 + np.exp(-(g - 1)))).astype(np.float64)
    res, _ = _check(B, F, vals, byt == 255, rows, cols, covar, y, D=D)
    assert np.isfinite(res.estim).sum() > 50


def test_constant_empty_and_separated(B, codes, y01):
    byt = codes.copy()
    byt[:, 0] = 1
    byt[:, 1] = 0
    byt[:, 2] = 2 * y01.astype(np.uint8)  # perfectly separated: IRLS does not meet tol, the host refits it
    F = B.Bed.from_fbm(byt)
    rng = np.random.default_rng(13)
    res, _ = _check(B, F, byt, byt == 3, np.arange(1, N + 1), np.arange(1, 40), rng.normal(size=(N, 2)), y01)
    assert np.isnan(res.estim[:2]).all() and np.isnan(res.std_err[:2]).all() and np.all(res.niter[:2] == 0)
    assert res.refitted[2] and res.refitted.sum() == 1
    empty = B.big_univLogReg(F, y01, ind_col=np.zeros(0, dtype=np.int32))
    assert empty.estim.size == 0 and empty.std_err.size == 0


def test_ld_synthetic_with_pcs(B):
    from tests.synth_ref import synth_matrix_ld

    n, m = 100_000, 2000
    X = B.Bed.synthetic(n, m, seed=77, ld_rho=0.9, ld_block=50)
    vals = synth_matrix_ld(n, m, seed=77, rho=0.9, ld_block=50)
    svd = B.bed_randomSVD(X, k=10)
    pcs = svd["u"] * svd["d"]
    rng = np.random.default_rng(14)
    g = 0.3 * (vals[:, 100].astype(float) - vals[:, 100].mean()) + pcs[:, 0] / np.std(pcs[:, 0])
    liab = g + rng.normal(size=n)
    y = (liab > np.quantile(liab, 0.7)).astype(np.float64)  # liability threshold, 30 % cases
    cols = rng.permutation(m) + 1
    res, _ = _check(B, X, vals, vals == 3, np.arange(1, n + 1), cols, pcs, y)
    assert abs(res.score[cols == 101][0]) > 5


def test_determinism(B, codes, y01):
    """A SNP's bytes do not depend on the other columns of the call, their order, repeats, or the call."""
    rng = np.random.default_rng(15)
    X = B.Bed(os.path.join(GOLDEN, "example.bed"))
    covar = rng.normal(size=(N, 5))
    full = B.big_univLogReg(X, y01, covar_train=covar)
    again = B.big_univLogReg(X, y01, covar_train=covar)
    _same_res(full, again)
    for cols in (rng.permutation(M) + 1, rng.choice(M, 37, replace=False) + 1,
                 np.concatenate([rng.choice(M, 500) + 1, [3, 3, 3]]), np.array([M])):
        r = B.big_univLogReg(X, y01, ind_col=cols, covar_train=covar)
        _same(r.estim, full.estim[cols - 1])
        _same(r.std_err, full.std_err[cols - 1])
        assert np.array_equal(r.niter, full.niter[cols - 1])


def test_errors(B, codes, y01):
    import ctypes as C

    from bigsnpr_b200 import _lib

    X = B.Bed(os.path.join(GOLDEN, "example.bed"))
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        B.big_univLogReg(X, y01[:-1])
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        B.big_univLogReg(X, y01, covar_train=np.ones((N - 1, 2)))
    y2 = y01.copy()
    y2[3] = 0.5
    with pytest.raises(ValueError, match="0s and 1s"):
        B.big_univLogReg(X, y2)
    with pytest.raises(ValueError, match="both"):
        B.big_univLogReg(X, np.zeros(N))
    with pytest.raises(B.BsgError) as e:
        B.big_univLogReg(X, y01, ind_col=[1, M + 1])
    assert e.value.code == 2
    with pytest.raises(B.BsgError) as e:
        B.big_univLogReg(X, y01[:3], ind_train=[1, 2, N + 1])
    assert e.value.code == 2
    code256 = np.full(256, np.nan)
    code256[:3] = [0, 0.1234567, 2]  # not a dosage table
    with pytest.raises(B.BsgError) as e:
        B.big_univLogReg(B.Bed.from_fbm(codes, code256), y01)
    assert e.value.code == 10
    with pytest.raises(B.BsgError) as e:
        B.big_univLogReg(X, y01, tol=0)
    assert e.value.code == 9
    with pytest.raises(B.BsgError) as e:
        B.big_univLogReg(X, y01, maxiter=0)
    assert e.value.code == 9
    # the C ABI's own checks: non-finite U or gamma0, a y01 entry other than 0 / 1
    L_ = _lib.lib()
    U = np.full(N, 1 / np.sqrt(N))
    g0 = np.zeros(1)
    out = np.empty(2), np.empty(2), np.empty(2, dtype=np.int32)
    cols = np.array([1, 2], dtype=np.int32)

    def call(U, g0, y):
        return L_.bsg_univlogreg(X._h, None, N, cols.ctypes.data_as(_lib.c_int_p), 2, U.ctypes.data_as(_lib.c_dbl_p), 1,
                                 g0.ctypes.data_as(_lib.c_dbl_p), y.ctypes.data_as(_lib.c_dbl_p), C.c_double(1e-8), 20,
                                 out[0].ctypes.data_as(_lib.c_dbl_p), out[1].ctypes.data_as(_lib.c_dbl_p),
                                 out[2].ctypes.data_as(_lib.c_int_p))

    assert call(U, g0, y01) == 0
    Ub = U.copy()
    Ub[4] = np.nan
    assert call(Ub, g0, y01) == 9
    assert call(U, np.array([np.inf]), y01) == 9
    assert call(U, g0, y2) == 9


def test_prs_pipeline_reference(B, codes, y01):
    """tests/testthat/test-6-PRS.R on the device: snp_autoSVD -> big_univLogReg(covar.train = u) -> p-values against
    pval.rds -> snp_clumping(S = abs(score), size = 250) against clumping.rds -> snp_PRS at thresholds 0, 0.5, .., 5."""
    bim = np.loadtxt(os.path.join(GOLDEN, "example.bim"), dtype=str)
    chrs, pos = bim[:, 0].astype(int), bim[:, 3].astype(float)
    F = B.Bed.from_fbm(codes)
    X = B.Bed(os.path.join(GOLDEN, "example.bed"))
    svd = B.snp_autoSVD(F, chrs, pos)
    keep = np.asarray(svd["subset"])
    Xk = codes[:, keep - 1].astype(np.float64)
    p = Xk.mean(axis=0) / 2
    u = np.linalg.svd((Xk - 2 * p) / np.sqrt(2 * p * (1 - p)), full_matrices=False)[0][:, :10]
    cl = np.load(os.path.join(GOLDEN, "prs_clumping.npz"))
    ref, ok = cl["pval"], ~np.isnan(cl["pval"])
    figures = {}
    for name, U in (("dense", u), ("device", svd["u"])):
        g = B.big_univLogReg(X, y01, covar_train=U)
        pv = g.predict(log10=False)
        assert np.array_equal(ok, ~np.isnan(pv))
        figures[name] = np.mean(np.abs(pv[ok] - ref[ok])) / np.mean(np.abs(ref[ok]))
        if name == "dense":
            gw = g
    print("mean relative difference to pval.rds: dense U %.3g, device U %.3g" % (figures["dense"], figures["device"]))
    assert figures["dense"] < 1e-4
    S = np.abs(gw.score)
    S[np.isnan(S)] = 0
    kept = B.snp_clumping(F, chrs, S=S, size=250, infos_pos=pos)
    assert np.mean(np.isin(kept, cl["keep"])) > 0.98
    prs = B.snp_PRS(X, gw.estim[kept - 1], ind_keep=kept, lpS_keep=-gw.predict()[kept - 1], thr_list=np.arange(11) * 0.5)
    assert np.asarray(prs).shape == (N, 11)
