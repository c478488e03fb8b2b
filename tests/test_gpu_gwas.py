"""big_univLinReg on the device (bsg_univlinreg): byte-identical to the exact model of tests/gwas_ref.py and within the
model's bound of the literal fp64 statistic, on both storage forms, dosages, subsets and multisets, K = 1 / 11 / 21
(two passes), plus the error paths and an SCT-style pipeline."""
import os

import numpy as np
import pytest

from tests import gwas_ref as G

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
N, M = 517, 4542
NM, MM = 200, 500  # example-missing.bed


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


def _same(a, b):
    na, nb = np.isnan(a), np.isnan(b)
    assert np.array_equal(na, nb)
    assert np.array_equal(a[~na].view(np.int64), b[~nb].view(np.int64))


def _check(B, X, vals, na, rows, cols, covar, y, D=1, bound=True):
    """rows / cols 1-based.  Device result == model, bytes; model within its bound of the fp64 statistic."""
    res = B.big_univLinReg(X, y, ind_train=rows, ind_col=cols, covar_train=covar)
    U = B.api.univlinreg_covar_basis(covar, len(rows))
    est, se, parts = G.univlinreg_model(vals, na, np.asarray(rows) - 1, np.asarray(cols) - 1, U, y, D=D, with_parts=True)
    _same(res.estim, est)
    _same(res.std_err, se)
    _same(res.score, est / se)
    assert res.df == len(rows) - U.shape[1] - 1
    if bound and len(cols):
        r0, c0 = np.asarray(rows) - 1, np.asarray(cols) - 1
        e0, s0 = np.empty(len(cols)), np.empty(len(cols))
        for b in range(0, len(cols), 256):  # column blocks keep the dense copies small
            Xd = vals[np.ix_(r0, c0[b:b + 256])].astype(np.float64) / D
            Xd[na[np.ix_(r0, c0[b:b + 256])]] = np.nan
            e0[b:b + 256], s0[b:b + 256], _ = G.univlinreg_fp64(Xd, y, U)
        be, bs = G.model_bound(parts, est, se)
        ok = ~np.isnan(est)
        assert np.array_equal(ok, ~np.isnan(e0))
        assert np.all(np.abs(est - e0)[ok] <= be[ok])
        assert np.all(np.abs(se - s0)[ok] <= bs[ok])
    return res, U


@pytest.mark.parametrize("K", [0, 10, 20])
def test_example_bed(B, codes, K):
    rng = np.random.default_rng(K)
    X = B.Bed(os.path.join(GOLDEN, "example.bed"))
    covar = rng.normal(size=(N, K)) if K else None
    y = rng.normal(size=N) + 0.5 * codes[:, 3].astype(float)
    res, U = _check(B, X, codes, codes == 3, np.arange(1, N + 1), np.arange(1, M + 1), covar, y)
    assert U.shape[1] == K + 1
    # the FBM.code256 twin gives the same bytes
    F = B.Bed.from_fbm(codes)
    r2 = B.big_univLinReg(F, y, covar_train=covar)
    _same(r2.estim, res.estim)
    _same(r2.std_err, res.std_err)


def test_example_missing_subsets(B, codes_missing):
    rng = np.random.default_rng(11)
    X = B.Bed(os.path.join(GOLDEN, "example-missing.bed"))
    F = B.Bed.from_fbm(codes_missing)
    rows = np.concatenate([rng.choice(NM, 150, replace=False), rng.choice(NM, 30)]) + 1
    cols = np.concatenate([rng.choice(MM, 700) + 1, [5, 5, 1, MM]])
    covar = rng.normal(size=(rows.size, 3))
    y = 100 + rng.normal(size=rows.size)
    res, _ = _check(B, X, codes_missing, codes_missing == 3, rows, cols, covar, y)
    assert np.isnan(res.estim).any() and np.isfinite(res.estim).any()
    r2 = B.big_univLinReg(F, y, ind_train=rows, ind_col=cols, covar_train=covar)
    _same(r2.estim, res.estim)
    _same(r2.std_err, res.std_err)


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
    _check(B, F, vals, byt == 255, rows, cols, covar, rng.normal(size=rows.size), D=D)


def test_constant_and_empty(B, codes):
    byt = codes.copy()
    byt[:, 0] = 1
    byt[:, 1] = 0
    F = B.Bed.from_fbm(byt)
    rng = np.random.default_rng(13)
    y = rng.normal(size=N)
    res, _ = _check(B, F, byt, byt == 3, np.arange(1, N + 1), np.arange(1, 40), rng.normal(size=(N, 2)), y)
    assert np.isnan(res.estim[:2]).all() and np.isnan(res.std_err[:2]).all()
    empty = B.big_univLinReg(F, y, ind_col=np.zeros(0, dtype=np.int32))
    assert empty.estim.size == 0 and empty.std_err.size == 0


def test_ld_synthetic_with_pcs(B):
    from tests.synth_ref import synth_matrix_ld

    n, m = 100_000, 2000
    X = B.Bed.synthetic(n, m, seed=77, ld_rho=0.9, ld_block=50)
    vals = synth_matrix_ld(n, m, seed=77, rho=0.9, ld_block=50)
    svd = B.bed_randomSVD(X, k=10)
    pcs = svd["u"] * svd["d"]
    rng = np.random.default_rng(14)
    y = 0.05 * vals[:, 100].astype(float) + pcs[:, 0] / np.std(pcs[:, 0]) + rng.normal(size=n)
    rows = np.sort(rng.choice(n, 80_000, replace=False)) + 1
    cols = rng.permutation(m) + 1
    _check(B, X, vals, vals == 3, rows, cols, pcs[rows - 1], y[rows - 1])


def test_errors(B, codes):
    X = B.Bed(os.path.join(GOLDEN, "example.bed"))
    y = np.random.default_rng(15).normal(size=N)
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        B.big_univLinReg(X, y[:-1])
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        B.big_univLinReg(X, y, covar_train=np.ones((N - 1, 2)))
    y2 = y.copy()
    y2[7] = np.inf
    with pytest.raises(B.BsgError) as e:
        B.big_univLinReg(X, y2)
    assert e.value.code == 9 and "finite" in str(e.value)
    with pytest.raises(B.BsgError) as e:
        B.big_univLinReg(X, y, ind_col=[1, M + 1])
    assert e.value.code == 2
    with pytest.raises(B.BsgError) as e:
        B.big_univLinReg(X, y[:3], ind_train=[1, 2, N + 1])
    assert e.value.code == 2
    code256 = np.full(256, np.nan)
    code256[:3] = [0, 0.1234567, 2]  # not a dosage table: no scale D makes every code an integer byte
    G2 = B.Bed.from_fbm(codes, code256)
    with pytest.raises(B.BsgError) as e:
        B.big_univLinReg(G2, y)
    assert e.value.code == 10


def test_simu_pheno_effects(B, codes):
    # tests/testthat/test-8-simu-pheno.R: the marginal effects of 20 causal SNPs follow their simulated effects
    X = B.Bed(os.path.join(GOLDEN, "example.bed"))
    Xd = codes.astype(float)
    Xd[codes == 3] = np.nan
    mu, sd = np.nanmean(Xd, axis=0), np.nanstd(Xd, axis=0)
    good = np.where(sd > 0.3)[0]
    cors = []
    for it in range(20):
        rng = np.random.default_rng(100 + it)
        s = rng.choice(good, 20, replace=False)
        eff = rng.normal(size=20)
        g = ((np.nan_to_num(Xd[:, s], nan=0.0) - mu[s]) / sd[s]) @ eff
        y = g / np.std(g) * np.sqrt(0.8) + rng.normal(size=N) * np.sqrt(0.2)
        res = B.big_univLinReg(X, y)
        cors.append(np.corrcoef(res.estim[s], eff)[0, 1])
    assert np.median(cors) > 0.15


def test_pipeline_clumping_prs(B, codes):
    X = B.Bed(os.path.join(GOLDEN, "example.bed"))
    F = B.Bed.from_fbm(codes)
    bim = np.loadtxt(os.path.join(GOLDEN, "example.bim"), dtype=str)
    chrs, pos = bim[:, 0].astype(int), bim[:, 3].astype(int)
    rng = np.random.default_rng(16)
    y = rng.normal(size=N) + 0.4 * codes[:, 10].astype(float)
    gw = B.big_univLinReg(X, y)
    U = B.api.univlinreg_covar_basis(None, N)
    est, se = G.univlinreg_model(codes, codes == 3, np.arange(N), np.arange(M), U, y)
    outs = []
    for e, s in ((gw.estim, gw.std_err), (est, se)):
        r = B.MHTest(e, s, e / s, gw.df)
        S = np.abs(r.score)
        S[np.isnan(S)] = 0
        keep = B.snp_clumping(F, chrs, S=S, infos_pos=pos)
        lp = -r.predict()[keep - 1]
        prs = B.snp_PRS(X, e[keep - 1], ind_keep=keep, lpS_keep=lp, thr_list=[0, 1, 2])
        outs.append((keep, np.asarray(prs)))
    assert np.array_equal(outs[0][0], outs[1][0])
    assert np.array_equal(outs[0][1], outs[1][1])
    assert outs[0][0].size > 10
