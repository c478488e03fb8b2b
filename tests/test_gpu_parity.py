"""GPU parity tests: the CUDA path, called through the C ABI (ctypes -> libbsgpu.so), against the CPU oracle
on the same seeded inputs.  They mirror the reference's testthat files for this path (cited per test).

Tolerances: bit-exact for counts / indices / decodes / correlations (integer sums + fp64 epilogue in the
reference's operation order; here on the fixtures, and in tests/test_gpu_cor.py across tile, batch and window edges
against the exact model of tests/cor_ref.py); matvecs agree with the oracle to 1e-11 relative to the vector scale (the
reference's own tests ask for 1.5e-8, north_star for 1e-6).  That tolerance is loose on purpose: it is the
oracle's own rounding (one fp64 add per element) that it allows for.  The engine's accuracy is far tighter --
|error| <= sum_t |g_t| 2^(-e-1) + a few ulps, about 2^-61 of max|v| sum|g| (2^-30 with two vectors per pass) --
and tests/test_gpu_fixedpoint.py holds every X.y / Xt.y path to the exact bytes of tests/fixedpoint_ref.py.
"""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def B():
    import bigsnpr_b200 as b

    from bigsnpr_b200 import build

    build.build()
    return b


@pytest.fixture(scope="module")
def gbed(B):
    return B.Bed(os.path.join(GOLDEN, "example.bed"))


@pytest.fixture(scope="module")
def gbed_na(B):
    return B.Bed(os.path.join(GOLDEN, "example-missing.bed"))


def _close(got, want, scale=None, tol=1e-11):
    got, want = np.asarray(got), np.asarray(want)
    s = np.max(np.abs(want)) if scale is None else scale
    s = np.maximum(np.asarray(s, dtype=float), 1e-300)
    assert got.shape == want.shape
    err = float(np.max(np.abs(got - want) / s)) if got.size else 0.0
    assert err < tol, err


# ---------------------------------------------------------------------------------------------------
def test_staging_roundtrip_and_validation(B, gbed, gbed_na, obed, obed_na, tmp_path):
    # tests/testthat/test-1-readBed.R (decode) + src/bed-acc-xptr.cpp:21-34 (errors)
    assert repr(gbed) == "A 'bed' object with 517 samples and 4542 variants."
    assert len(gbed) == 517 * 4542
    for g, o in ((gbed, obed), (gbed_na, obed_na)):
        packed = g.export_packed()
        nb = (o.nrow + 3) // 4
        want = o.bytes.reshape(o.ncol, nb).copy()
        if o.nrow % 4:
            want[:, -1] &= (1 << (2 * (o.nrow % 4))) - 1  # pad slots are exported as 00
        assert np.array_equal(packed.reshape(o.ncol, nb), want)
    assert not gbed.has_na and gbed_na.has_na
    good = os.path.join(GOLDEN, "example.bed")
    with pytest.raises(B.BsgError, match="n or p does not match the dimensions of the file."):
        B.Bed(good, 517, 4541)
    raw = bytearray(open(good, "rb").read())
    bad = tmp_path / "bad.bed"
    r2 = bytearray(raw); r2[1] = 0
    bad.write_bytes(r2)
    with pytest.raises(B.BsgError, match="File is not a binary PED file."):
        B.Bed(str(bad), 517, 4542)
    r3 = bytearray(raw); r3[2] = 0
    bad.write_bytes(r3)
    with pytest.raises(B.BsgError, match="Variant-major is the only mode supported."):
        B.Bed(str(bad), 517, 4542)
    with pytest.raises(B.BsgError, match="out of bounds"):
        B.bed_counts(gbed, ind_row=[1, 518])
    # column shard == same columns of the whole file
    shard = B.Bed(good, col_range=(1000, 1500))
    assert shard.shape == (517, 500)
    assert np.array_equal(B.bed_counts(shard), B.bed_counts(gbed, ind_col=np.arange(1001, 1501)))


def test_read_bed_accessor(B, gbed_na, oracle, obed_na, rng):
    # tests/testthat/test-1-readBed.R:71-87,91-115: indices with replacement, bed[i, j]
    ir = rng.integers(1, obed_na.nrow + 1, 150)
    ic = rng.integers(1, obed_na.ncol + 1, 170)
    assert np.array_equal(B.read_bed(gbed_na, ir, ic), oracle.read_bed(obed_na, ir, ic))
    assert np.array_equal(gbed_na[ir, ic], oracle.read_bed(obed_na, ir, ic))
    c, s = rng.normal(size=ic.size), rng.uniform(0.1, 1, size=ic.size)
    assert np.array_equal(B.read_bed_scaled(gbed_na, ir, ic, c, s), oracle.read_bed_scaled(obed_na, ir, ic, c, s))
    full = gbed_na[:, :]
    assert full.shape == (200, 500) and int((full == B.NA_INTEGER).sum()) == 2788


def test_counts_maf_scaling_bit_exact(B, gbed, gbed_na, oracle, obed, obed_na, rng):
    # tests/testthat/test-2-bed-clumping-SVD.R:95-136: identical() to the reference counts
    for g, o in ((gbed, obed), (gbed_na, obed_na)):
        ir = rng.choice(o.nrow, min(300, o.nrow - 10), replace=False) + 1
        ic = rng.choice(o.ncol, min(4000, o.ncol - 10), replace=False) + 1
        for byrow in (False, True):
            assert np.array_equal(B.bed_counts(g, ir, ic, byrow=byrow), oracle.bed_counts(o, ir, ic, byrow=byrow))
            assert np.array_equal(B.bed_counts(g, byrow=byrow), oracle.bed_counts(o, byrow=byrow))
        assert np.array_equal(B.bed_counts(g, ind_col=ic), oracle.bed_counts(o, ind_col=ic))
        # multiset rows (sample(replace = TRUE))
        irr = rng.integers(1, o.nrow + 1, 333)
        assert np.array_equal(B.bed_counts(g, irr, ic), oracle.bed_counts(o, irr, ic))
        assert np.array_equal(B.bed_counts(g, irr, ic, byrow=True), oracle.bed_counts(o, irr, ic, byrow=True))
        for a, b in ((ir, ic), (o.rows_along(), o.cols_along())):
            st, so = B.bed_colstats(g, a, b), oracle.bed_colstats(o, a, b)
            for k in ("sumX", "denoX", "nb_nona_col"):
                assert np.array_equal(st[k], so[k], equal_nan=True)
            sc, sco = B.bed_scaleBinom(g, a, b), oracle.bed_scaleBinom(o, a, b)
            assert np.array_equal(sc["center"], sco["center"], equal_nan=True)
            assert np.array_equal(sc["scale"], sco["scale"], equal_nan=True)
            mf, mfo = B.bed_MAF(g, a, b), oracle.bed_MAF(o, a, b)
            for k in mf:
                assert np.array_equal(mf[k], mfo[k], equal_nan=True)
        assert np.array_equal(B.bed_scaleBinom(g, ir, ic)["center"], 2 * B.bed_MAF(g, ir, ic)["af"])


def test_prodvec_equality_with_dense(B, gbed_na, oracle, obed_na, rng):
    # tests/testthat/test-5-bed-prod-vec.R:18-41: 20 random subsets, default and random center / scale
    N, M = obed_na.nrow, obed_na.ncol
    for rep in range(20):
        n, m = int(rng.integers(1, N + 1)), int(rng.integers(1, M + 1))
        ir = rng.choice(N, n, replace=False) + 1
        ic = rng.choice(M, m, replace=False) + 1
        y_col, y_row = rng.normal(size=m), rng.normal(size=n)
        X = oracle.read_bed_scaled(obed_na, ir, ic, np.zeros(m), np.ones(m))
        sa, sb = np.abs(X) @ np.abs(y_col), np.abs(X.T) @ np.abs(y_row)
        _close(B.bed_prodVec(gbed_na, y_col, ir, ic), X @ y_col, scale=sa + 1e-6 * sa.max() + 1e-300)
        _close(B.bed_cprodVec(gbed_na, y_row, ir, ic), X.T @ y_row, scale=sb + 1e-6 * sb.max() + 1e-300)
        c, s = rng.normal(size=m), rng.uniform(size=m)
        _close(B.bed_prodVec(gbed_na, y_col, ir, ic, c, s), oracle.bed_prodVec(obed_na, y_col, ir, ic, c, s),
               scale=np.max(np.abs(y_col / s)) * m * 3)
        _close(B.bed_cprodVec(gbed_na, y_row, ir, ic, c, s), oracle.bed_cprodVec(obed_na, y_row, ir, ic, c, s),
               scale=np.max(np.abs(y_row)) * n * 3 / np.min(s))


def test_prodvec_dimension_errors(B, gbed_na, rng):
    # tests/testthat/test-5-bed-prod-vec.R:43-50
    ir = rng.choice(200, 21, replace=False) + 1
    ic = rng.choice(500, 11, replace=False) + 1
    with pytest.raises(ValueError, match=B.ERROR_DIM):
        B.bed_prodVec(gbed_na, rng.normal(size=21), ir, ic)
    with pytest.raises(ValueError, match=B.ERROR_DIM):
        B.bed_cprodVec(gbed_na, rng.normal(size=11), ir, ic)
    with pytest.raises(ValueError, match=B.ERROR_DIM):
        B.bed_prodVec(gbed_na, rng.normal(size=11), ir, ic, center=np.zeros(3), scale=np.ones(3))


def test_prodvec_multiset_indices(B, gbed, gbed_na, oracle, obed, obed_na, rng):
    # tests/testthat/test-7-OpenMP.R:27-63: indices with replacement, unsorted; ncores accepted
    for g, o in ((gbed, obed), (gbed_na, obed_na)):
        ir = rng.integers(1, o.nrow + 1, o.nrow)
        ic = rng.integers(1, o.ncol + 1, min(o.ncol, 3000))
        c, s = rng.normal(size=ic.size), rng.uniform(0.2, 1.5, size=ic.size)
        y_col, y_row = rng.normal(size=ic.size), rng.normal(size=ir.size)
        _close(B.bed_prodVec(g, y_col, ir, ic, c, s, ncores=2), oracle.bed_prodVec(o, y_col, ir, ic, c, s),
               scale=np.max(np.abs(y_col / s)) * ic.size)
        _close(B.bed_cprodVec(g, y_row, ir, ic, c, s, ncores=2), oracle.bed_cprodVec(o, y_row, ir, ic, c, s),
               scale=np.max(np.abs(y_row)) * ir.size / np.min(s))


def test_single_copy_kernel_matches_oracle(B, oracle, obed, obed_na, rng):
    """X.y from the SNP-major copy alone (k_pmvT, handles opened without the sample-major copy) against the oracle
    and against the two-copy path: subsets, multisets, scaling, missing values, non-finite input, projections."""
    for name, o in (("example-missing.bed", obed_na), ("example.bed", obed)):
        f = os.path.join(GOLDEN, name)
        g2 = B.Bed(f, layouts=B.LAYOUT_SNP_MAJOR | B.LAYOUT_SAMPLE_MAJOR)
        g1 = B.Bed(f, layouts=B.LAYOUT_SNP_MAJOR)
        assert g2.layouts == 3 and g1.layouts == 1
        N, M = o.nrow, o.ncol
        cases = [(np.arange(1, N + 1), np.arange(1, M + 1)),
                 (rng.choice(N, N // 3, replace=False) + 1, rng.choice(M, M // 2, replace=False) + 1),
                 (rng.integers(1, N + 1, N), rng.integers(1, M + 1, min(M, 1500))),
                 (np.array([N]), np.array([M, 1, M]))]
        for ir, ic in cases:
            m = ic.size
            y = rng.normal(size=m)
            c, s = rng.normal(size=m), rng.uniform(0.2, 1.5, size=m)
            for cs in ((None, None), (c, s)):
                a = B.bed_prodVec(g1, y, ir, ic, *cs)
                b = B.bed_prodVec(g2, y, ir, ic, *cs)
                want = oracle.bed_prodVec(o, y, ir, ic, *cs)
                sc = np.max(np.abs(y / (s if cs[0] is not None else 1.0))) * m * 3
                _close(a, want, scale=sc)
                _close(a, b, scale=sc, tol=1e-13)
        sc = oracle.bed_scaleBinom(o)
        ir, ic = np.arange(1, N + 1), np.arange(1, M + 1)
        V = rng.normal(size=(M, 3))
        XV, rss = B.prod_and_rowSumsSq(g1, ir, ic, sc["center"], sc["scale"], V)
        XVo, rsso = oracle.prod_and_rowSumsSq(o, ir, ic, sc["center"], sc["scale"], V)
        _close(XV, XVo, tol=1e-8)  # two columns of V per pass: 30-bit fixed point per vector (bsg_pmv.cu k_quantT<2>)
        _close(rss, rsso, tol=1e-12)
        y = rng.normal(size=M)
        y[5] = np.nan
        with np.errstate(all="ignore"):
            a, want = B.bed_prodVec(g1, y), oracle.bed_prodVec(o, y)
        assert np.array_equal(np.isnan(a), np.isnan(want))
        svd1, svd2 = B.bed_randomSVD(g1, k=4), B.bed_randomSVD(g2, k=4)
        np.testing.assert_allclose(svd1["d"], svd2["d"], rtol=1e-9)
    # the same handle through both kernels (process-wide switch of the C ABI)
    g = B.Bed.synthetic(3000, 7001, seed=11, na_rate=0.02)
    y = rng.normal(size=7001)
    sc = B.bed_scaleBinom(g)
    a = B.bed_prodVec(g, y, center=sc["center"], scale=sc["scale"])
    B._lib.check(B._lib.lib().bsg_set_prodvec_path(1))
    try:
        b = B.bed_prodVec(g, y, center=sc["center"], scale=sc["scale"])
    finally:
        B._lib.check(B._lib.lib().bsg_set_prodvec_path(0))
    _close(a, b, scale=np.max(np.abs(y / sc["scale"])) * 7001, tol=1e-13)


def test_nonfinite_inputs_follow_reference(B, gbed_na, oracle, obed_na, rng):
    """Inf / NaN in the vector or a zero scale propagate like the reference's table arithmetic (src/bed-acc.h:98-111)."""
    y = rng.normal(size=500)
    y[7] = np.inf
    with np.errstate(all="ignore"):
        want = oracle.bed_prodVec(obed_na, y)
        got = B.bed_prodVec(gbed_na, y)
        assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(np.isinf(got), np.isinf(want))
        s = np.ones(500); s[3] = 0.0
        yr = rng.normal(size=200)
        want = oracle.bed_cprodVec(obed_na, yr, center=np.full(500, 0.5), scale=s)
        got = B.bed_cprodVec(gbed_na, yr, center=np.full(500, 0.5), scale=s)
        ok = np.isfinite(want)
        assert np.array_equal(np.isfinite(got), ok)
        _close(got[ok], want[ok], scale=np.max(np.abs(yr)) * 200)


def test_cor_matches_oracle_and_plink(B, gbed, oracle, obed, golden_dir):
    # tests/testthat/test-2-corr.R:14-58: r^2 vs PLINK (1e-6) with the same sparsity; bit-exact vs the oracle
    thr = np.full(obed.nrow, np.sqrt(0.2))
    pos = np.arange(1, obed.ncol + 1, dtype=float)
    rows = [l.split() for l in open(os.path.join(golden_dir, "example.ld"))][1:]
    a = np.array([int(r[2][3:]) for r in rows]); b = np.array([int(r[5][3:]) for r in rows])
    r2 = np.array([float(r[6]) for r in rows])
    for size in (13, 200):
        p, i, x = B.corMat(gbed, gbed.rows_along(), gbed.cols_along(), size, thr, pos, fill_diag=False)
        po, io, xo = oracle.corMat(obed, obed.rows_along(), obed.cols_along(), size, thr, pos, fill_diag=False,
                                   ncores=oracle.max_threads())
        assert np.array_equal(p, po) and np.array_equal(i, io) and np.array_equal(x, xo)
        j = np.repeat(np.arange(obed.ncol), np.diff(p))
        keep = (b - a) <= size
        got = {(ii, jj): v * v for ii, jj, v in zip(i.tolist(), j.tolist(), x.tolist())}
        want = {(ii, jj): v for ii, jj, v in zip(a[keep].tolist(), b[keep].tolist(), r2[keep].tolist())}
        assert set(got) == set(want) and max(abs(got[k] - want[k]) for k in want) < 1e-6


def test_cor_with_missing_alpha_and_fbm(B, oracle, rng, tmp_path):
    # tests/testthat/test-2-corr.R:62-159 ; test-2-ld-scores.R:15-64
    N, M = 500, 100
    G = rng.integers(0, 4, size=(N, M))
    ofbm = oracle.OracleFBM(G.astype(np.uint8))
    path = oracle.write_bed(str(tmp_path / "fake.bed"), G)
    gb, gf = B.Bed(path), B.Bed.from_fbm(G.astype(np.uint8))
    ir = rng.choice(N, N // 2, replace=False) + 1
    ic = np.sort(rng.choice(M, M // 2, replace=False)) + 1
    for kw in (dict(size=30), dict(size=30, alpha=0.07, fill_diag=False), dict(size=5, thr_r2=0.02),
               dict(size=5e3, infos_pos=1e6 * np.arange(1, ic.size + 1), alpha=0.3)):
        po, io, xo = oracle.cor0(ofbm, ir, ic, **kw)
        for g in (gb, gf):
            p, i, x = B.bed_cor(g, ir, ic, **kw)
            assert np.array_equal(p, po) and np.array_equal(i, io) and np.array_equal(x, xo, equal_nan=True)
    p6, i6, x6 = B.bed_cor(gb, ir, ic, size=5e-3, infos_pos=1000.0 * np.arange(1, ic.size + 1), fill_diag=False)
    assert x6.size == 0
    for size in (20, 37):
        ld = B.bed_ld_scores(gf, ir, ic, size=size)
        np.testing.assert_allclose(ld, oracle.ld0(ofbm, ir, ic, size=size), rtol=1e-12)
        p, i, x = B.bed_cor(gb, ir, ic, size=size)
        m = ic.size
        sym = np.zeros((m, m)); sym[i, np.repeat(np.arange(m), np.diff(p))] = x
        sym = sym + sym.T - np.diag(np.diag(sym))
        np.testing.assert_allclose(ld, (sym ** 2).sum(0), rtol=1e-12)  # ld == colSums(corr^2)
    assert np.all(B.bed_ld_scores(gb, size=0.5) == 1.0)
    # zero variance -> NaN + warning (tests/testthat/test-2-corr.R:163-171)
    G2 = rng.integers(0, 3, size=(10, 10)); G2[:, 0] = 0
    g2 = B.Bed.from_fbm(G2.astype(np.uint8))
    with pytest.warns(UserWarning, match="NA or NaN values"):
        p, i, x = B.snp_cor(g2)
    po, io, xo = oracle.cor0(oracle.OracleFBM(G2.astype(np.uint8)))
    assert np.array_equal(i, io) and np.array_equal(x, xo, equal_nan=True)
    # a code table that is not 0 / 1 / 2 / NA (dosages) stages a generic handle: the packed engine refuses it by name
    gd = B.Bed.from_fbm(G2.astype(np.uint8), code256=np.linspace(0, 2, 256))
    with pytest.raises(B.BsgError, match="needs hard calls"):
        B.bed_prodVec(gd, np.ones(10))
    gd.close()


def test_synthetic_matches_numpy_mirror_and_oracle(B, oracle, rng):
    """Device generator == NumPy mirror bit for bit; matvecs on a mid-size synthetic matrix vs the oracle."""
    from tests.synth_ref import synth_matrix

    n, m = 3001, 2203
    for na_rate in (0.0, 0.02):
        g = B.Bed.synthetic(n, m, seed=11, na_rate=na_rate)
        G = synth_matrix(n, m, seed=11, na_rate=na_rate)
        o = oracle.OracleBed.from_packed(g.export_packed(), n, m)
        assert np.array_equal(oracle.decode_dense(o), G)
        assert g.has_na == (na_rate > 0)
        sc = B.bed_scaleBinom(g)
        y_col, y_row = rng.normal(size=m), rng.normal(size=n)
        nt = oracle.max_threads()
        _close(B.bed_prodVec(g, y_col, center=sc["center"], scale=sc["scale"]),
               oracle.bed_prodVec(o, y_col, center=sc["center"], scale=sc["scale"], ncores=nt),
               scale=np.max(np.abs(y_col / sc["scale"])) * m)
        _close(B.bed_cprodVec(g, y_row, center=sc["center"], scale=sc["scale"]),
               oracle.bed_cprodVec(o, y_row, center=sc["center"], scale=sc["scale"], ncores=nt),
               scale=np.max(np.abs(y_row)) * n / np.min(sc["scale"]))
        shard = B.Bed.synthetic(n, 500, seed=11, na_rate=na_rate, col_offset=1000)
        assert np.array_equal(B.bed_counts(shard), B.bed_counts(g, ind_col=np.arange(1001, 1501)))


def test_full_size_properties(B):
    """BASELINE configs[1] shape (50,000 x 500,000): size-independent properties of the two products.

    * column sums: t(X) 1 against the exact popcount statistics (sumX - center * nb_nona) / scale;
    * adjoint identity: y^T (X x) == (X^T y)^T x;
    * linearity in the vector.
    """
    import torch

    free, _ = torch.cuda.mem_get_info()
    n, m = (50000, 500000) if free > 40e9 else (20000, 50000)
    g = B.Bed.synthetic(n, m, seed=20250926, na_rate=0.01)
    st = B.bed_colstats(g)
    sc = B.bed_scaleBinom(g)
    v = B.View(g, center=sc["center"], scale=sc["scale"])
    ones = np.ones(n)
    colsum = v.cprodvec(ones)
    want = (st["sumX"] - sc["center"] * st["nb_nona_col"]) / sc["scale"]
    _close(colsum, want, scale=n / np.min(sc["scale"]), tol=1e-12)
    rng = np.random.default_rng(1)
    x, y = rng.normal(size=m), rng.normal(size=n)
    Ax, Aty = v.prodvec(x), v.cprodvec(y)
    lhs, rhs = float(y @ Ax), float(Aty @ x)
    assert abs(lhs - rhs) <= 1e-10 * (np.linalg.norm(y) * np.linalg.norm(Ax))
    x2 = rng.normal(size=m)
    _close(v.prodvec(x + 2 * x2), Ax + 2 * v.prodvec(x2), tol=1e-11, scale=np.max(np.abs(Ax)) * 10)


def test_randomsvd_and_grm(B, gbed, gbed_na, oracle, obed, obed_na):
    # tests/testthat/test-2-bed-clumping-SVD.R:41-57,72-79: singular values vs the dense decomposition and vs
    # sqrt(eigen(K)); north_star tolerance 1e-6 relative (the reference's own test: 1.5e-8)
    for g, o, ic in ((gbed_na, obed_na, np.arange(1, 501, 2)), (gbed, obed, np.arange(1, 4543, 3))):
        ic = ic.astype(np.int32)
        svd = B.bed_randomSVD(g, ind_col=ic, k=10)
        want = oracle.bed_randomSVD(o, ind_col=ic, k=10)
        np.testing.assert_allclose(svd["d"], want["d"], rtol=1e-7)
        assert np.array_equal(svd["center"], want["center"]) and np.array_equal(svd["scale"], want["scale"])
        cu = np.abs(np.sum(svd["u"] * want["u"], axis=0))
        cv = np.abs(np.sum(svd["v"] * want["v"], axis=0))
        assert cu.min() > 1 - 1e-6 and cv.min() > 1 - 1e-6
        np.testing.assert_allclose(np.linalg.norm(svd["u"], axis=0), 1.0, rtol=1e-10)
        K, c, s = B.bed_tcrossprodSelf(g, ind_col=ic)
        Ko, co, so = oracle.bed_tcrossprodSelf(o, ind_col=ic, block_size=200)
        # weights carry 28 bits (4 base-128 digit slices, exact integer Gram per slice): |dK| <= 2^-28 * wmax * sum a_i a_j
        assert np.max(np.abs(K - Ko)) < 1e-8 * np.max(np.abs(Ko))
        assert np.array_equal(c, co) and np.array_equal(s, so)
        ev = np.linalg.eigvalsh(K)[::-1][:10]
        np.testing.assert_allclose(np.sqrt(ev), svd["d"], rtol=1e-7)
    if not gbed.has_na:  # colMeans(u) == 0 without missing values (:52)
        svd = B.bed_randomSVD(gbed, k=5)
        assert np.max(np.abs(svd["u"].mean(0))) < 1.5e-8  # expect_equal tolerance of the reference, tol = 1e-4
    with pytest.raises(ValueError, match="can't be `NULL`"):
        B.bed_randomSVD(gbed, ind_row=None)


def test_clumping_identical_to_oracle(B, gbed, gbed_na, oracle, obed, obed_na, rng):
    # tests/testthat/test-2-bed-clumping-SVD.R:28-49,62-70,83: kept indices identical; window rescaling invariance;
    # `exclude`; ncores accepted.  (The clumping.rds golden: test_clumping_against_reference_rds_golden below.)
    for g, o in ((gbed, obed), (gbed_na, obed_na)):
        want = oracle.bed_clumping(o)
        got = B.bed_clumping(g, ncores=2)
        assert np.array_equal(got, want)
        for kw in (dict(thr_r2=0.05), dict(thr_r2=0.5, size=50), dict(exclude=np.arange(1, 101))):
            assert np.array_equal(B.bed_clumping(g, **kw), oracle.bed_clumping(o, **kw))
        S = rng.uniform(size=o.ncol)
        assert np.array_equal(B.bed_clumping(g, S=S), oracle.bed_clumping(o, S=S))
        ir = rng.choice(o.nrow, o.nrow // 2, replace=False) + 1
        assert np.array_equal(B.bed_clumping(g, ind_row=ir), oracle.bed_clumping(o, ind_row=ir))
        chrom, pos = g.map["chromosome"], g.map["physical.pos"]
        k2 = B.bed_clumping(g, infos_chr=chrom, infos_pos=pos * 1e6, size=500 * 1e6)
        assert np.array_equal(k2, want)
    assert B.bed_clumping(gbed, exclude=np.arange(1, 101)).min() > 100
    with pytest.raises(ValueError, match="can't be `NULL`"):
        B.bed_clumping(gbed, ind_row=None)


def test_scaling_reuse_shortcut_is_opt_in_and_tracks_changes(B, gbed, oracle, obed, rng):
    # include/bsgpu.h: the 9-argument calls upload center / scale every time (like the reference re-reads them); with
    # bsg_set_scaling_reuse(1) an unchanged scaling (same address, length and sampled values) is not uploaded again.
    from bigsnpr_b200 import _lib

    L = _lib.lib()
    m = obed.ncol
    y = rng.normal(size=m)
    sc = oracle.bed_scaleBinom(obed)
    c, s = sc["center"].copy(), sc["scale"].copy()
    want = oracle.bed_prodVec(obed, y, center=c, scale=s)
    tol = 1e-12 * np.max(np.abs(want))
    for mode in (0, 1):
        _lib.check(L.bsg_set_scaling_reuse(mode))
        try:
            a1 = B.bed_prodVec(gbed, y, center=c, scale=s)
            a2 = B.bed_prodVec(gbed, y, center=c, scale=s)          # same vectors again
            assert np.array_equal(a1, a2) and np.max(np.abs(a1 - want)) < tol
            s2 = 2.0 * s                                            # a different vector (new address)
            assert np.max(np.abs(B.bed_prodVec(gbed, y, center=c, scale=s2) - want / 2)) < tol
            s *= 4.0                                                # the SAME buffer rewritten in place
            assert np.max(np.abs(B.bed_prodVec(gbed, y, center=c, scale=s) - want / 4)) < tol
            s /= 4.0
            if mode == 0:                                           # default: even a one-element edit in place is seen
                j = 1234                                            # (not one of the 2,048 + 1 sampled positions of 4,542)
                assert j not in set((np.arange(2048) * m // 2048).tolist()) | {m - 1}
                keep = s[j]
                s[j] = 7.0 * keep
                got = B.bed_prodVec(gbed, y, center=c, scale=s)
                assert np.max(np.abs(got - oracle.bed_prodVec(obed, y, center=c, scale=s))) < tol
                s[j] = keep
                B.bed_prodVec(gbed, y, center=c, scale=s)           # uploads the restored vector (mode 1 would not notice)
        finally:
            _lib.check(L.bsg_set_scaling_reuse(0))


def test_randomSVD_degenerate_scaling_fails_loudly(B, gbed):
    # ADVICE r1 (low): the device-vector products turn a zero scale into an all-NaN result; the SVD built on them must not
    # iterate on NaNs and hand back garbage -- it reports the degenerate operator (RSpectra fails on it as well)
    def zero_scale(obj, ind_row=None, ind_col=None, **kw):
        m = len(ind_col)
        return {"center": np.zeros(m), "scale": np.r_[0.0, np.ones(m - 1)]}

    with pytest.raises(B.BsgError, match="non-finite"):
        B.bed_randomSVD(gbed, fun_scaling=zero_scale, k=3)
    # and the handle is still usable afterwards
    assert B.bed_randomSVD(gbed, k=2)["d"].shape == (2,)


def test_clumping_against_reference_rds_golden(B, gbed, oracle, obed, golden_dir):
    # tests/testthat/test-6-PRS.R:25-31: the reference's stored snp_clumping result (testdata/clumping.rds) with the priority
    # order recovered from testdata/pval.rds (p-value = decreasing function of abs(gwas$score); only the order of S matters).
    # Fixture: tests/golden/prs_clumping.npz, made from the two RDS files by tests/golden/make_rds_golden.py.  The bar is the
    # reference's own (> 98 % of the kept variants are in the stored set); against the oracle the indices are identical.
    import os

    gold = np.load(os.path.join(golden_dir, "prs_clumping.npz"))
    pval, keep2 = gold["pval"], gold["keep"]
    chrom, pos = oracle.read_bim(obed.bedfile)
    G = oracle.read_bed(obed, obed.rows_along(), obed.cols_along(), na_val=3).astype(np.uint8)
    gf, of = B.Bed.from_fbm(G), oracle.OracleFBM(G)
    keep = B.snp_clumping(gf, chrom, S=-pval, size=250, infos_pos=pos)
    assert np.mean(np.isin(keep, keep2)) > 0.98
    assert np.array_equal(keep, oracle.snp_clumping(of, chrom, S=-pval, size=250, infos_pos=pos))
    assert np.array_equal(B.bed_clumping(gbed, S=-pval, size=250), keep)
    gf.close()


def test_prod_and_rowSumsSq_and_projection(B, gbed, gbed_na, oracle, obed, obed_na, rng):
    # src/bed-fun.cpp:103-133 against the oracle; tests/testthat/test-2-pca-project.R:8-22,43-55:
    # simple_proj[ind.row, ] == predict(obj.svd) (1e-4), dimension and NULL errors
    for g, o in ((gbed_na, obed_na), (gbed, obed)):
        n, m = o.nrow, o.ncol
        sc = oracle.bed_scaleBinom(o)
        for ir, ic in ((np.arange(1, n + 1), np.arange(1, m + 1)),
                       (rng.choice(n, n // 2, replace=False) + 1, rng.choice(m, m // 3, replace=False) + 1),
                       (rng.integers(1, n + 1, size=37), rng.integers(1, m + 1, size=211))):  # multisets
            c, s = sc["center"][ic - 1], sc["scale"][ic - 1]
            V = rng.normal(size=(ic.size, 4))
            XV, rss = B.prod_and_rowSumsSq(g, ir, ic, c, s, V)
            XVo, rsso = oracle.prod_and_rowSumsSq(o, ir, ic, c, s, V)
            _close(XV, XVo, tol=1e-8)  # two columns of V per pass: 30-bit fixed point per vector (bsg_pmv.cu k_quantT<2>)
            _close(rss, rsso, tol=1e-12)
        # identity scaling and a vector V
        ic = np.arange(1, m + 1)
        XV, rss = B.prod_and_rowSumsSq(g, np.arange(1, n + 1), ic, np.zeros(m), np.ones(m), rng.normal(size=m))
        dense = oracle.read_bed_scaled(o, np.arange(1, n + 1), ic, np.zeros(m), np.ones(m))
        assert np.array_equal(rss, (dense ** 2).sum(1))  # integer-valued: exact
    # handle without the sample-major copy: accessor kernels, same numbers
    g1 = B.Bed(os.path.join(GOLDEN, "example-missing.bed"), layouts=B.LAYOUT_SNP_MAJOR)
    sc = oracle.bed_scaleBinom(obed_na)
    ir, ic = np.arange(1, obed_na.nrow + 1), np.arange(1, obed_na.ncol + 1)
    V = rng.normal(size=(ic.size, 2))
    XV, rss = B.prod_and_rowSumsSq(g1, ir, ic, sc["center"], sc["scale"], V)
    XVo, rsso = oracle.prod_and_rowSumsSq(obed_na, ir, ic, sc["center"], sc["scale"], V)
    _close(XV, XVo, tol=1e-8)  # two columns of V per pass: 30-bit fixed point per vector (bsg_pmv.cu k_quantT<2>)
    _close(rss, rsso, tol=1e-12)
    # zero scale: the reference's Inf / NaN pattern (table arithmetic), not a crash
    s0 = sc["scale"].copy(); s0[3] = 0.0
    with np.errstate(all="ignore"):
        XV, rss = B.prod_and_rowSumsSq(gbed_na, ir, ic, sc["center"], s0, V)
        XVo, rsso = oracle.prod_and_rowSumsSq(obed_na, ir, ic, sc["center"], s0, V)
    assert np.array_equal(np.isfinite(rss), np.isfinite(rsso)) and np.array_equal(np.isfinite(XV), np.isfinite(XVo))
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        B.prod_and_rowSumsSq(gbed_na, ir, ic, sc["center"][1:], sc["scale"][1:], V)
    # projection of the training samples reproduces the PC scores u d
    ind_row = np.sort(rng.choice(obed.nrow, 400, replace=False)) + 1
    svd = B.bed_randomSVD(gbed, ind_row=ind_row, k=6)
    with pytest.raises(ValueError, match="'ind.col' can't be `NULL`."):
        B.bed_projectSelfPCA(svd, gbed, ind_row=ind_row)
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        B.bed_projectSelfPCA(svd, gbed, ind_row=ind_row, ind_col=np.arange(1, 6))
    proj = B.bed_projectSelfPCA(svd, gbed, ind_row=np.arange(1, obed.nrow + 1), ind_col=np.arange(1, obed.ncol + 1))
    np.testing.assert_allclose(proj["simple_proj"][ind_row - 1], svd["u"] * svd["d"], rtol=0, atol=1e-4 * svd["d"][0])
    assert proj["X_norm"].shape == (obed.nrow,) and np.all(proj["X_norm"] > 0)


def test_multLinReg_pcadapt(B, gbed, gbed_na, oracle, obed, obed_na, rng):
    # src/multLinReg.cpp:8-88 against the oracle (bed and FBM.code256 handles), R/pcadapt.R:3-27
    for g, o in ((gbed_na, obed_na), (gbed, obed)):
        n, m = o.nrow, o.ncol
        for ir, ic, K in ((np.arange(1, n + 1), np.arange(1, m + 1), 3),
                          (rng.choice(n, n // 2, replace=False) + 1, rng.choice(m, m // 4, replace=False) + 1, 1),
                          (rng.integers(1, n + 1, size=150), rng.integers(1, m + 1, size=97), 2)):
            U = np.linalg.qr(rng.normal(size=(ir.size, K)))[0]
            t = B.multLinReg(g, ir, ic, U)
            to = oracle.multLinReg(o, ir, ic, U, ncores=2)
            assert np.array_equal(np.isnan(t), np.isnan(to))
            ok = ~np.isnan(to)
            # K >= 2: two columns of U per pass, 30-bit fixed point each (bsg_pmv.cu view_planes_pair_dev); K = 1: 61 bits
            assert np.max(np.abs(t[ok] - to[ok]) / (1.0 + np.abs(to[ok]))) < (1e-7 if K >= 2 else 1e-9)
    # FBM.code256 handle == bed handle; constant column -> NA (deno == 0)
    G = rng.integers(0, 4, size=(120, 40)).astype(np.uint8)
    G[:, 5] = 1
    G[:119, 6] = 3  # one genotype present: nona < 2 -> NA
    G[:118, 7] = 3  # two present: a perfect fit, deno is 0 up to rounding -> NA or 0, not comparable
    gf, of = B.Bed.from_fbm(G), oracle.OracleFBM(G)
    ir, ic = np.arange(1, 121), np.arange(1, 41)
    U = np.linalg.qr(rng.normal(size=(120, 2)))[0]
    t, to = B.multLinReg(gf, ir, ic, U), oracle.multLinReg(of, ir, ic, U)
    assert np.isnan(to[5]).all() and np.isnan(to[6]).all() and np.isnan(t[5]).all() and np.isnan(t[6]).all()
    assert np.all(np.isnan(t[7]) | (np.abs(t[7]) < 1e-6))
    t[7] = to[7] = np.nan
    assert np.array_equal(np.isnan(t), np.isnan(to))
    ok = ~np.isnan(to)
    assert np.max(np.abs(t[ok] - to[ok]) / (1.0 + np.abs(to[ok]))) < 1e-7
    res = B.bed_pcadapt(gbed, U_row=np.linalg.qr(rng.normal(size=(obed.nrow, 1)))[0][:, 0])
    assert res["tscores"].shape == (obed.ncol, 1) and res["score"].shape == (obed.ncol,)
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        B.bed_pcadapt(gbed, U_row=np.ones((10, 2)))


def test_bed_fbm_conversions(B, gbed, gbed_na, oracle, obed, obed_na, rng, tmp_path):
    # tests/testthat/test-1-readBed.R:91-115 (snp_readBed2 == the accessor), test-1-writeBed.R (write -> read round
    # trip); bytes against the oracle's restatement of src/write-plink.cpp:29-47
    for g, o in ((gbed_na, obed_na), (gbed, obed)):
        n, m = o.nrow, o.ncol
        for ir, ic in ((np.arange(1, n + 1), np.arange(1, m + 1)),
                       (rng.choice(n, n // 2 + 1, replace=False) + 1, rng.choice(m, m // 3, replace=False) + 1),
                       (rng.integers(1, n + 1, size=203), rng.integers(1, m + 1, size=77))):
            G = B.readbina2(g, ir, ic)
            want = oracle.read_bed(o, ir, ic, na_val=3).astype(np.uint8)
            assert G.dtype == np.uint8 and np.array_equal(G, want)
            path = str(tmp_path / ("sub_%d_%d.bed" % (ir.size, ic.size)))
            if os.path.exists(path):
                os.remove(path)
            B.snp_writeBed(g, path, ir, ic)
            raw = np.fromfile(path, dtype=np.uint8)
            assert raw[:3].tolist() == [108, 27, 1]
            assert np.array_equal(raw[3:].reshape(ic.size, -1), oracle.write_bed_bytes(want))
            with pytest.raises(FileExistsError):
                B.snp_writeBed(g, path, ir, ic)
            g2 = B.Bed(path, nrow=ir.size, ncol=ic.size)  # read back what was written
            assert np.array_equal(B.readbina2(g2, np.arange(1, ir.size + 1), np.arange(1, ic.size + 1)), want)
            g2.close()
    # FBM.code256-staged handle -> .bed (snp_writeBed's direction) and snp_readBed2 with a backing file
    Gf = rng.integers(0, 4, size=(37, 11)).astype(np.uint8)
    gf = B.Bed.from_fbm(Gf)
    p2 = str(tmp_path / "from_fbm.bed")
    B.snp_writeBed(gf, p2)
    assert np.array_equal(np.fromfile(p2, dtype=np.uint8)[3:].reshape(11, -1), oracle.write_bed_bytes(Gf))
    with open(p2[:-4] + ".bim", "w") as f:
        for j in range(11):
            f.write("1\ts%d\t0\t%d\tA\tC\n" % (j, 1000 * (j + 1)))
    with open(p2[:-4] + ".fam", "w") as f:
        for i in range(37):
            f.write("f%d i%d 0 0 0 -9\n" % (i, i))
    res = B.snp_readBed2(p2, backingfile=str(tmp_path / "bk1"), ind_col=np.arange(2, 9))
    assert np.array_equal(res["genotypes"], Gf[:, 1:8]) and res["map"]["physical.pos"][0] == 2000.0
    assert np.array_equal(np.fromfile(res["backingfile"], dtype=np.uint8).reshape(7, 37).T, Gf[:, 1:8])
    with pytest.raises(FileExistsError):
        B.snp_readBed2(p2, backingfile=str(tmp_path / "bk1"))


def test_snp_clumping_identical_to_oracle(B, gbed, oracle, obed, rng):
    # tests/testthat/test-2-bed-clumping-SVD.R:34-36,47-48 and R/clumping.R:62-137: FBM.code256 clumping, indices
    # identical to the oracle; equal to bed_clumping on a file without missing values; missing genotypes never prune
    chrom, pos = oracle.read_bim(obed.bedfile)
    G = oracle.read_bed(obed, obed.rows_along(), obed.cols_along(), na_val=3).astype(np.uint8)
    gf, of = B.Bed.from_fbm(G), oracle.OracleFBM(G)
    k = B.snp_clumping(gf, chrom, infos_pos=pos)
    assert np.array_equal(k, oracle.snp_clumping(of, chrom, infos_pos=pos))
    assert np.array_equal(k, B.bed_clumping(gbed))
    ir = rng.choice(obed.nrow, 300, replace=False) + 1
    S = rng.uniform(size=obed.ncol)
    for kw in (dict(thr_r2=0.1, size=50), dict(thr_r2=0.5, infos_pos=pos, size=200, S=S),
               dict(ind_row=ir, exclude=np.arange(1, 500), thr_r2=0.2)):
        assert np.array_equal(B.snp_clumping(gf, chrom, **kw), oracle.snp_clumping(of, chrom, **kw))
    G2 = G[:, :600].copy()
    G2[rng.uniform(size=G2.shape) < 0.01] = 3
    g2, o2 = B.Bed.from_fbm(G2), oracle.OracleFBM(G2)
    ch2 = chrom[:600]
    assert np.array_equal(B.snp_clumping(g2, ch2, thr_r2=0.2), oracle.snp_clumping(o2, ch2, thr_r2=0.2))
    with pytest.raises(ValueError, match=B.ERROR_DIM):
        B.snp_clumping(gf, chrom[:-1])


def test_bed_autoSVD_flow(B, gbed, oracle, obed, capsys):
    # tests/testthat/test-2-autoSVD.R:68-100 (structure: errors, messages, subset / lrldr attributes); the outlier
    # statistic is bigutilsr's (host R code), so a synthetic outlier function drives the pruning loop here
    with pytest.raises(ValueError, match="no variation; set min.mac > 0"):
        B.bed_autoSVD(gbed, min_mac=0)
    svd = B.bed_autoSVD(gbed, k=5, outlier_fun=None)  # first iteration only: MAF / MAC filter -> clumping -> SVD
    keep = svd["subset"]
    info = B.bed_MAF(gbed)
    ok = np.where(~((info["mac"] < 10) | (info["maf"] < 0.02)))[0] + 1
    want_keep = oracle.bed_clumping(obed, exclude=np.setdiff1d(np.arange(1, obed.ncol + 1), ok))
    assert np.array_equal(keep, want_keep) and svd["lrldr"] == []
    ref = oracle.bed_randomSVD(obed, ind_col=keep, k=5)
    np.testing.assert_allclose(svd["d"], ref["d"], rtol=1e-7)
    B.bed_autoSVD(gbed, thr_r2=np.nan, k=3, verbose=True)
    assert "Skipping clumping." in capsys.readouterr().out
    calls = []

    def fake_outliers(v, chr_keep):  # first round: a run of 30 consecutive variants + 2 isolated ones; then none
        calls.append(v.shape)
        return np.r_[100:130, 500, 900] if len(calls) == 1 else np.zeros(0, dtype=int)

    svd2 = B.bed_autoSVD(gbed, k=5, outlier_fun=fake_outliers)
    assert len(calls) == 2 and svd2["subset"].size == keep.size - 32
    assert len(svd2["lrldr"]) == 1 and svd2["lrldr"][0][3] == 1 and svd2["lrldr"][0][1] <= svd2["lrldr"][0][2]
    svd3 = B.bed_autoSVD(gbed, k=3, max_iter=1, outlier_fun=lambda v, c: np.array([0]), verbose=True)
    assert "Maximum number of iterations reached." in capsys.readouterr().out and svd3["subset"].size == keep.size - 1
    # snp_autoSVD on the FBM.code256 twin of the same (missing-free) data: same subset, same singular values
    chrom, pos = oracle.read_bim(obed.bedfile)
    Gf = oracle.read_bed(obed, obed.rows_along(), obed.cols_along(), na_val=3).astype(np.uint8)
    gf = B.Bed.from_fbm(Gf)
    svd4 = B.snp_autoSVD(gf, chrom, pos, k=5, outlier_fun=None)
    assert np.array_equal(svd4["subset"], keep)
    np.testing.assert_allclose(svd4["d"], svd["d"], rtol=1e-9)
    with pytest.raises(ValueError, match=B.ERROR_DIM):
        B.snp_autoSVD(gf, chrom[:-1], pos)
    # the default detector (OGK distance -> rolling mean -> adjusted Tukey fence, R/autoSVD.R:295-302) drives the loop:
    # whatever it removes, the result is a fixed point of the reference's iteration -- the statistic applied to the final
    # loadings flags nothing, unless the iteration cap was hit -- and the removed variants come out of the clumped set
    from bigsnpr_b200.outliers import autosvd_outlier_fun

    svd5 = B.bed_autoSVD(gbed, k=5, roll_size=10, verbose=True)
    out = capsys.readouterr().out
    assert set(svd5["subset"]) <= set(keep) and svd5["v"].shape == (svd5["subset"].size, 5)
    if "Maximum number of iterations reached." not in out:
        assert "Converged!" in out
        assert autosvd_outlier_fun(10, 0.05)(svd5["v"], chrom[svd5["subset"] - 1]).size == 0


def test_edge_shapes_and_empty_selections(B, oracle, rng, tmp_path):
    """Ragged and degenerate inputs through every product path: empty ind.row / ind.col, 1 x 1, n not a multiple of 4,
    fewer columns than one IMMA step, out-of-bounds subscripts (src/bed-acc.h:64-65)."""
    for n, m in ((1, 1), (3, 2), (5, 33), (130, 31), (257, 1030)):
        G = rng.integers(0, 4, size=(n, m)).astype(np.uint8)
        if n * m > 4:
            G[0, 0], G[-1, -1] = 3, 2
        path = oracle.write_bed(str(tmp_path / ("e_%d_%d.bed" % (n, m))), G)
        o = oracle.OracleBed(path)
        for layouts in (B.LAYOUT_SNP_MAJOR, B.LAYOUT_SNP_MAJOR | B.LAYOUT_SAMPLE_MAJOR):
            g = B.Bed(path, layouts=layouts)
            y_col, y_row = rng.normal(size=m), rng.normal(size=n)
            c, s = rng.normal(size=m), rng.uniform(0.5, 1.5, size=m)
            _close(B.bed_prodVec(g, y_col, center=c, scale=s), oracle.bed_prodVec(o, y_col, center=c, scale=s),
                   scale=np.max(np.abs(y_col / s)) * m * 3 + 1e-300)
            _close(B.bed_cprodVec(g, y_row, center=c, scale=s), oracle.bed_cprodVec(o, y_row, center=c, scale=s),
                   scale=np.max(np.abs(y_row)) * n * 3 / np.min(s) + 1e-300)
            assert np.array_equal(B.bed_counts(g), oracle.bed_counts(o))
            assert np.array_equal(B.bed_counts(g, byrow=True), oracle.bed_counts(o, byrow=True))
            e = np.zeros(0, dtype=np.int32)
            allr, allc = np.arange(1, n + 1), np.arange(1, m + 1)
            assert B.bed_prodVec(g, np.zeros(m), e, allc).shape == (0,)
            assert np.array_equal(B.bed_prodVec(g, np.zeros(0), allr, e), np.zeros(n))
            assert np.array_equal(B.bed_cprodVec(g, np.zeros(0), e, allc), np.zeros(m))
            assert B.bed_cprodVec(g, np.zeros(n), allr, e).shape == (0,)
            assert B.bed_counts(g, allr, e).shape == (4, 0) and B.readbina2(g, e, allc).shape == (0, m)
            XV, rss = B.prod_and_rowSumsSq(g, allr, allc, c, s, rng.normal(size=(m, 2)))
            assert XV.shape == (n, 2) and rss.shape == (n,)
            with pytest.raises(B.BsgError, match="out of bounds"):
                B.bed_prodVec(g, np.zeros(1), allr, np.array([m + 1]))
            with pytest.raises(B.BsgError, match="out of bounds"):
                B.bed_cprodVec(g, np.zeros(1), np.array([0]), allc)
            g.close()


def test_sparse_missing_lists_equal_plane_path(B, oracle, obed_na, rng, monkeypatch):
    """Missing values handled by the blocked-ELL lists (default for rates <= 4 %, bsg_naell.cu) and by the flag plane give
    the same numbers: both sum the same integers exactly and differ only in the fp64 rounding of the last combination
    (the lists deliver the sum as two 32-bit halves, the plane as eight digit slices)."""
    f = os.path.join(GOLDEN, "example-missing.bed")
    N, M = obed_na.nrow, obed_na.ncol
    monkeypatch.setenv("BSG_NA_LIST_MAX_RATE", "1.0")
    g_list = B.Bed(f)
    monkeypatch.setenv("BSG_NA_LISTS", "0")
    g_plane = B.Bed(f)
    sc = oracle.bed_scaleBinom(obed_na)
    cases = [(np.arange(1, N + 1), np.arange(1, M + 1)),
             (rng.choice(N, N // 2, replace=False) + 1, rng.choice(M, M // 2, replace=False) + 1),
             (rng.integers(1, N + 1, N + 7), rng.integers(1, M + 1, M + 9))]
    for ir, ic in cases:
        y_col, y_row = rng.normal(size=ic.size), rng.normal(size=ir.size)
        for cs in ((None, None), (sc["center"][ic - 1], sc["scale"][ic - 1])):
            monkeypatch.setenv("BSG_NA_LISTS", "1")
            a1, b1 = B.bed_prodVec(g_list, y_col, ir, ic, *cs), B.bed_cprodVec(g_list, y_row, ir, ic, *cs)
            monkeypatch.setenv("BSG_NA_LISTS", "0")
            a0, b0 = B.bed_prodVec(g_plane, y_col, ir, ic, *cs), B.bed_cprodVec(g_plane, y_row, ir, ic, *cs)
            _close(a1, a0, scale=np.max(np.abs(a0)), tol=1e-14)
            _close(b1, b0, scale=np.max(np.abs(b0)), tol=1e-14)
            s = cs[1] if cs[1] is not None else 1.0
            _close(a1, oracle.bed_prodVec(obed_na, y_col, ir, ic, *cs), scale=np.max(np.abs(y_col / s)) * ic.size * 3)
            _close(b1, oracle.bed_cprodVec(obed_na, y_row, ir, ic, *cs),
                   scale=np.max(np.abs(y_row)) * ir.size * 3 / (np.min(cs[1]) if cs[1] is not None else 1.0))
    monkeypatch.setenv("BSG_NA_LISTS", "1")
    svd1 = B.bed_randomSVD(g_list, k=5)
    svd0 = B.bed_randomSVD(g_plane, k=5)
    np.testing.assert_allclose(svd1["d"], svd0["d"], rtol=1e-12)


def test_snp_colstats_direct_with_missing(B, oracle, rng):
    """src/colstats.cpp:8-35 on an FBM.code256 handle, compared with the oracle directly: no NA handling, so a column with
    a missing code propagates NaN to sumX and denoX (x += NA_real in the reference); clean columns are bit-equal.  Row and
    column multisets included (tests/testthat/test-2-bed-clumping-SVD.R:21-27 uses snp_colstats through snp_clumping)."""
    n, m = 733, 411
    G = rng.integers(0, 3, size=(n, m)).astype(np.uint8)
    na_cols = rng.choice(m, 60, replace=False)
    for j in na_cols:
        G[rng.choice(n, rng.integers(1, 20), replace=False), j] = 3
    gf, of = B.Bed.from_fbm(G), oracle.OracleFBM(G)
    cases = [(gf.rows_along(), gf.cols_along()),
             (rng.choice(n, 300, replace=False).astype(np.int32) + 1, rng.choice(m, 200, replace=False).astype(np.int32) + 1),
             (rng.integers(1, n + 1, size=500).astype(np.int32), rng.integers(1, m + 1, size=500).astype(np.int32))]
    for ir, ic in cases:
        got = B.snp_colstats(gf, ir, ic)
        want = oracle.snp_colstats(of, ir, ic)
        for key in ("sumX", "denoX"):
            assert np.array_equal(np.isnan(got[key]), np.isnan(want[key])), key
            ok = ~np.isnan(want[key])
            assert np.array_equal(got[key][ok], want[key][ok]), key
        # a column is NaN exactly when one of its selected rows is missing
        has_na = (G[np.ix_(ir - 1, ic - 1)] == 3).any(axis=0)
        assert np.array_equal(np.isnan(got["sumX"]), has_na)
    # snp_MAF / snp_scaleBinom on the same statistics (R/binom-scaling.R:62-106)
    clean = np.setdiff1d(np.arange(m), na_cols)[:50].astype(np.int32) + 1
    af = oracle.snp_colstats(of, of.rows_along(), clean)["sumX"] / (2 * n)
    assert np.array_equal(B.snp_MAF(gf, ind_col=clean), np.minimum(af, 1 - af))
    sc = B.snp_scaleBinom()(gf, ind_col=clean)
    sco = oracle.snp_scaleBinom(of, None, clean)
    assert np.array_equal(sc["center"], sco["center"]) and np.array_equal(sc["scale"], sco["scale"])
    gf.close()


def test_ld_structured_generator_matches_its_twins(B, oracle):
    """bsg_open_synth_ld == the NumPy mirror == the oracle's C twin, bit for bit; shards by global column; rho = 0 is the
    i.i.d. generator; neighbouring SNPs inside a block are really correlated."""
    from tests.synth_ref import synth_matrix, synth_matrix_ld

    n, m = 1003, 237
    for na_rate, off in ((0.0, 0), (0.03, 33)):
        g = B.Bed.synthetic(n, m, seed=9, na_rate=na_rate, col_offset=off, ld_rho=0.9, ld_block=50)
        G = synth_matrix_ld(n, m, seed=9, na_rate=na_rate, col_offset=off, rho=0.9, ld_block=50)
        o = oracle.OracleBed.from_packed(g.export_packed(), n, m)
        assert np.array_equal(oracle.decode_dense(o), G)
        o2 = oracle.synth_bed(n, m, seed=9, na_rate=na_rate, col_offset=off, ld_rho=0.9, ld_block=50)
        assert np.array_equal(oracle.decode_dense(o2), G)
        g.close()
    import ctypes as C

    from bigsnpr_b200 import _lib

    h = C.c_void_p()
    _lib.check(_lib.lib().bsg_open_synth_ld(n, m, 9, 0.02, 5, 0.0, 50, 0, 0, C.byref(h)))
    g0 = B.Bed(_handle=h, _shape=(n, m))
    assert np.array_equal(oracle.decode_dense(oracle.OracleBed.from_packed(g0.export_packed(), n, m)),
                          synth_matrix(n, m, seed=9, na_rate=0.02, col_offset=5))
    g0.close()
    big = B.Bed.synthetic(20000, 200, seed=2, ld_rho=0.9, ld_block=50)
    p, i, x = B.bed_cor(big, size=1, thr_r2=0.0)  # adjacent pairs only (1 kb = 1 SNP)
    adj = np.array([x[p[j]] for j in range(1, 200) if p[j + 1] - p[j] == 2])
    inside = np.array([j % 50 != 0 for j in range(1, 200) if p[j + 1] - p[j] == 2])
    assert np.mean(adj[inside] ** 2) > 0.2 and np.mean(adj[~inside] ** 2) < 0.01
    big.close()


def test_group_entry_points_vs_oracle(B, oracle, rng):
    """The single-process multi-GPU entry points of the C ABI (bsg_group_*, SURVEY.md section 8e): column shards over up to
    two of the visible devices (one on a single-GPU box: same code path, no exchange), against the oracle on the whole
    matrix -- products with global multiset indices, bed_randomSVD vs the dense decomposition, the GRM."""
    from bigsnpr_b200 import _lib

    ndev = max(1, min(2, _lib.lib().bsg_device_count()))
    n, m = 2003, 6011
    grp = B.Group.synthetic(n, m, list(range(ndev)), seed=13, na_rate=0.02)
    o = oracle.synth_bed(n, m, seed=13, na_rate=0.02)
    sc = grp.scaleBinom()
    sco = oracle.bed_scaleBinom(o)
    assert np.array_equal(sc["center"], sco["center"]) and np.array_equal(sc["scale"], sco["scale"])
    x, y = rng.normal(size=m), rng.normal(size=n)
    _close(grp.prodVec(x, center=sc["center"], scale=sc["scale"]), oracle.bed_prodVec(o, x, center=sc["center"], scale=sc["scale"]),
           scale=np.max(np.abs(x / sc["scale"])) * m)
    _close(grp.cprodVec(y, center=sc["center"], scale=sc["scale"]), oracle.bed_cprodVec(o, y, center=sc["center"], scale=sc["scale"]),
           scale=np.max(np.abs(y)) * n / np.min(sc["scale"]))
    ir = rng.integers(1, n + 1, size=700).astype(np.int32)
    ic = rng.integers(1, m + 1, size=900).astype(np.int32)  # unsorted, with duplicates, spanning both shards
    xs, ys = rng.normal(size=ic.size), rng.normal(size=ir.size)
    _close(grp.prodVec(xs, ind_row=ir, ind_col=ic), oracle.bed_prodVec(o, xs, ind_row=ir, ind_col=ic), scale=np.max(np.abs(xs)) * ic.size)
    _close(grp.cprodVec(ys, ind_row=ir, ind_col=ic), oracle.bed_cprodVec(o, ys, ind_row=ir, ind_col=ic), scale=np.max(np.abs(ys)) * ir.size)
    with pytest.raises(B.BsgError, match="out of bounds"):
        grp.prodVec(np.zeros(1), ind_col=[m + 1])
    sub = np.arange(1, m + 1, 3).astype(np.int32)
    svd = grp.randomSVD(ind_col=sub, k=6)
    dense = oracle.bed_randomSVD(o, ind_col=sub, k=6)
    assert np.max(np.abs(svd["d"] - dense["d"]) / dense["d"]) < 1e-7
    assert np.min(np.abs(np.sum(svd["u"] * dense["u"], axis=0))) > 1 - 1e-6
    assert np.min(np.abs(np.sum(svd["v"] * dense["v"], axis=0))) > 1 - 1e-6
    assert np.array_equal(svd["center"], sc["center"][sub - 1])
    K = grp.tcrossprodSelf(sc["center"][sub - 1], sc["scale"][sub - 1], ind_col=sub)
    K0, _, _ = oracle.bed_tcrossprodSelf(o, ind_col=sub)
    assert np.max(np.abs(K - K0)) / np.max(np.abs(K0)) < 1e-8
    grp.close()


def test_dosage_fbm_generic_code_fallback(B, oracle, rng):
    """SURVEY.md section 8f row 3: an FBM.code256 whose codes are dosages (CODE_DOSAGE-like: byte / 100 for 0..200, NA above;
    R/bigSNP-class.R:13) is served by the fp64 kernels of bsg_generic.cu with the reference's per-element semantics
    (code256[byte], NA -> 3 for the pairwise statistics): snp_colstats, snp_cor, snp_ld_scores, snp_clumping, multLinReg /
    snp_pcadapt against the oracle's literal loops.  Sums of non-integers: 1e-10, far inside the 1e-6 contract."""
    n, m = 811, 403
    code = np.full(256, np.nan)
    code[:201] = np.arange(201) / 100.0
    # correlated dosages: blocks of 20 columns share a latent variable, so clumping prunes and thresholds matter
    lat = rng.normal(size=(n, (m + 19) // 20))
    prob = 1 / (1 + np.exp(-(0.9 * lat[:, np.arange(m) // 20] + 0.6 * rng.normal(size=(n, m)))))
    G = np.clip(np.rint(200 * prob), 0, 200).astype(np.uint8)
    na = rng.random(size=(n, m)) < 0.01
    na[:, :50] = False  # the first 50 columns stay complete
    G[na] = 255
    gf, of = B.Bed.from_fbm(G, code256=code), oracle.OracleFBM(G, code256=code)
    ir = np.sort(rng.choice(n, 700, replace=False)).astype(np.int32) + 1
    ic = np.arange(1, m + 1, dtype=np.int32)
    st, st0 = B.snp_colstats(gf, ir, ic), oracle.snp_colstats(of, ir, ic)
    for k in ("sumX", "denoX"):
        assert np.array_equal(np.isnan(st[k]), np.isnan(st0[k]))
        ok = ~np.isnan(st0[k])
        assert np.allclose(st[k][ok], st0[k][ok], rtol=1e-12)
    assert np.isnan(st0["sumX"]).any() and not np.isnan(st0["sumX"][:50]).any()
    for kw in (dict(size=30, thr_r2=0.0), dict(size=30, thr_r2=0.1), dict(size=12, alpha=0.01)):
        p, i, x = B.snp_cor(gf, ir, ic, **kw)
        p0, i0, x0 = oracle.cor0(of, ir, ic, **kw)
        assert np.array_equal(p, p0) and np.array_equal(i, i0)
        assert np.allclose(x, x0, rtol=0, atol=1e-10)
    ld, ld0 = B.snp_ld_scores(gf, ir, ic, size=30), oracle.ld0(of, ir, ic, size=30)
    assert np.allclose(ld, ld0, rtol=1e-10)
    chrom = np.ones(m, dtype=int)
    excl = np.nonzero(np.isnan(st0["sumX"]))[0] + 1  # like the reference, clumping on columns with NA statistics is moot
    for kw in (dict(thr_r2=0.2), dict(thr_r2=0.05, size=40)):
        k1 = B.snp_clumping(gf, chrom, ind_row=ir, exclude=excl, **kw)
        k0 = oracle.snp_clumping(of, chrom, ind_row=ir, exclude=excl, **kw)
        assert np.array_equal(k1, k0)
    assert k1.size < m - excl.size
    U = np.linalg.qr(rng.normal(size=(ir.size, 3)))[0]
    t, t0 = B.multLinReg(gf, ir, ic, U), oracle.multLinReg(of, ir, ic, U)
    assert np.array_equal(np.isnan(t), np.isnan(t0)) and np.allclose(t[~np.isnan(t0)], t0[~np.isnan(t0)], rtol=1e-9)
    with pytest.raises(B.BsgError, match="needs hard calls"):
        B.bed_counts(gf)
    with pytest.raises(B.BsgError, match="needs hard calls"):
        B.bed_tcrossprodSelf(gf, fun_scaling=lambda *a, **k: {"center": np.zeros(m), "scale": np.ones(m)})
    gf.close()
