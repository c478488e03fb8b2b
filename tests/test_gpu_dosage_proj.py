"""PCA projection and autoSVD on FBM.code256 handles: prod_and_rowSumsSq2 / snp_projectSelfPCA (src/project-utils.cpp:11-43,
R/bed-projectPCA.R:252-281) on dosage and hard-call FBMs with NA codes, snp_autoSVD on a mean2-imputed dosage FBM
(R/autoSVD.R:96-101: snp_MAF, then snp_clumping), and the two R-shim entry points that reach these paths.

References: the literal loop of project-utils.cpp written out in NumPy (x = (code256[b] - c) / s, NA code = NA_real); the
oracle's snp_colstats / snp_clumping for the autoSVD subset; a dense SVD for d.
"""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CODE_DOSAGE = np.concatenate([[0, 1, 2, np.nan, 0, 1, 2], np.arange(201) * 0.01, np.full(48, np.nan)])
CODE_012 = np.r_[[0.0, 1.0, 2.0], np.full(253, np.nan)]


@pytest.fixture(scope="module")
def B():
    import bigsnpr_b200 as b

    from bigsnpr_b200 import build

    build.build()
    return b


def _imputed_example(B):
    """example-missing.bed -> FBM codes -> snp_fastImputeSimple(method = "mean2") (src/impute-simple.cpp): a missing call
    becomes code 7 + round(100 * mean of the observed calls); ties at exact .5 need not match R's rounding."""
    gb = B.Bed(os.path.join(GOLDEN, "example-missing.bed"))
    G = gb[None, None]
    chrom = gb.map["chromosome"]
    gb.close()
    G = np.where(G == B.NA_INTEGER, 3, G).astype(np.uint8)
    for j in range(G.shape[1]):
        na = G[:, j] == 3
        if na.any():
            G[na, j] = 7 + int(np.rint(100 * G[~na, j].mean()))
    return G, chrom


def _lit_proj(G, code, ir, ic, c, s, V):
    """the reference's loop: x = (code256[b] - c_j) / s_j; rowSumsSq += x^2; XV += x V[j, ]"""
    with np.errstate(all="ignore"):
        X = (code[G[np.ix_(ir - 1, ic - 1)]] - c) / s
        XV = np.stack([(X * V[:, k][None, :]).sum(axis=1) for k in range(V.shape[1])], axis=1)
        return XV, (X * X).sum(axis=1)


def _check(got, want, tol=1e-12):
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    assert ok.any()
    assert np.max(np.abs(got[ok] - want[ok])) / np.max(np.abs(want[ok])) < tol


@pytest.mark.parametrize("kind", ["dosage", "hard_calls"])
def test_prod_and_rowSumsSq2_vs_literal_loop(B, kind):
    rng = np.random.default_rng(31)
    n, m = 611, 1301
    if kind == "dosage":
        G = (7 + rng.integers(0, 201, size=(n, m))).astype(np.uint8)
        G[rng.random(size=(n, m)) < 0.3] = rng.integers(0, 3, size=1)[0] + 4  # codes 4-6 mixed in
        G[rng.random(size=(n, m)) < 0.0005] = 240  # NA codes
        code = CODE_DOSAGE
    else:
        G = rng.integers(0, 3, size=(n, m)).astype(np.uint8)
        G[rng.random(size=(n, m)) < 0.0005] = 3
        code = CODE_012
    g = B.Bed.from_fbm(G, code256=code)
    assert g.dosage_scale == (100 if kind == "dosage" else 0)
    for ir, ic in ((np.arange(1, n + 1, dtype=np.int32), rng.permutation(m)[:900].astype(np.int32) + 1),
                   (rng.integers(1, n + 1, size=400).astype(np.int32), np.arange(1, m + 1, dtype=np.int32))):
        c, s = rng.uniform(0.2, 1.8, size=ic.size), rng.uniform(0.3, 1.2, size=ic.size)
        V = rng.normal(size=(ic.size, 5))
        XV, rss = B.prod_and_rowSumsSq2(g, ir, ic, c, s, V)
        XV0, rss0 = _lit_proj(G, code, ir, ic, c, s, V)
        assert np.isnan(rss0).any() and not np.isnan(rss0).all()
        _check(XV, XV0)
        _check(rss, rss0)
        assert np.array_equal(np.isnan(XV).any(axis=1), np.isnan(rss))
    # snp_projectSelfPCA takes ind.col from the SVD's subset
    ic = np.arange(1, m + 1, 2, dtype=np.int32)
    svd = {"v": np.linalg.qr(rng.normal(size=(ic.size, 4)))[0], "d": np.arange(4, 0, -1.0),
           "center": rng.uniform(0.2, 1.8, size=ic.size), "scale": rng.uniform(0.3, 1.2, size=ic.size), "subset": ic}
    ir = np.arange(1, n + 1, dtype=np.int32)
    pr = B.snp_projectSelfPCA(svd, g, ir)
    XV0, rss0 = _lit_proj(G, code, ir, ic, svd["center"], svd["scale"], svd["v"])
    _check(pr["simple_proj"], XV0)
    _check(pr["X_norm"], rss0)
    g.close()


def test_prod_and_rowSumsSq2_refusals(B):
    G = np.zeros((20, 10), dtype=np.uint8)
    g = B.Bed.from_fbm(G, code256=np.linspace(0, 2, 256))  # not a dosage table: the packed engine refuses it by name
    with pytest.raises(B.BsgError, match="needs hard calls"):
        B.prod_and_rowSumsSq2(g, np.arange(1, 21), np.arange(1, 11), np.zeros(10), np.ones(10), np.ones((10, 2)))
    g.close()
    bed = B.Bed(os.path.join(GOLDEN, "example.bed"))
    with pytest.raises(B.BsgError, match="FBM.code256"):
        B.prod_and_rowSumsSq2(bed, np.arange(1, 21), np.arange(1, 11), np.zeros(10), np.ones(10), np.ones((10, 2)))
    bed.close()


def test_snp_autoSVD_on_imputed_dosages(B, oracle):
    G, chrom = _imputed_example(B)
    n, m = G.shape
    g = B.Bed.from_fbm(G, code256=CODE_DOSAGE)
    assert g.dosage_scale == 100
    k = 5
    svd = B.snp_autoSVD(g, chrom, k=k, outlier_fun=None)  # no outlier rounds: the subset is the first iteration's
    # oracle: snp_MAF with the reference's rule, then snp_clumping on the kept variants (R/autoSVD.R:96-112)
    of = oracle.OracleFBM(G, code256=CODE_DOSAGE)
    ir, ic = np.arange(1, n + 1, dtype=np.int32), np.arange(1, m + 1, dtype=np.int32)
    af = oracle.snp_colstats(of, ir, ic)["sumX"] / (2 * n)
    maf0 = np.minimum(af, 1 - af)
    maf = B.snp_MAF(g)
    assert np.allclose(maf, maf0, rtol=1e-12, atol=0)
    keep = ic[~(maf0 < max(0.02, 10 / (2 * n)))]
    assert np.array_equal(keep, ic[~(maf < max(0.02, 10 / (2 * n)))])
    excl = np.setdiff1d(ic, keep)
    # mean-imputed columns share MAF values up to the last bits of their fp64 sums, so the greedy order of the clumping
    # is taken from the engine's MAF (the priority S of R/clumping.R:93-137) and the oracle's pair statistics decide
    sub0 = oracle.snp_clumping(of, chrom, ind_row=ir, S=maf, exclude=excl, thr_r2=0.2, size=500)
    assert np.array_equal(np.sort(svd["subset"]), np.sort(np.asarray(sub0))) and 0 < svd["subset"].size < m
    st = B.snp_scaleBinom()(g, ind_col=svd["subset"])
    with np.errstate(all="ignore"):
        X = (CODE_DOSAGE[G[:, svd["subset"] - 1]] - st["center"]) / st["scale"]
    d = np.linalg.svd(X, compute_uv=False)[:k]
    assert np.max(np.abs(svd["d"] - d) / d) < 1e-7
    g.close()


@pytest.fixture(scope="module")
def R(tmp_path_factory):
    from tests.test_abi import build_shim_with_minir
    from tests.test_gpu_shim import MiniR

    return MiniR(build_shim_with_minir(tmp_path_factory.mktemp("shim_dosage")))


def test_shim_dosage_fbm_entry_points(R, tmp_path):
    rng = np.random.default_rng(33)
    n, m = 403, 707
    # four strong components (separated singular values) plus noise, dosages x 100 in 0..200
    lat = rng.normal(size=(n, 4)) * np.array([4.0, 3.0, 2.0, 1.5])
    val = 100 + 12 * lat @ rng.normal(size=(4, m)) + 15 * rng.normal(size=(n, m))
    G = (7 + np.clip(np.rint(val), 0, 200)).astype(np.uint8)
    G[rng.random(size=(n, m)) < 0.001] = 250
    bk = tmp_path / "dosage.bk"
    np.asfortranarray(G).T.tofile(bk)  # column-major n x m bytes, as the .bk file
    fbm = R.env(backingfile=R.s(str(bk)), nrow=R.ints([n]), ncol=R.ints([m]), code256=R.reals(CODE_DOSAGE))
    ir = np.arange(1, n + 1, dtype=np.int32)
    ic = rng.permutation(m)[:500].astype(np.int32) + 1
    c, s = rng.uniform(0.2, 1.8, size=ic.size), rng.uniform(0.3, 1.2, size=ic.size)
    V = rng.normal(size=(ic.size, 3))
    pr = R.call("_bigsnpr_prod_and_rowSumsSq2", fbm, R.ints(ir), R.ints(ic), R.reals(c), R.reals(s), R.mat(V))
    XV0, rss0 = _lit_proj(G, CODE_DOSAGE, ir, ic, c, s, V)
    _check(R.vec(R.L.minir_list_get(pr, 0)), XV0)
    _check(R.vec(R.L.minir_list_get(pr, 1)), rss0)
    # big_randomSVD's branch of snp_autoSVD: the FBM environment with explicit (snp_scaleBinom-like) scaling
    ok = np.nonzero(~(G == 250).any(axis=0))[0].astype(np.int32) + 1
    X0 = CODE_DOSAGE[G[:, ok - 1]]
    cen = X0.mean(axis=0)
    sca = np.sqrt(cen / 2 * (1 - cen / 2) * 2)
    sv = R.call("_bigsnpr_bed_randomSVD_gpu", fbm, R.ints(ir), R.ints(ok), R.reals(cen), R.reals(sca), R.ints([4]),
                R.reals([1e-4]))
    d = R.vec(R.named(sv, "d"))
    d0 = np.linalg.svd((X0 - cen) / sca, compute_uv=False)[:4]
    assert np.max(np.abs(d - d0) / d0) < 1e-7
    R.L.minir_run_finalizers()
