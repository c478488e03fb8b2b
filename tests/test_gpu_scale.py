"""GPU parity at BASELINE.json's sizes: the CUDA path (through the C ABI) against the CPU ORACLE -- not against
itself -- on the shapes whose code paths do not exist at fixture size:

* configs[1] in full (50,000 x 500,000): one bed_pMatVec4 and one bed_cpMatVec4 of the oracle's literal port on all host
  threads, both HBM layouts, counts and binomial scaling bit for bit;
* 487,000 x 4,096 and 4,096 x 600,000: every line longer than 262,144 codes is k-split (bsg_pmv.cu MAX_CHUNKS_PER_ITEM),
  which is what every configs[4] cprodVec (n = 487,000) and every configs[1] prodVec (m = 500,000) runs; with and without
  1 % missing values, SNP-major copy alone and both copies;
* a configs[2]-shaped slice (100,000 x 2,000, 500-SNP window, LD-structured data): bed_cor, bed_ld_scores, bed_clumping;
* a configs[3]-shaped slice (10,000 x 20,000): bed_tcrossprodSelf.

The relational form is the reference's own (tests/testthat/test-5-bed-prod-vec.R:18-41: products == dense decode %*% vector,
default and random center / scale); the oracle's loops are that dense product restated literally.  Tolerances are the
north_star's: bit-exact for counts / indices, 1e-6 relative for floating point -- the tests ask for much less
(1e-11 of the vector scale for the products, 1e-8 for K: 28-bit weights); r is held to the oracle's bytes.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SEED_CFG2 = 20250924 + 1


@pytest.fixture(scope="module")
def B():
    import bigsnpr_b200 as b
    from bigsnpr_b200 import build

    build.build()
    return b


def _relerr(got, want, scale):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape
    return float(np.max(np.abs(got - want)) / scale)


def _free_gb():
    import torch

    return torch.cuda.mem_get_info()[0] / 1e9


def _products_vs_oracle(B, oracle, g, o, rng, tol=1e-11, random_scaling=True):
    """bed_prodVec / bed_cprodVec == oracle, with binomial scaling and (reference test :32-39) random center / scale."""
    n, m = o.nrow, o.ncol
    nt = oracle.max_threads()
    sc = B.bed_scaleBinom(g)
    sco = oracle.bed_scaleBinom(o, ncores=nt)
    assert np.array_equal(sc["center"], sco["center"]) and np.array_equal(sc["scale"], sco["scale"])
    y_col, y_row = rng.normal(size=m), rng.normal(size=n)
    worst = 0.0
    scalings = [(sc["center"], sc["scale"])]
    if random_scaling:
        scalings.append((rng.normal(size=m), rng.uniform(0.05, 1.0, size=m)))
    for center, scale in scalings:
        a = B.bed_prodVec(g, y_col, center=center, scale=scale)
        a0 = oracle.bed_prodVec(o, y_col, center=center, scale=scale, ncores=nt)
        b = B.bed_cprodVec(g, y_row, center=center, scale=scale)
        b0 = oracle.bed_cprodVec(o, y_row, center=center, scale=scale, ncores=nt)
        # scale of the sums: every term is bounded by |y| * max(|g - c|) / s
        sa = np.max(np.abs(y_col) * (3 + np.abs(center)) / scale) * np.sqrt(m)
        sb = np.max(np.abs(y_row)) * np.sqrt(n) * np.max((3 + np.abs(center)) / scale)
        ea, eb = _relerr(a, a0, sa), _relerr(b, b0, sb)
        assert ea < tol and eb < tol, (ea, eb)
        # and in the plain sense of the reference's expect_equal (relative to the result's own size)
        assert _relerr(a, a0, np.max(np.abs(a0))) < 1e-9 and _relerr(b, b0, np.max(np.abs(b0))) < 1e-9
        worst = max(worst, ea, eb)
    return worst


def test_cfg2_full_size_vs_oracle(B, oracle, rng):
    """configs[1] in full: 50,000 x 500,000 (6.25 GB packed).  The oracle's generator is the bit-exact twin of the device
    generator, so both sides see the same matrix; ~1-2 s per oracle product on 64 threads."""
    if _free_gb() < 30:
        pytest.skip("needs ~14 GB of HBM")
    n, m = 50_000, 500_000
    o = oracle.synth_bed(n, m, seed=SEED_CFG2)
    nt = oracle.max_threads()
    for layouts in (B.LAYOUT_SNP_MAJOR, B.LAYOUT_SNP_MAJOR | B.LAYOUT_SAMPLE_MAJOR):
        g = B.Bed.synthetic(n, m, seed=SEED_CFG2, layouts=layouts)
        assert g.layouts == layouts
        if layouts == B.LAYOUT_SNP_MAJOR:
            assert np.array_equal(B.bed_counts(g), oracle.bed_col_counts_cpp(o, o.rows_along(), o.cols_along(), nt))
        _products_vs_oracle(B, oracle, g, o, rng, random_scaling=(layouts == B.LAYOUT_SNP_MAJOR))
        g.close()


@pytest.mark.parametrize("shape", [(487_000, 4_096), (4_096, 600_000)])
@pytest.mark.parametrize("na_rate", [0.0, 0.01])
def test_ksplit_shapes_vs_oracle(B, oracle, rng, shape, na_rate):
    """Lines longer than 262,144 codes are split (k-split >= 2) on the side whose contraction is long: Xt.y for
    n = 487,000 (configs[4]'s sample count), X.y for m = 600,000.  Both HBM layouts, with and without missing values."""
    n, m = shape
    o = oracle.synth_bed(n, m, seed=77, na_rate=na_rate)
    for layouts in (B.LAYOUT_SNP_MAJOR, B.LAYOUT_SNP_MAJOR | B.LAYOUT_SAMPLE_MAJOR):
        g = B.Bed.synthetic(n, m, seed=77, na_rate=na_rate, layouts=layouts)
        assert g.has_na == (na_rate > 0)
        _products_vs_oracle(B, oracle, g, o, rng)
        # multiset indices on the long side (duplicates scatter-add in integers)
        ir = rng.integers(1, n + 1, size=min(n, 3000)).astype(np.int32)
        ic = rng.integers(1, m + 1, size=min(m, 3000)).astype(np.int32)
        y = rng.normal(size=ic.size)
        nt = oracle.max_threads()
        a = B.bed_prodVec(g, y, ind_row=ir, ind_col=ic)
        a0 = oracle.bed_prodVec(o, y, ind_row=ir, ind_col=ic, ncores=nt)
        assert _relerr(a, a0, np.max(np.abs(a0)) + 1) < 1e-11
        yr = rng.normal(size=ir.size)
        b = B.bed_cprodVec(g, yr, ind_row=ir, ind_col=ic)
        b0 = oracle.bed_cprodVec(o, yr, ind_row=ir, ind_col=ic, ncores=nt)
        assert _relerr(b, b0, np.max(np.abs(b0)) + 1) < 1e-11
        g.close()


@pytest.mark.parametrize("na_rate", [0.0, 0.005])
def test_cfg3_slice_cor_ld_clumping_vs_oracle(B, oracle, na_rate):
    """configs[2]-shaped slice: 100,000 samples x 2,000 SNPs, 500-SNP window, LD-structured synthetic data (blocks of 50
    correlated SNPs) so thresholds and pruning are exercised.  r is compared byte for byte with the same sparsity pattern,
    LD scores to 1e-10 against the oracle (another summation order) and byte for byte against tests/cor_ref.py, clumping
    indices exactly."""
    n, m = 100_000, 2_000
    kw = dict(seed=31, na_rate=na_rate, ld_rho=0.9, ld_block=50)
    o = oracle.synth_bed(n, m, **kw)
    g = B.Bed.synthetic(n, m, **kw)
    nt = oracle.max_threads()
    pos = 1000.0 * np.arange(1, m + 1)
    for thr_r2 in (0.0, 0.2):
        p, i, x = B.bed_cor(g, size=500, thr_r2=thr_r2, infos_pos=pos)
        p0, i0, x0 = oracle.cor0(o, size=500, thr_r2=thr_r2, infos_pos=pos, ncores=nt)
        assert np.array_equal(p, p0) and np.array_equal(i, i0)
        assert np.array_equal(x, x0, equal_nan=True)
        if thr_r2 > 0:
            assert 0 < x.size < 0.5 * m * 500  # the threshold really prunes on this data
    assert np.mean(np.abs(x) > 0.3) > 0.01
    ld = B.bed_ld_scores(g, size=500, infos_pos=pos)
    ld0 = oracle.ld0(o, size=500, infos_pos=pos, ncores=nt)
    assert np.max(np.abs(ld - ld0) / ld0) < 1e-10 and np.max(ld0) > 3
    from tests import cor_ref

    assert np.array_equal(ld, cor_ref.ld_scores(oracle.decode_dense(o), 500 * 1000.0, pos))  # k_ld_reduce's order, exactly
    # clumping on the first 500 SNPs, +-100 SNP window (the oracle's sweep is single-threaded by construction)
    sub = np.arange(1, 501, dtype=np.int32)
    excl = np.arange(501, m + 1)
    chrom = np.ones(m, dtype=int)
    k = B.bed_clumping(g, thr_r2=0.2, size=100, exclude=excl, infos_chr=chrom, infos_pos=pos)
    k0 = oracle.bed_clumping(o, thr_r2=0.2, size=100, exclude=excl, infos_chr=chrom, infos_pos=pos)
    assert np.array_equal(k, k0)
    assert 20 < k.size < sub.size  # pruning happened
    g.close()


def test_cfg4_slice_grm_vs_oracle(B, oracle):
    """configs[3]-shaped slice: 10,000 samples x 20,000 SNPs (78 row tiles x 157 chunks: multi-tile bands and several
    accumulation passes of the Gram kernel).  K against the oracle's block loop (decode + fp64 GEMM)."""
    n, m = 10_000, 20_000
    for na_rate in (0.0, 0.01):
        o = oracle.synth_bed(n, m, seed=41, na_rate=na_rate)
        g = B.Bed.synthetic(n, m, seed=41, na_rate=na_rate)
        K, c, s = B.bed_tcrossprodSelf(g)
        K0, c0, s0 = oracle.bed_tcrossprodSelf(o, block_size=2000)
        assert np.array_equal(c, c0) and np.array_equal(s, s0)
        err = np.max(np.abs(K - K0)) / np.max(np.abs(K0))
        assert err < 1e-8, err  # 28-bit weights (4 base-128 digit slices), exact integer Gram per slice
        assert np.array_equal(K, K.T)
        g.close()


_IN_KERNEL_EXPANSION_RUN = """
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import bigsnpr_b200 as B

out = {}
pos = 1000.0 * np.arange(1, 1001)
for na in (0.0, 0.005):
    g = B.Bed.synthetic(20_000, 1_000, seed=31, na_rate=na, ld_rho=0.9, ld_block=50)
    out["cor_%g" % na] = B.bed_cor(g, size=500, thr_r2=0.0, infos_pos=pos)
    g.close()
for na in (0.0, 0.01):
    g = B.Bed.synthetic(3_000, 10_000, seed=41, na_rate=na)
    out["grm_%g" % na] = B.bed_tcrossprodSelf(g)[0]
    g.close()
np.savez(sys.argv[2], **{k + "_%d" % j: v for k, vs in out.items() for j, v in enumerate(vs if isinstance(vs, tuple) else (vs,))})
"""


def test_in_kernel_expansion_gram_tiles_vs_oracle(B, oracle, tmp_path):
    """The Gram kernels that expand the 2-bit codes inside the tile (bsg_gram5.cu: k_gram5, k_wgram5) serve bed_cor when
    the expanded operand planes do not fit in HBM and the GRM with more than four weight digits.  BSG_GRAM_TMA=0 selects
    them for the whole process (the switch is read once), hence the subprocess: windowed correlations with and without
    missing values (missing-free tiles and six-plane tiles) and the weighted GRM, against the oracle."""
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = tmp_path / "gram5.npz"
    r = subprocess.run([sys.executable, "-c", _IN_KERNEL_EXPANSION_RUN, root, str(res)], capture_output=True, text=True,
                       env=dict(os.environ, BSG_GRAM_TMA="0"), timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = np.load(res)
    nt = oracle.max_threads()
    pos = 1000.0 * np.arange(1, 1001)
    for na in (0.0, 0.005):
        o = oracle.synth_bed(20_000, 1_000, seed=31, na_rate=na, ld_rho=0.9, ld_block=50)
        p0, i0, x0 = oracle.cor0(o, size=500, thr_r2=0.0, infos_pos=pos, ncores=nt)
        key = "cor_%g" % na
        assert np.array_equal(got[key + "_0"], p0) and np.array_equal(got[key + "_1"], i0)
        assert np.array_equal(got[key + "_2"], x0, equal_nan=True)
    for na in (0.0, 0.01):
        o = oracle.synth_bed(3_000, 10_000, seed=41, na_rate=na)
        K0 = oracle.bed_tcrossprodSelf(o, block_size=2000)[0]
        K = got["grm_%g_0" % na]
        assert np.max(np.abs(K - K0)) / np.max(np.abs(K0)) < 1e-8
        assert np.array_equal(K, K.T)


def test_products_on_the_default_stream_are_ordered(B):
    """ADVICE r1 (high): a NULL stream means the legacy default stream.  The product is enqueued between two torch
    operations on torch's default stream with no synchronisation in between; repeated with fresh inputs it must always see
    the input written just before and be seen by the reduction enqueued just after."""
    import torch

    n, m = 20_000, 40_000
    g = B.Bed.synthetic(n, m, seed=3)
    sc = B.bed_scaleBinom(g)
    v = B.View(g, center=sc["center"], scale=sc["scale"])
    dev = torch.device("cuda", 0)
    base = torch.randn(m, dtype=torch.float64, device=dev)
    ref_out = torch.empty(n, dtype=torch.float64, device=dev)
    v.prodvec_dev(base.data_ptr(), ref_out.data_ptr(), 0)
    torch.cuda.synchronize()
    want = float(ref_out.sum())
    x = torch.zeros(m, dtype=torch.float64, device=dev)
    out = torch.zeros(n, dtype=torch.float64, device=dev)
    for it in range(30):
        big = torch.randn(8_000_000, device=dev).sum()  # keeps the default stream busy before the input is written
        x.copy_(base * (it + 1))                       # produced on torch's default stream ...
        v.prodvec_dev(x.data_ptr(), out.data_ptr(), 0)  # ... consumed by the library on stream NULL
        s = out.sum() / (it + 1)                        # ... and reduced by torch right after
        out.zero_()
        assert abs(float(s) - want) <= 1e-9 * abs(want) + 1e-6, it
        del big
    v.close()
    g.close()
