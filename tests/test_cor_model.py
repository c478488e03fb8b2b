"""tests/cor_ref.py (the exact model of the windowed pair band) against the CPU oracle, no GPU needed.

The oracle is built with -ffp-contract=off and accumulates exact integer sums, so r is held to the oracle's bytes; LD
scores to a few ulps (the oracle adds the pairs in another order); the clumping sweep over the model's conflict flags to
the oracle's keep vectors.  The tiling metadata (batches, tile modes) is checked on cases small enough to count by hand.
"""
import os

import numpy as np
import pytest

from tests import cor_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _sel(oracle, o, ir, ic):
    return oracle.read_bed(o, ir, ic, na_val=3).astype(np.uint8)


def _model_cor0(G, size=500, alpha=1.0, thr_r2=0.0, fill_diag=True, infos_pos=None):
    from oracle import ref

    thr = ref.cor_thresholds(G.shape[0], alpha, thr_r2)
    return R.bed_cor(G, size * 1000.0, thr, infos_pos, fill_diag)


def _same_csc(a, b):
    return (np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
            and np.array_equal(a[2].view(np.int64), b[2].view(np.int64)))


@pytest.fixture(scope="module")
def small(oracle):
    rng = np.random.default_rng(7)
    G = rng.integers(0, 4, size=(500, 100)).astype(np.uint8)
    return oracle.OracleFBM(G), G


def test_r_bytes_on_the_fixtures(oracle, obed, obed_na, rng):
    nt = oracle.max_threads()
    for o in (obed, obed_na):
        ir, ic = o.rows_along(), o.cols_along()
        G = _sel(oracle, o, ir, ic)
        for kw in (dict(size=50), dict(size=200, alpha=0.05, fill_diag=False), dict(size=100, thr_r2=0.2)):
            want = oracle.cor0(o, ir, ic, ncores=nt, **kw)
            assert _same_csc(_model_cor0(G, **kw), want), kw
        # multisets of rows and columns (sorted columns keep the positions sorted), irregular positions with ties
        ir2 = rng.integers(1, o.nrow + 1, size=o.nrow // 2).astype(np.int32)
        ic2 = np.sort(rng.integers(1, o.ncol + 1, size=300)).astype(np.int32)
        pos = np.cumsum(rng.choice([0.0, 0.5, 1.25, 7.0], size=ic2.size))
        for kw in (dict(size=5e-3, infos_pos=pos), dict(size=0.0, infos_pos=pos, alpha=0.05, thr_r2=0.02)):
            want = oracle.cor0(o, ir2, ic2, ncores=nt, **kw)
            assert _same_csc(_model_cor0(_sel(oracle, o, ir2, ic2), **kw), want), kw


def test_r_bytes_on_random_matrices(oracle, small, rng):
    o, G = small
    for kw in (dict(size=30), dict(size=30, alpha=0.07, fill_diag=False), dict(size=5, thr_r2=0.02),
               dict(size=1e4, alpha=0.3)):
        ir = rng.choice(500, 250, replace=False) + 1
        ic = np.sort(rng.choice(100, 50, replace=False)) + 1
        want = oracle.cor0(o, ir, ic, **kw)
        assert _same_csc(_model_cor0(G[ir - 1][:, ic - 1], **kw), want), kw
    # constant, all-missing, single-valued, identical and negated columns: NaN r, deno 0 and the clamp at +-1
    H = rng.integers(0, 3, size=(40, 12)).astype(np.uint8)
    H[:, 1] = 1
    H[:, 2] = 3
    H[:, 3] = 3
    H[5, 3] = 2
    H[:, 5] = H[:, 4]
    H[:, 6] = 2 - H[:, 4]
    H[-1, 8] = 3
    want = oracle.cor0(oracle.OracleFBM(H), size=1e4)
    got = _model_cor0(H, size=1e4)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert np.array_equal(got[2], want[2], equal_nan=True) and np.isnan(got[2]).any()
    col = np.repeat(np.arange(H.shape[1]), np.diff(got[0]))
    assert got[2][(col == 5) & (got[1] == 4)] == 1.0 and got[2][(col == 6) & (got[1] == 4)] == -1.0


def test_ld_scores_within_ulps(oracle, obed_na, small):
    o, G = small
    for obj, Gs in ((o, G), (obed_na, _sel(oracle, obed_na, obed_na.rows_along(), obed_na.cols_along()))):
        for size in (3, 37, 1e4):
            want = oracle.ld0(obj, size=size, ncores=1)
            got = R.ld_scores(Gs, size * 1000.0)
            np.testing.assert_allclose(got, want, rtol=8 * np.finfo(float).eps, atol=0)


def _bed_clump_chr(oracle):
    def f(obj, ind_row, ind_col, center, scale, ordv, rank, pos, size, thr):
        G = _sel(oracle, obj, ind_row, ind_col)
        band = R.Band(pos, size, both=True)
        flag = R.clump_epilogue(R.pair_sums(G, band), center, scale, thr)
        return R.clump_sweep(band, flag, pos, size, ordv)

    return f


def test_clumping_sweep_over_model_flags(oracle, obed, obed_na):
    f = _bed_clump_chr(oracle)
    for o in (obed, obed_na):
        chrom = np.ones(o.ncol, dtype=int)
        for kw in (dict(thr_r2=0.2, size=100), dict(thr_r2=0.05, size=20), dict(thr_r2=0.5, size=500)):
            pos = 1000.0 * np.arange(1, o.ncol + 1)
            want = oracle.bed_clumping(o, infos_chr=chrom, infos_pos=pos, **kw)
            got = oracle.bed_clumping(o, infos_chr=chrom, infos_pos=pos, clump_chr=f, **kw)
            assert np.array_equal(got, want) and 0 < got.size < o.ncol, kw


def test_levels_sweep_over_model_flags(oracle, obed, rng):
    ir = rng.choice(obed.nrow, 300, replace=False) + 1
    G = _sel(oracle, obed, obed.rows_along(), obed.cols_along())
    G[rng.integers(0, G.shape[0], 50), rng.integers(0, G.shape[1], 50)] = 3  # missing values: level 0 by rule
    fbm = oracle.OracleFBM(G)

    def f(Gf, rowInd, colInd, ordv, rank, pos, sumX, denoX, size, thr):
        Gs = G[np.asarray(rowInd) - 1][:, np.asarray(colInd) - 1]
        band = R.Band(pos, size, both=True)
        S = R.pair_sums(Gs, band)
        lev = R.levels_epilogue(S, Gs.shape[0], sumX, denoX, [thr], (Gs == 3).any(axis=0))
        return R.clump_sweep(band, lev > 0, pos, size, ordv)

    chrom = np.ones(G.shape[1], dtype=int)
    for kw in (dict(thr_r2=0.2, size=50), dict(thr_r2=0.05, size=10, ind_row=ir)):
        want = oracle.snp_clumping(fbm, chrom, **kw)
        got = oracle.snp_clumping(fbm, chrom, clump_chr=f, **kw)
        assert np.array_equal(got, want) and 0 < got.size < G.shape[1], kw


def test_window_rules():
    pos = np.array([1.0, 2.0, 2.0, 3.0, 10.0, 11.0, 11.5])
    b = R.Band(pos, 1.0)
    assert b.wlen.tolist() == [0, 1, 2, 2, 0, 1, 1] and b.reach.tolist() == [2, 3, 3, 3, 5, 6, 6]
    assert b.boff.tolist() == [0, 0, 1, 3, 5, 5, 6, 7]
    assert R.Band(pos, 0.0).wlen.tolist() == [0, 0, 1, 0, 0, 0, 0]  # ties pair up at size 0
    # the `both` rule: pos[j0] - size rounds below pos[j] while pos[j] + size rounds to pos[j0]
    p2 = np.array([0.1, 0.1 + 0.2])
    s = 0.2
    assert not p2[0] >= p2[1] - s and p2[1] <= p2[0] + s
    assert R.Band(p2, s).wlen.tolist() == [0, 0] and R.Band(p2, s, both=True).wlen.tolist() == [0, 1]


def test_batch_plan_hand_counted():
    T = R.TM * R.CTN
    # 1,024 columns, one-SNP window: row block ib holds tiles (ib - 1, ib) (block 0: one tile)
    nc = 1024
    band = R.Band(np.arange(nc, dtype=float), 1.0)
    na = np.zeros(nc, dtype=bool)
    na[[5, 300]] = True  # column blocks 0 and 2 hold a missing value
    plan = R.Plan(na, band)
    assert plan.nbatches == 1 and plan.ntiles.tolist() == [1] + [2] * 7
    tiles = plan.batches[0][2]
    assert [(ib, jb, md) for ib, jb, md in tiles[:5]] == [(0, 0, 1), (1, 0, 1), (1, 1, 0), (2, 1, 1), (2, 2, 1)]
    assert plan.batches[0][3] == T * (6 + 6 + 1 + 6 + 6 + 6 + 1 + 2 * 4)
    # row pair (2, 3) over column block 2: block 2 is mode 1 (missing), block 3 sees block 2 with mode 1 -> not mixed;
    # pair (0, 1) over column block 0: both halves mode 1; pair (0, 1) over block 1: only half 1 -> not a pair
    assert (0, 1, 2) not in plan.mixed_pairs()
    na2 = np.zeros(nc, dtype=bool)
    na2[128 * 3] = True  # only column block 3: pair (2, 3) over block 2 has half 2 mode 0 and half 3 mode 1
    assert (0, 1, 2) in R.Plan(na2, band).mixed_pairs()
    # a bound of 20 tile units, missing values everywhere: row blocks 0 (6 units) and 1 (12) share a batch, then one each
    small = R.Plan(np.ones(nc, dtype=bool), band, max_sum_ints=20 * T)
    assert [b[:2] for b in small.batches] == [(0, 2), (2, 3), (3, 4), (4, 5), (5, 6), (6, 7), (7, 8)]
    assert small.split_pairs() == [3, 5, 7]
    # a row block needing more than the bound still runs, alone; a row block without pairs joins the open batch
    gaps = R.Band(np.r_[np.arange(200.0), 1e6 + 1e3 * np.arange(300), 2e6 + np.arange(100)], 500.0)
    plan = R.Plan(np.ones(600, dtype=bool), gaps, max_sum_ints=T)
    assert plan.ntiles.tolist() == [1, 2, 0, 1, 2]
    assert [b[:2] for b in plan.batches] == [(0, 1), (1, 3), (3, 4), (4, 5)]
