"""snp_PRS / snp_grid_PRS on the device (bsg_prs_grid) against the exact model of tests/prs_ref.py, byte for byte, and
against R's literal loop within the fixed-point bound; non-finite weights, the column layout and the ABI errors."""
import ctypes as C
import os

import numpy as np
import pytest

import bigsnpr_b200 as B
from bigsnpr_b200 import _lib
from tests import prs_ref as P
from tests.test_prs_oracle import bound

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def twin(G):
    """FBM.code256 twin of a code matrix (NA code 3 -> byte 3, code256[3] = NA), as snp_readBed2 makes it."""
    return B.Bed.from_fbm(np.asarray(G, dtype=np.uint8))


@pytest.fixture(scope="module", params=["example.bed", "example-missing.bed"])
def example(request):
    g = B.Bed(os.path.join(GOLD, request.param), device=0)
    G = B.read_bed(g, g.rows_along(), g.cols_along(), na_val=3)
    return g, twin(G), G


def grid_call(h, ind_row, sets, beta, same, lpS, thr, out_double=True):
    """bsg_prs_grid with per-entry arrays (sets concatenated)."""
    ncol = len(sets) * (1 if thr is None else len(thr))
    out = np.zeros((len(ind_row), ncol), dtype=np.float64 if out_double else np.float32, order="F")
    B.api._prs_call(h, np.asarray(ind_row, dtype=np.int32), sets, beta, same, lpS, thr, out)
    return out


def model(G, ind_row, sets, beta, same, lpS, thr, fn=P.exact):
    cols, o = [], 0
    for s in sets:
        sl = slice(o, o + len(s))
        cols.append(fn(G, ind_row, s, beta[sl], None if same is None else same[sl].astype(bool),
                       None if lpS is None else lpS[sl], thr))
        o += len(s)
    return np.concatenate(cols, axis=1)


def check_same(got, want):
    assert got.shape == want.shape
    assert np.array_equal(got, want, equal_nan=True), np.nanmax(np.abs(got - want))


def test_example_bit_identical(example):
    g, f, G = example
    rng = np.random.default_rng(5)
    n, m = G.shape
    ir = np.concatenate([rng.integers(1, n + 1, 300), [1, 1, 2]])
    sets = [rng.choice(m, 700, replace=True) + 1, rng.choice(m, 33, replace=False) + 1, np.zeros(0, np.int64),
            np.arange(1, m + 1)]
    L = sum(len(s) for s in sets)
    beta = rng.normal(size=L) * 10.0 ** rng.integers(-4, 1, size=L)
    same = (rng.random(L) < 0.6).astype(np.int32)
    lpS = rng.exponential(2.0, size=L)
    lpS[:5] = 1.5  # equal to a threshold: strict >
    thr = np.array([1.5, 0.0, 3.0, 1.5, 7.0, 0.5, 100.0])
    want = model(G, ir, sets, beta, same, lpS, thr)
    for h in (g, f):
        check_same(grid_call(h, ir, sets, beta, same, lpS, thr), want)
        check_same(grid_call(h, ir, sets, beta, same, lpS, thr, out_double=False), want.astype(np.float32))
    # thresholding disabled
    check_same(grid_call(f, ir, sets, beta, same, None, None), model(G, ir, sets, beta, same, None, None))
    # within the fixed-point bound of R's loop
    lit = model(G, ir, sets[:2], beta[:733], same[:733], lpS[:733], thr, fn=P.literal)
    got = grid_call(f, ir, sets[:2], beta[:733], same[:733], lpS[:733], thr)
    assert np.array_equal(np.isnan(lit), np.isnan(got))
    tol = max(bound(G, ir, sets[0], beta[:700], same[:700].astype(bool)).max(),
              bound(G, ir, sets[1], beta[700:733], same[700:733].astype(bool)).max()) + 1e-13 * np.nanmax(np.abs(lit))
    assert np.nanmax(np.abs(got - lit)) <= tol


@pytest.mark.parametrize("na_rate", [0.01, 0.10])
def test_grid_clumping_sets_and_na_rates(na_rate):
    """A synthetic LD chromosome, its snp_grid_clumping keep sets, 50 thresholds; NA rates below and above the 4 % cut
    of the missing-value lists."""
    rng = np.random.default_rng(7)
    s = B.Bed.synthetic(1200, 3000, seed=3, na_rate=na_rate, ld_rho=0.9, ld_block=50)
    G = B.read_bed(s, s.rows_along(), s.cols_along(), na_val=3)
    s.close()
    f = twin(G)
    lpS = -np.log10(rng.uniform(size=G.shape[1])) * 3
    betas = rng.normal(size=G.shape[1]) * 0.01
    pos = np.arange(1, G.shape[1] + 1) * 100.0
    keep = B.snp_grid_clumping(f, np.ones(G.shape[1], dtype=int), pos, lpS, grid_base_size=(50, 200))
    res = B.snp_grid_PRS(f, keep, betas, lpS, type="double")
    thr = res.grid_lpS_thr
    assert thr.size == 50 and res.shape == (1200, len(keep[0]) * 50)
    want = P.grid(G, np.arange(1, 1201), keep, betas, lpS, thr)
    check_same(np.asarray(res), want)
    assert np.isnan(want).any()
    assert res.all_keep is keep and res.betas is not None and res.lpS is not None


def test_long_set_over_int32_cap():
    """70,000 entries in one step: the int32 accumulators are drained into int64 totals on the way."""
    g = B.Bed(os.path.join(GOLD, "example-missing.bed"), device=0)
    G = B.read_bed(g, g.rows_along(), g.cols_along(), na_val=3)
    rng = np.random.default_rng(9)
    cols = rng.integers(1, G.shape[1] + 1, 70000)
    beta = rng.normal(size=cols.size)
    lpS = rng.exponential(1.0, size=cols.size)
    thr = np.array([0.5, 0.0, 2.0])
    ir = np.arange(1, G.shape[0] + 1)
    check_same(grid_call(g, ir, [cols], beta, None, lpS, thr), model(G, ir, [cols], beta, None, lpS, thr))


def test_nonfinite_beta_is_the_literal_loop(example):
    g, f, G = example
    rng = np.random.default_rng(4)
    cols = rng.integers(1, G.shape[1] + 1, 300)
    beta = rng.normal(size=300)
    beta[17] = np.inf
    lpS = rng.exponential(1.0, size=300)
    lpS[17] = 0.8
    thr = np.array([2.0, 0.5, 1.0, 0.0])
    ir = np.arange(1, G.shape[0] + 1)
    got = grid_call(f, ir, [cols, cols[100:150]], np.concatenate([beta, beta[100:150]]), None,
                    np.concatenate([lpS, lpS[100:150]]), thr)
    lit = P.literal(G, ir, cols, beta, None, lpS, thr)
    np.testing.assert_allclose(got[:, :4], lit, rtol=1e-12, atol=1e-12)
    assert np.array_equal(np.isnan(got[:, :4]), np.isnan(lit))
    check_same(got[:, 4:], P.exact(G, ir, cols[100:150], beta[100:150], None, lpS[100:150], thr))


def test_snp_PRS_and_grid_layout(example, tmp_path, capsys):
    g, f, G = example
    rng = np.random.default_rng(8)
    keep = np.sort(rng.choice(G.shape[1], 500, replace=False)) + 1
    beta = rng.normal(size=500)
    same = rng.random(500) < 0.5
    s0 = B.snp_PRS(f, beta, ind_keep=keep, same_keep=same)
    assert "Thresholding disabled" in capsys.readouterr().err and s0.shape == (G.shape[0], 1)
    lpS = rng.exponential(1.0, size=500)
    thr = np.array([0.0, 1.0, 0.5])
    s1 = B.snp_PRS(f, beta, ind_keep=keep, same_keep=same, lpS_keep=lpS, thr_list=thr)
    assert np.array_equal(s1.thr_list, thr)
    check_same(np.asarray(s1), P.exact(G, np.arange(1, G.shape[0] + 1), keep, beta, same, lpS, thr))
    # grid: chromosome-major sets, column (ic - 1) n_thr + t; float by default; disk-backed
    m = G.shape[1]
    betas, lpS_all = rng.normal(size=m), rng.exponential(1.0, size=m)
    all_keep = [[keep[:100], keep[100:300]], [keep[300:]]]
    ir = np.array([3, 1, 3, 10])
    res = B.snp_grid_PRS(f, all_keep, betas, lpS_all, n_thr_lpS=5, ind_row=ir, backingfile=str(tmp_path / "grid"))
    assert res.dtype == np.float32 and res.shape == (4, 15) and os.path.exists(str(tmp_path / "grid.bk"))
    want = P.grid(G, ir, all_keep, betas, lpS_all, res.grid_lpS_thr)
    check_same(np.asarray(res), want.astype(np.float32))
    want_thr = 0.9999 * B.seq_log(max(0.1, lpS_all.min()), lpS_all.max(), 5)
    assert np.array_equal(res.grid_lpS_thr, want_thr)


def test_abi_errors(example):
    g, f, G = example
    L = _lib.lib()
    one = np.array([1], dtype=np.int32)
    b = np.array([1.0])
    out = np.zeros(64)
    pi = lambda a: a.ctypes.data_as(_lib.c_int_p)  # noqa: E731
    pd = lambda a: a.ctypes.data_as(_lib.c_dbl_p)  # noqa: E731
    optr = C.c_void_p(out.ctypes.data)
    # thr NULL with nthr != 1, a negative set length, a negative lpS, a column out of range
    assert L.bsg_prs_grid(f._h, None, 0, 1, pi(one), pi(one), pd(b), None, pd(b), 2, None, 1, optr) == 9
    assert L.bsg_prs_grid(f._h, None, 0, 1, pi(np.array([-1], np.int32)), pi(one), pd(b), None, pd(b), 1, None, 1,
                          optr) == 9
    assert L.bsg_prs_grid(f._h, pi(one), 1, 1, pi(one), pi(one), pd(b), None, pd(np.array([-1.0])), 1, pd(b), 1, optr) == 9
    assert L.bsg_prs_grid(f._h, pi(one), 1, 1, pi(one), pi(np.array([G.shape[1] + 1], np.int32)), pd(b), None, pd(b), 1,
                          pd(b), 1, optr) == 2
    # a row out of range
    assert L.bsg_prs_grid(f._h, pi(np.array([G.shape[0] + 1], np.int32)), 1, 1, pi(one), pi(one), pd(b), None, None, 1,
                          None, 1, optr) == 2
    # a generic table (codes that are not multiples of 1 / D)
    code = np.full(256, np.nan)
    code[:201] = np.sqrt(np.arange(201))
    d = B.Bed.from_fbm(np.asarray(G % 3 * 50, dtype=np.uint8), code256=code)
    assert d.dosage_scale == 0
    assert L.bsg_prs_grid(d._h, pi(one), 1, 1, pi(one), pi(one), pd(b), None, None, 1, None, 1, optr) == 10
    # scratch larger than the device from the sizes alone: 40,000 columns of 1,000,000 samples
    s = B.Bed.synthetic(1_000_000, 2, seed=1)
    thr = np.linspace(0, 1, 40000)
    assert L.bsg_prs_grid(s._h, pi(one), 1, 1, pi(one), pi(one), pd(b), None, pd(b), thr.size, pd(thr), 1, optr) == 7
    assert "bytes of device memory" in L.bsg_last_error().decode()


CODE_DOSAGE = np.concatenate([[0, 1, 2, np.nan, 0, 1, 2], np.arange(201) * 0.01, np.full(48, np.nan)])


def dosage_matrix(rng, n, m, na_rate):
    """Raw bytes of a CODE_DOSAGE FBM.code256 (bytes 7 .. 207 = dosages 0 .. 2, a few hard-call codes 0 .. 2, NA as
    byte 3 and as bytes above 207) and the handle, D = 100."""
    raw = rng.integers(7, 208, size=(n, m)).astype(np.uint8)
    raw[rng.random((n, m)) < 0.05] = rng.integers(0, 3, dtype=np.uint8)
    na = rng.random((n, m)) < na_rate
    raw[na] = np.where(rng.random(int(na.sum())) < 0.5, 3, 230).astype(np.uint8)
    h = B.Bed.from_fbm(np.asfortranarray(raw), code256=CODE_DOSAGE)
    assert h.dosage_scale == 100
    return raw, h


@pytest.mark.parametrize("na_rate", [0.0, 0.01, 0.10])
def test_dosage_bit_identical(na_rate):
    rng = np.random.default_rng(11)
    raw, h = dosage_matrix(rng, 700, 900, na_rate)
    V, NA = P.dosage_bytes(raw, CODE_DOSAGE, 100)
    ir = np.concatenate([rng.integers(1, 701, 400), [5, 5]])
    sets = [rng.choice(900, 1200, replace=True) + 1, rng.choice(900, 40, replace=False) + 1, np.arange(1, 901)]
    L = sum(len(x) for x in sets)
    beta = rng.normal(size=L) * 10.0 ** rng.integers(-3, 1, size=L)
    same = (rng.random(L) < 0.6).astype(np.int32)
    lpS = rng.exponential(2.0, size=L)
    thr = np.array([1.0, 0.0, 3.0, 1.0, 6.0])
    want = model(V, ir, sets, beta, same, lpS, thr, fn=lambda *a: P.exact(*a, D=100, na_mask=NA))
    check_same(grid_call(h, ir, sets, beta, same, lpS, thr), want)
    check_same(grid_call(h, ir, sets, beta, same, lpS, thr, out_double=False), want.astype(np.float32))
    assert np.isnan(want).any() == (na_rate > 0)
    # within the bound of R's loop on the codes (NA codes as NaN)
    X = CODE_DOSAGE[raw]
    lit = P.literal(np.where(np.isnan(X), 3, X), ir, sets[1], beta[1200:1240], same[1200:1240], lpS[1200:1240], thr)
    got = grid_call(h, ir, sets[1:2], beta[1200:1240], same[1200:1240], lpS[1200:1240], thr)
    assert np.array_equal(np.isnan(lit), np.isnan(got))
    assert np.nanmax(np.abs(got - lit)) <= 1e-12 * max(1.0, np.nanmax(np.abs(lit)))
    # a non-finite beta: R's loop on the codes
    b2 = beta[1200:1240].copy()
    b2[3] = -np.inf
    got = grid_call(h, ir, sets[1:2], b2, None, lpS[1200:1240], thr)
    lit = P.literal(np.where(np.isnan(X), 3, X), ir, sets[1], b2, None, lpS[1200:1240], thr)
    np.testing.assert_allclose(got, lit, rtol=1e-12, atol=1e-12)


def test_several_blocks_and_long_sets():
    """n = 5,000 (3 blocks of 2,048 samples, the last partial, its last four warps past the line stride) with sets longer
    than 65,536 lines: the per-block drain buffers, the stride clamp of the last block and the gather across blocks, on
    hard calls and on dosages."""
    rng = np.random.default_rng(12)
    n, m = 5000, 300
    s = B.Bed.synthetic(n, m, seed=9, na_rate=0.002)
    G = B.read_bed(s, s.rows_along(), s.cols_along(), na_val=3)
    ir = np.concatenate([np.arange(1, n + 1), [n, 1, 2049, 4097]])
    sets = [rng.integers(1, m + 1, 70000), rng.integers(1, m + 1, 500), rng.integers(1, m + 1, 66000)]
    L = sum(len(x) for x in sets)
    beta = rng.normal(size=L)
    same = (rng.random(L) < 0.8).astype(np.int32)
    lpS = rng.exponential(1.0, size=L)
    thr = np.array([0.2, 1.5, 0.0])
    want = model(G, ir, sets, beta, same, lpS, thr)
    for h in (s, twin(G)):
        check_same(grid_call(h, ir, sets, beta, same, lpS, thr), want)
    raw, hd = dosage_matrix(rng, n, m, 0.002)
    V, NA = P.dosage_bytes(raw, CODE_DOSAGE, 100)
    want = model(V, ir, sets, beta, same, lpS, thr, fn=lambda *a: P.exact(*a, D=100, na_mask=NA))
    check_same(grid_call(hd, ir, sets, beta, same, lpS, thr), want)


def test_reference_scores_on_device(obed, oracle):
    """R's snp_PRS output (tests/golden/prs_scores.npz), thresholds 1.5 .. 5, from the recovered betas on the FBM twin of
    example.bed, through snp_PRS with the thresholds in the reference's order and shuffled."""
    from tests.test_prs_oracle import reference_fixture

    G = oracle.decode_dense(obed)
    keep, lpS, beta, scores, thr, _, _ = reference_fixture(G)
    f = twin(G)
    got = np.asarray(B.snp_PRS(f, beta, ind_keep=keep, lpS_keep=lpS, thr_list=thr))
    assert np.max(np.abs(got[:, 3:] - scores[:, 3:])) <= 1e-12
    check_same(got, P.exact(G, np.arange(1, G.shape[0] + 1), keep, beta, None, lpS, thr))
    perm = np.random.default_rng(1).permutation(thr.size)
    check_same(np.asarray(B.snp_PRS(f, beta, ind_keep=keep, lpS_keep=lpS, thr_list=thr[perm])), got[:, perm])


def test_grid_threshold_zero_disables_thresholding(example):
    g, f, G = example
    rng = np.random.default_rng(13)
    m = G.shape[1]
    betas, lpS = rng.normal(size=m), rng.exponential(1.0, size=m)
    lpS[:3] = np.nan  # not read when thresholding is disabled
    all_keep = [[np.arange(4, 60), np.arange(100, 300)]]
    res = B.snp_grid_PRS(f, all_keep, betas, lpS, grid_lpS_thr=0, type="double")
    want = P.grid(G, np.arange(1, G.shape[0] + 1), all_keep, betas, lpS, None)
    check_same(np.asarray(res), want)
    with pytest.raises(IndexError):
        B.snp_grid_PRS(f, [[np.arange(1, 5)], [np.array([m + 1])]], betas, np.abs(np.nan_to_num(lpS)), n_thr_lpS=3)
