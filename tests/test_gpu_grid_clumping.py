"""snp_grid_clumping on the device (bsg_grid_clumping_chr) against the CPU oracle of R/SCT.R + clumping_chr_cached
(tests/grid_ref.py): identical keep lists on hard calls, missing calls, mean2-imputed and raw dosages and an LD-structured
slice; exact integer dosage pair sums past the int32 span; the R shim's _bigsnpr_clumping_chr_cached; edge cases."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import grid_ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
# CODE_DOSAGE: 0, 1, 2, NA, 0, 1, 2, seq(0, 2, by = 0.01), NA x 48
CODE_DOSAGE = np.concatenate([[0, 1, 2, np.nan, 0, 1, 2], 0 + np.arange(201) * 0.01, np.full(48, np.nan)])


@pytest.fixture(scope="module")
def B():
    import bigsnpr_b200 as b
    from bigsnpr_b200 import build

    build.build()
    return b


def _bim_pos(name):
    return np.array([float(ln.split()[3]) for ln in open(os.path.join(GOLDEN, name + ".bim"))])


@pytest.fixture(scope="module")
def ex(oracle):
    G = oracle.decode_dense(oracle.OracleBed(os.path.join(GOLDEN, "example.bed"))).astype(np.uint8)
    chr_ = np.repeat([1, 2], [2542, 2000])
    return G, chr_, _bim_pos("example"), -np.log10(np.random.default_rng(6).uniform(size=G.shape[1]))


def _same(got, want):
    want_lists, want_grid = want
    assert len(got) == len(want_lists)
    for a, b in zip(got, want_lists):
        assert len(a) == len(b)
        for i, (x, y) in enumerate(zip(a, b)):
            assert np.array_equal(x, y), (i, x.size, y.size)
    for k, v in want_grid.items():
        assert np.array_equal(got.grid[k], v), k


def _both(B, oracle, G, code256, *args, **kw):
    g = B.Bed.from_fbm(G, code256=code256)
    o = oracle.OracleFBM(G, code256)
    got = B.snp_grid_clumping(g, *args, **kw)
    want = grid_ref.snp_grid_clumping(o, *args, **kw)
    _same(got, want)
    return got, g


def test_example_default_grid(B, oracle, ex):
    G, chr_, pos, lp = ex
    got, g = _both(B, oracle, G, None, chr_, pos, lp)
    assert len(got) == 2 and len(got[0]) == 28 and len(got.grid["size"]) == 28
    sizes = {len(k) for k in got[0]}
    assert len(sizes) > 5 and min(sizes) > 0  # the grid points prune differently
    # hard calls: each grid point is bit for bit a separate clumping_chr call (bsg_clumping_chr_fbm)
    ind_chr = np.arange(1, 2543, dtype=np.int32)
    ir = g.rows_along()
    st = B.snp_colstats(g, ir, ind_chr)
    ordv = (grid_ref._order_decreasing(lp[:2542])).astype(np.int32)
    for i in (0, 5, 13, 27):
        thr, base = got.grid["thr_r2"][i], np.unique([50, 100, 200, 500])[i % 4]
        keep = B.clumping_chr(g, ir, ind_chr, ordv, None, pos[:2542], st["sumX"], st["denoX"], 1000 * base / thr, thr)
        assert np.array_equal(ind_chr[keep == 1], got[0][i]), i


def test_example_imputation_and_groups(B, oracle, ex):
    G, chr_, pos, lp = ex
    infos = np.random.default_rng(7).uniform(0.2, 1.0, size=G.shape[1])
    kw = dict(grid_thr_r2=(0.05, 0.2, 0.8), grid_base_size=(100, 200))
    k3, _ = _both(B, oracle, G, None, chr_, pos, lp, infos_imp=infos, grid_thr_imp=(0.3, 0.8, 0.95), **kw)
    groups = [np.flatnonzero(infos >= t) + 1 for t in (0.3, 0.8, 0.95)]
    k4, _ = _both(B, oracle, G, None, chr_, pos, lp, groups=groups, **kw)
    for a, b in zip(k3, k4):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    k5, _ = _both(B, oracle, G, None, chr_, pos, lp, groups=[[], [1], np.arange(1, G.shape[1] + 1)], exclude=[3, 4000],
                  **kw)
    assert all(k.size == 0 for k in k5[0][:6]) and all(k.tolist() == [1] for k in k5[0][6:12])


def test_example_missing_na_rule(B, oracle):
    G = oracle.decode_dense(oracle.OracleBed(os.path.join(GOLDEN, "example-missing.bed"))).astype(np.uint8)
    assert (G == 3).any()
    m = G.shape[1]
    lp = -np.log10(np.random.default_rng(3).uniform(size=m))
    _both(B, oracle, G, None, np.repeat([1, 2], [m // 2, m - m // 2]), _bim_pos("example-missing"), lp)


def _mean2(G):
    """method "mean2" of snp_fastImputeSimple: a missing call becomes the column mean rounded to 2 decimals (CODE_DOSAGE
    code 7 + 100 * value)."""
    G = G.astype(np.uint8).copy()
    for j in range(G.shape[1]):
        na = G[:, j] == 3
        if na.any():
            G[na, j] = 7 + int(np.rint(100 * (G[~na, j].mean() if (~na).any() else 0.0)))
    return G


def test_dosage_mean2_imputed(B, oracle):
    G = _mean2(oracle.decode_dense(oracle.OracleBed(os.path.join(GOLDEN, "example-missing.bed"))))
    m = G.shape[1]
    lp = -np.log10(np.random.default_rng(4).uniform(size=m))
    got, g = _both(B, oracle, G, CODE_DOSAGE, np.repeat([1, 2], [m // 2, m - m // 2]), _bim_pos("example-missing"), lp,
                   grid_base_size=(50, 500))
    assert g.dosage_scale == 100


def test_dosage_raw_with_na_codes(B, oracle):
    rng = np.random.default_rng(5)
    n, m = 700, 900
    lat = rng.normal(size=(n, m // 30))
    prob = 1 / (1 + np.exp(-(1.2 * lat[:, np.arange(m) // 30] + 0.5 * rng.normal(size=(n, m)))))
    G = (7 + np.clip(np.rint(200 * prob), 0, 200)).astype(np.uint8)
    G[rng.random(size=(n, m)) < 0.002] = 3  # NA code: its columns never prune (NaN r2)
    pos = np.sort(rng.uniform(0, 3e7, size=m)).round()
    lp = -np.log10(rng.uniform(size=m))
    ir = np.sort(rng.choice(n, 600, replace=False) + 1)  # rows other than the identity
    _both(B, oracle, G, CODE_DOSAGE, np.ones(m, dtype=int), pos, lp, ind_row=ir, grid_thr_r2=(0.05, 0.2, 0.5),
          grid_base_size=(50, 200), infos_imp=rng.uniform(size=m), grid_thr_imp=(0.2, 0.6))


def test_ld_structured_slice(B, oracle):
    """Windows hold thousands of pairs and the thresholds prune (LD blocks of 50 SNPs)."""
    o = oracle.synth_bed(1200, 3000, seed=11, ld_rho=0.85, ld_block=50)
    G = oracle.decode_dense(o).astype(np.uint8)
    m = G.shape[1]
    pos = np.cumsum(np.random.default_rng(8).integers(1000, 9000, size=m)).astype(np.float64)
    lp = -np.log10(np.random.default_rng(9).uniform(size=m))
    got, _ = _both(B, oracle, G, None, np.repeat([1, 2], [1800, 1200]), pos, lp, grid_thr_r2=(0.01, 0.1, 0.5, 0.9),
                   grid_base_size=(50, 200))
    n_kept = [len(k) for k in got[0]]
    assert min(n_kept) < 1800 // 2 and len(set(n_kept)) > 2


def _call_grid(B, g, ind_row, ind_col, pos, sumX, denoX, subsets, thr, size):
    from bigsnpr_b200 import _lib

    lens = np.array([len(c) for c, _ in subsets], dtype=np.int32)
    cols = np.concatenate([np.asarray(c, dtype=np.int32) for c, _ in subsets] + [np.zeros(0, np.int32)]).astype(np.int32)
    ords = np.concatenate([np.asarray(o, dtype=np.int32) for _, o in subsets] + [np.zeros(0, np.int32)]).astype(np.int32)
    thr, size = np.asarray(thr, dtype=np.float64), np.asarray(size, dtype=np.float64)
    keep = np.full(max(int(lens.sum()) * thr.size, 1), -1, dtype=np.int32)
    ip = lambda a: a.ctypes.data_as(_lib.c_int_p)  # noqa: E731
    dp = lambda a: a.ctypes.data_as(_lib.c_dbl_p)  # noqa: E731
    _lib.check(_lib.lib().bsg_grid_clumping_chr(g._h, ip(ind_row), ind_row.size, ip(ind_col), ind_col.size, dp(pos), dp(sumX),
                                                dp(denoX), len(subsets), ip(lens), ip(cols), ip(ords), thr.size, dp(thr),
                                                dp(size), ip(keep)))
    return keep


def test_dosage_sums_exact_past_int32_span(B):
    """Near-maximal bytes (q up to 255) on 70,000 samples: S reaches 4.5e9, past int32 and past one 32,768-sample span.
    Thresholds a hair (1e-12 relative) either side of the exact r2 (NumPy int64) must fall on the right sides."""
    rng = np.random.default_rng(12)
    n = 70000
    code = np.arange(256) / 100.0  # D = 100, q = byte
    q = np.full((n, 2), 255, dtype=np.uint8)
    q[rng.random(n) < 0.02, 0] = 0
    q[rng.random(n) < 0.02, 1] = 0
    q[rng.random(n) < 0.3, 1] = 254
    g = B.Bed.from_fbm(q, code256=code)
    assert g.dosage_scale == 100
    ir = g.rows_along()
    ic = np.array([1, 2], dtype=np.int32)
    st = B.snp_colstats(g, ir, ic)
    S = int(np.dot(q[:, 0].astype(np.int64), q[:, 1].astype(np.int64)))
    assert S > 2**32
    num = S / 1e4 - st["sumX"][1] * st["sumX"][0] / n
    r2 = num * num / (st["denoX"][1] * st["denoX"][0])
    assert 0 < r2 < 1
    thr = [r2 * (1 - 1e-12), r2 * (1 + 1e-12)]
    keep = _call_grid(B, g, ir, ic, np.array([1.0, 2.0]), st["sumX"], st["denoX"], [([1, 2], [1, 2])], thr, [10.0, 10.0])
    assert keep.tolist() == [1, 0, 1, 1]


def test_edge_cases(B, ex):
    G, chr_, pos, lp = ex
    g = B.Bed.from_fbm(G[:, :300])
    ir = g.rows_along()
    ic = np.arange(1, 301, dtype=np.int32)
    st = B.snp_colstats(g, ir, ic)
    p = pos[:300]
    # an empty subset, a single column, the whole set: one call
    ordv = grid_ref._order_decreasing(lp[:300]).astype(np.int32)
    keep = _call_grid(B, g, ir, ic, p, st["sumX"], st["denoX"], [([], []), ([7], [1]), (ic, ordv)], [0.2], [5e5])
    assert keep[0] == 1 and set(keep[1:].tolist()) <= {0, 1}
    ref = B.clumping_chr(g, ir, ic, ordv, None, p, st["sumX"], st["denoX"], 5e5, 0.2)
    assert np.array_equal(keep[1:], ref)
    # a NaN threshold keeps every variant (r2 > NaN is false)
    assert np.all(B.clumping_chr(g, ir, ic, ordv, None, p, st["sumX"], st["denoX"], 5e5, np.nan) == 1)
    # nc = 0, and no grid point: nothing to do
    e = np.zeros(0, dtype=np.int32)
    _call_grid(B, g, ir, e, np.zeros(0), np.zeros(0), np.zeros(0), [([], [])], [0.2], [5e5])
    _call_grid(B, g, ir, ic, p, st["sumX"], st["denoX"], [(ic, ordv)], [], [])
    from bigsnpr_b200 import BsgError

    with pytest.raises(BsgError, match="ascending"):
        _call_grid(B, g, ir, ic, p, st["sumX"], st["denoX"], [([3, 2], [1, 2])], [0.2], [5e5])
    with pytest.raises(BsgError, match="not sorted"):
        _call_grid(B, g, ir, ic, p[::-1].copy(), st["sumX"], st["denoX"], [([1], [1])], [0.2], [5e5])
    # the priority order must list every position once: a repeated entry is out of bounds in all three entry points
    dup = ordv.copy()
    dup[1] = dup[0]
    with pytest.raises(BsgError, match="out of bounds"):
        _call_grid(B, g, ir, ic, p, st["sumX"], st["denoX"], [(ic, dup)], [0.2], [5e5])
    with pytest.raises(BsgError, match="out of bounds"):
        B.clumping_chr(g, ir, ic, dup, None, p, st["sumX"], st["denoX"], 5e5, 0.2)
    gb = B.Bed(os.path.join(GOLDEN, "example.bed"))
    with pytest.raises(BsgError, match="out of bounds"):
        B.bed_clumping_chr(gb, gb.rows_along(), ic, np.zeros(300), np.ones(300), dup, None, p, 5e5, 0.2)
    gb.close()


def test_shim_clumping_chr_cached(B, oracle, ex, tmp_path_factory):
    """_bigsnpr_clumping_chr_cached through the shim linked against the stand-in for R's C API: registered under the
    reference's name with 14 arguments; called with the objects R/SCT.R passes, keep equals the oracle's and sqcor comes
    back as passed.  The stand-in's .Call dispatcher stops at 12 arguments, so the registered routine is called directly
    (no error is raised on this path)."""
    from tests.test_abi import build_shim_with_minir
    from tests.test_gpu_shim import MiniR

    R = MiniR(build_shim_with_minir(tmp_path_factory.mktemp("shim_grid")))
    R.L.minir_routine_name.restype = C.c_char_p
    table = {R.L.minir_routine_name(i).decode(): R.L.minir_routine_nargs(i) for i in range(R.L.minir_routine_count())}
    assert table["_bigsnpr_clumping_chr_cached"] == 14
    f = R.L._bigsnpr_clumping_chr_cached
    f.restype = C.c_void_p
    f.argtypes = [C.c_void_p] * 14
    G, chr_, pos, lp = ex
    n, m = G.shape
    d = tmp_path_factory.mktemp("fbm")
    np.asfortranarray(G).T.tofile(d / "geno.bk")
    fbm = R.env(backingfile=R.s(str(d / "geno.bk")), nrow=R.ints([n]), ncol=R.ints([m]),
                code256=R.reals(np.r_[[0.0, 1.0, 2.0], np.full(253, np.nan)]))
    of = oracle.OracleFBM(G)
    ir = np.arange(1, n + 1, dtype=np.int32)
    ind_chr = np.arange(1, 2543, dtype=np.int32)
    sub = np.flatnonzero(np.arange(ind_chr.size) % 4 != 0)
    ic = ind_chr[sub]
    st = oracle.snp_colstats(of, ir, ic)
    ordv = grid_ref._order_decreasing(lp[ic - 1]).astype(np.int32)
    rank = np.empty_like(ordv)
    rank[ordv - 1] = np.arange(1, ordv.size + 1)
    one = R.ints([1])
    sq = R.env(Dim=R.ints([ind_chr.size, ind_chr.size]))  # stands for the dgCMatrix: passed through untouched
    kb = d / "keep.bk"
    for thr, base in ((0.01, 500), (0.2, 100), (0.8, 50)):
        np.full(ic.size, -1, dtype=np.int32).tofile(kb)
        keep = R.env(backingfile=R.s(str(kb)), nrow=R.ints([1]), ncol=R.ints([ic.size]))
        size = 1000 * base / thr
        out = f(fbm, keep, sq, R.ints(sub), R.ints(ir), R.ints(ic), R.ints(ordv), R.ints(rank), R.reals(pos[ic - 1]),
                R.reals(st["sumX"]), R.reals(st["denoX"]), R.reals([size]), R.reals([thr]), one)
        assert out == sq and R.L.minir_protect_depth() == 0
        want = np.full(ic.size, -1, dtype=np.int32)
        grid_ref.clumping_chr_cached(of, want, np.zeros((ind_chr.size,) * 2), sub, ir, ic, ordv, rank, pos[ic - 1],
                                     st["sumX"], st["denoX"], size, thr)
        assert np.array_equal(np.fromfile(kb, dtype=np.int32), want), (thr, base)
