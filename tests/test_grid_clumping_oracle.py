"""snp_grid_clumping's oracle (tests/grid_ref.py) against the reference's own checks (tests/testthat/test-6-SCT.R:32-83) on
example.bed read as an FBM.code256, and the premise of the device design: the r2 cache of clumping_chr_cached never changes a
decision, so every grid point is a plain clumping_chr.  CPU only."""
import ctypes
import os

import numpy as np
import pytest

from tests import grid_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
THR, BASE = (0.05, 0.2, 0.8), (100, 200)


@pytest.fixture(scope="module")
def ex(oracle):
    o = oracle.OracleBed(os.path.join(GOLDEN, "example.bed"))
    G = oracle.OracleFBM(oracle.decode_dense(o).astype(np.uint8))
    pos = np.array([float(ln.split()[3]) for ln in open(os.path.join(GOLDEN, "example.bim"))])
    chr_ = np.repeat([1, 2], [2542, 2000])
    lp = -np.log10(np.random.default_rng(6).uniform(size=G.ncol))
    infos = np.random.default_rng(7).uniform(0.2, 1.0, size=G.ncol)
    return G, chr_, pos, lp, infos


@pytest.fixture(scope="module")
def all_keep(ex):
    G, chr_, pos, lp, _ = ex
    return grid_ref.snp_grid_clumping(G, chr_, pos, lp, grid_thr_r2=THR, grid_base_size=BASE)


def test_unsorted_positions(ex):
    G, chr_, pos, lp, _ = ex
    with pytest.raises(ValueError, match="'pos.chr' is not sorted."):
        grid_ref.snp_grid_clumping(G, chr_, np.random.default_rng(1).permutation(pos), lp)
    with pytest.raises(ValueError, match="Incompatibility between dimensions."):
        grid_ref.snp_grid_clumping(G, chr_[1:], pos, lp)


def test_three_chromosomes(ex):
    G, chr_, pos, lp, _ = ex
    res, grid = grid_ref.snp_grid_clumping(G, np.r_[chr_[1:], 22], np.r_[pos[1:], 1.0], lp, grid_thr_r2=0.2,
                                           grid_base_size=50)
    assert len(res) == 3 and all(len(r) == 1 for r in res) and grid["size"].tolist() == [250]


def test_grid_points_are_snp_clumping(oracle, ex, all_keep):
    """test-6-SCT.R:44-48: each grid point equals snp_clumping(thr.r2, size = grid$size) over both chromosomes."""
    G, chr_, pos, lp, _ = ex
    res, grid = all_keep
    assert len(res) == 2 and all(len(r) == 6 for r in res)
    assert grid["size"].tolist() == [2000, 4000, 500, 1000, 125, 250]
    for i in range(6):
        want = oracle.snp_clumping(G, chr_, S=lp, thr_r2=grid["thr_r2"][i], size=grid["size"][i], infos_pos=pos)
        assert np.array_equal(want, np.concatenate([res[0][i], res[1][i]])), i
    sizes = [len(res[0][i]) for i in range(6)]
    assert 0 < min(sizes) < 2542 and len(set(sizes)) > 3  # the thresholds and sizes prune, differently


def test_imputation_thresholds_equal_groups(ex):
    """test-6-SCT.R:50-72: thr.imp subsets equal the corresponding groups; the grid attribute's shape and columns."""
    G, chr_, pos, lp, infos = ex
    k3, g3 = grid_ref.snp_grid_clumping(G, chr_, pos, lp, grid_thr_r2=THR, grid_base_size=BASE, infos_imp=infos,
                                        grid_thr_imp=(0.3, 0.8, 0.95))
    assert sorted(g3) == ["grp_num", "size", "thr_imp", "thr_r2"] and g3["size"].size == 18
    assert np.array_equal(g3["thr_imp"], np.repeat([0.3, 0.8, 0.95], 6)) and np.all(g3["grp_num"] == 1)
    groups = [np.flatnonzero(infos >= t) + 1 for t in (0.3, 0.8, 0.95)]
    k4, g4 = grid_ref.snp_grid_clumping(G, chr_, pos, lp, grid_thr_r2=THR, grid_base_size=BASE, groups=groups)
    assert g4["size"].size == 18 and np.all(g4["thr_imp"] == 1)
    assert np.array_equal(g4["grp_num"], np.repeat([1, 2, 3], 6))
    for a, b in zip(k3, k4):
        assert len(a) == len(b) == 18 and all(np.array_equal(x, y) for x, y in zip(a, b))


def test_empty_and_singleton_groups(ex, all_keep):
    """test-6-SCT.R:74-83: groups = list(NULL, 1, all) -> empty sets, the singleton, then the plain grid."""
    G, chr_, pos, lp, _ = ex
    res, _ = all_keep
    k5, g5 = grid_ref.snp_grid_clumping(G, chr_, pos, lp, grid_thr_r2=THR, grid_base_size=BASE,
                                        groups=[[], [1], np.arange(1, G.ncol + 1)])
    assert np.array_equal(g5["grp_num"], np.repeat([1, 2, 3], 6))
    want = [[np.zeros(0)] * 6 + [np.array([1])] * 6 + res[0], [np.zeros(0)] * 12 + res[1]]
    for a, b in zip(k5, want):
        assert len(a) == 18 and all(np.array_equal(x, y) for x, y in zip(a, b))


def test_cached_equals_clumping_chr(oracle, ex):
    """clumping_chr_cached equals clumping_chr at every grid point while the cache is carried from call to call, and
    the cache holds r2 values that a recomputation reproduces."""
    G, chr_, pos, lp, _ = ex
    ind_chr = np.arange(1, 1201, dtype=np.int32)
    ir = np.arange(1, G.nrow + 1, dtype=np.int32)
    st = oracle.snp_colstats(G, ir, ind_chr)
    sub = np.flatnonzero(np.arange(ind_chr.size) % 3 != 1)  # a subset, as a group would give
    ordv = grid_ref._order_decreasing(lp[ind_chr[sub] - 1]).astype(np.int32)
    rank = np.empty_like(ordv)
    rank[ordv - 1] = np.arange(1, ordv.size + 1)
    sq = np.zeros((ind_chr.size, ind_chr.size), order="F")
    for thr in (0.01, 0.2, 0.8):
        for base in (50, 500):
            size = 1000 * base / thr
            keep = np.full(sub.size, -1, dtype=np.int32)
            sq = grid_ref.clumping_chr_cached(G, keep, sq, sub, ir, ind_chr[sub], ordv, rank, pos[ind_chr[sub] - 1],
                                              st["sumX"][sub], st["denoX"][sub], size, thr)
            want = oracle.clumping_chr(G, ir, ind_chr[sub], ordv, rank, pos[ind_chr[sub] - 1], st["sumX"][sub],
                                       st["denoX"][sub], size, thr)
            assert np.array_equal(keep, want), (thr, base)
    nz = np.argwhere(sq != 0)
    assert nz.shape[0] > 100
    X = np.where(np.isnan(G.code256[G.bytes]), np.nan, G.code256[G.bytes])
    for a, b in nz[:: max(1, nz.shape[0] // 50)]:
        ja, jb = ind_chr[a] - 1, ind_chr[b] - 1
        num = np.dot(X[:, ja], X[:, jb]) - st["sumX"][a] * st["sumX"][b] / G.nrow
        assert abs(num * num / (st["denoX"][a] * st["denoX"][b]) - sq[a, b]) < 1e-9


def test_grid_entry_point_is_exported():
    """bsg_grid_clumping_chr is declared in bsgpu.h, exported by libbsgpu and typed by the Python binding."""
    from bigsnpr_b200 import _lib, build

    so = build.build()
    assert hasattr(ctypes.CDLL(so), "bsg_grid_clumping_chr")
    res, args = _lib.SIGNATURES["bsg_grid_clumping_chr"]
    assert res is ctypes.c_int and len(args) == 16
    assert "bsg_grid_clumping_chr(" in open(os.path.join(ROOT, "include", "bsgpu.h")).read()


def test_grid_kernels_compile_without_spills():
    """The grid kernels keep everything in registers (no local memory) and the dosage pair tiles run on IMMA u8 x u8."""
    import subprocess

    from bigsnpr_b200 import build

    so = build.build()
    res = subprocess.run(["cuobjdump", "-res-usage", so], capture_output=True, text=True).stdout.splitlines()
    names = ("k_dos_pairs", "k_dos_compact", "k_grid_round", "k_cor_from_sumsILi4", "k_pairsILi4")
    found = {}
    for i, ln in enumerate(res):
        for nm in names:
            if nm in ln and i + 1 < len(res):
                found[nm] = res[i + 1]
    assert set(found) == set(names), found
    assert all("LOCAL:0" in v and "STACK:0" in v for v in found.values()), found
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    body = sass[sass.find("Function : _ZN3bsg4grid11k_dos_pairs"):]
    body = body[:body.find("Function :", 20)]
    assert "IMMA.16832.U8.U8" in body
