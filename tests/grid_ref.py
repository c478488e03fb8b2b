"""CPU oracle of snp_grid_clumping -- test infrastructure only.

* ``clumping_chr_cached``: ctypes wrapper over ``tests/grid_oracle.c``, the literal restatement of
  src/clumping-cached.cpp:11-110 (compiled on first use into a temporary directory).
* ``snp_grid_clumping``: NumPy restatement of R/SCT.R:32-151 over it, passing the r2 cache between the calls exactly as the R
  code does (``spcor.chr[ind, ind]`` at every threshold of imputation).  The cache is dense here; an entry the reference's
  sparse matrix does not hold reads 0, as it does there.

G is an ``oracle.ref.OracleFBM``; indices are 1-based like R's.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "grid_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), "bsg_grid_oracle_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "grid_oracle_%s.so" % hashlib.sha1(src).hexdigest()[:12])
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", _SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def clumping_chr_cached(G, keep, sqcor, spInd, rowInd, colInd, ordInd, rankInd, pos, sumX, denoX, size, thr):
    """src/clumping-cached.cpp:11-110: fills `keep` (int32, -1 on entry) and returns the new cache (a copy of sqcor with the
    r2 computed by this call)."""
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)  # noqa: E731
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)  # noqa: E731
    spInd, rowInd, colInd, ordInd, rankInd = i32(spInd), i32(rowInd), i32(colInd), i32(ordInd), i32(rankInd)
    pos, sumX, denoX = f64(pos), f64(sumX), f64(denoX)
    if spInd.size != colInd.size:
        raise ValueError("Incompatibility between dimensions.")
    sqcor = np.asfortranarray(sqcor, dtype=np.float64)
    new = sqcor.copy(order="F")
    assert keep.dtype == np.int32 and keep.flags.c_contiguous
    with np.errstate(all="ignore"):
        rc = lib().grc_clumping_chr_cached(
            _p(G.bytes, C.c_uint8), G.nrow, _p(G.code256, C.c_double), _p(sqcor, C.c_double), _p(new, C.c_double),
            sqcor.shape[0], _p(spInd, C.c_int), _p(rowInd, C.c_int), rowInd.size, _p(colInd, C.c_int), colInd.size,
            _p(ordInd, C.c_int), _p(rankInd, C.c_int), _p(pos, C.c_double), _p(sumX, C.c_double), _p(denoX, C.c_double),
            C.c_double(size), C.c_double(thr), _p(keep, C.c_int))
    if rc:
        raise MemoryError("grid oracle: allocation failure")
    return new


def _order_decreasing(x):
    """R's order(x, decreasing = TRUE), 1-based: ties by position, NA last."""
    x = np.asarray(x, dtype=np.float64)
    return np.argsort(np.where(np.isnan(x), np.inf, -x), kind="stable") + 1


def snp_grid_clumping(G, infos_chr, infos_pos, lpS, ind_row=None, grid_thr_r2=(0.01, 0.05, 0.1, 0.2, 0.5, 0.8, 0.95),
                      grid_base_size=(50, 100, 200, 500), infos_imp=None, grid_thr_imp=1, groups=None, exclude=None):
    """R/SCT.R:32-151 -> (list per chromosome of lists of 1-based index arrays, grid dict)."""
    from oracle import ref

    m = G.ncol
    infos_chr = np.asarray(infos_chr)
    infos_pos = np.asarray(infos_pos, dtype=np.float64)
    lpS = np.asarray(lpS, dtype=np.float64)
    infos_imp = np.ones(m) if infos_imp is None else np.asarray(infos_imp, dtype=np.float64)
    for v in (infos_chr, infos_pos, infos_imp, lpS):  # assert_lengths
        if len(v) != m:
            raise ValueError("Incompatibility between dimensions.")
    groups = [np.arange(1, m + 1)] if groups is None else [np.asarray(g, dtype=np.int64).reshape(-1) for g in groups]
    ind_row = np.arange(1, G.nrow + 1, dtype=np.int32) if ind_row is None else np.asarray(ind_row, dtype=np.int32)
    THR_IMP = np.unique(np.asarray(grid_thr_imp, dtype=np.float64).reshape(-1))
    THR_CLMP = np.unique(np.asarray(grid_thr_r2, dtype=np.float64).reshape(-1))
    BASE_SIZE_CLMP = np.unique(np.asarray(grid_base_size, dtype=np.float64).reshape(-1))
    rows = [(b, t, g, i) for i in THR_IMP for g in range(1, len(groups) + 1) for t in THR_CLMP for b in BASE_SIZE_CLMP]
    grid = {"size": np.array([int(b / t) for b, t, _, _ in rows], dtype=np.int32),
            "thr_r2": np.array([r[1] for r in rows]), "grp_num": np.array([r[2] for r in rows], dtype=np.int32),
            "thr_imp": np.array([r[3] for r in rows])}
    excl = np.asarray([] if exclude is None else exclude, dtype=np.int64)
    ind_noexcl = np.array([j for j in range(1, infos_chr.size + 1) if j not in set(excl.tolist())], dtype=np.int64)
    all_keep = []
    for chrom in sorted(set(infos_chr[ind_noexcl - 1].tolist())):
        ind_chr = ind_noexcl[infos_chr[ind_noexcl - 1] == chrom].astype(np.int32)
        ind_keep = []
        info_chr, S_chr, pos_chr = infos_imp[ind_chr - 1], lpS[ind_chr - 1], infos_pos[ind_chr - 1]
        stats = ref.snp_colstats(G, ind_row, ind_chr)
        sumX_chr, denoX_chr = stats["sumX"], stats["denoX"]
        spcor_chr = np.zeros((ind_chr.size, ind_chr.size), order="F")
        if np.any(np.diff(pos_chr) < 0):
            raise ValueError("'pos.chr' is not sorted.")
        for thr_imp in THR_IMP:
            ind = np.flatnonzero(info_chr >= thr_imp)
            ind_chr, info_chr, pos_chr, S_chr = ind_chr[ind], info_chr[ind], pos_chr[ind], S_chr[ind]
            spcor_chr = np.asfortranarray(spcor_chr[np.ix_(ind, ind)])
            sumX_chr, denoX_chr = sumX_chr[ind], denoX_chr[ind]
            for group in groups:
                ind2 = np.flatnonzero(np.isin(ind_chr, group))
                if ind2.size == 0:
                    ind_keep.extend(np.zeros(0, dtype=np.int32) for _ in range(THR_CLMP.size * BASE_SIZE_CLMP.size))
                    continue
                ind_chr_grp = ind_chr[ind2]
                ord_chr_grp = _order_decreasing(S_chr[ind2])
                rank_chr_grp = np.empty_like(ord_chr_grp)
                rank_chr_grp[ord_chr_grp - 1] = np.arange(1, ord_chr_grp.size + 1)
                keep = np.empty(ind_chr_grp.size, dtype=np.int32)
                for thr_clmp in THR_CLMP:
                    for base_size_clmp in BASE_SIZE_CLMP:
                        keep[:] = -1
                        spcor_chr = clumping_chr_cached(G, keep, spcor_chr, ind2, ind_row, ind_chr_grp, ord_chr_grp,
                                                        rank_chr_grp, pos_chr[ind2], sumX_chr[ind2], denoX_chr[ind2],
                                                        1000 * base_size_clmp / thr_clmp, thr_clmp)
                        assert np.all((keep == 0) | (keep == 1))
                        ind_keep.append(ind_chr_grp[keep == 1])
        all_keep.append(ind_keep)
    return all_keep, grid
