"""Exact model of the windowed pair band (bsg_cor.cu: pair_band, k_cor_from_sums, k_fill_csc, k_ld_reduce) and of the
clumping sweep that reads its conflict flags (bsg_grid.cu) -- test infrastructure only.

Every pair sum the device forms (nona, xSum, xxSum, ySum, yySum, xySum) is an exact integer that depends neither on the
tile mode, nor on the kernel, the batch or the tile order.  The model takes them from fp32 GEMMs of the planes
a = g (NA -> 0), b = [g valid], h = [g == 2] over the real rows (exact below 2^24) and then runs each epilogue with
IEEE double operations in the kernel's source order:

* COR, LD, LEVELS have no contractible operation (every product feeds a division, a square root or nothing), so NumPy's
  ``*``, ``/``, ``-`` and ``sqrt`` give the device's bytes;
* CLUMP's numerator is the pinned chain fma(cx*cy, nona, fma(cx, -ySum, fma(cy, -xSum, xySum))).  It is evaluated in
  plain doubles with a forward error bound, and with ``fixedpoint_ref.fma`` (exact rounding) on every pair whose flag
  the bound cannot decide.

G is the decoded selection (nr, nc) with codes 0 / 1 / 2 and 3 for NA (``oracle.read_bed(..., na_val=3)``); row and
column multisets are simply its repeated rows and columns.  Pad slots of the device's lines never appear here.
"""
from __future__ import annotations

import numpy as np

from tests.fixedpoint_ref import fma

TM = CTN = 128  # owners per row block, columns per column block
MAX_SUM_INTS = 768 << 20  # int32 tile sums per batch (pair_band's max_sum_ints)


# ---- windows ------------------------------------------------------------------------------------------------------------
class Band:
    """Window of every owner j0 (the columns j0 - wlen[j0] .. j0 - 1) and the band layout: pair (j0, j0 - 1 - k) at
    boff[j0] + k.  reach[j] = the largest owner whose window holds j (j itself when there is none)."""

    def __init__(self, pos, size, both=False):
        pos = np.asarray(pos, dtype=np.float64)
        nc = pos.size
        j0 = np.arange(nc)
        # first j with pos[j] >= pos[j0] - size (and, for the clumping kinds, first j with pos[j0] <= pos[j] + size):
        # both tests are monotone in j because pos is sorted and rounding is monotone
        left = np.searchsorted(pos, pos - size, side="left")
        if both:
            left = np.minimum(left, np.searchsorted(pos + size, pos, side="left"))
        left = np.minimum(left, j0)
        self.nc = nc
        self.left = left
        self.wlen = (j0 - left).astype(np.int64)
        self.boff = np.concatenate([[0], np.cumsum(self.wlen)]).astype(np.int64)
        self.total = int(self.boff[-1])
        last = np.searchsorted(left, j0, side="right") - 1  # windows are contiguous and their left edges ascend
        self.reach = np.maximum(j0, last)

    def entries(self, owners=None):
        """(o, j0, j) of every band entry of the given owners (all by default), in band order."""
        owners = np.arange(self.nc) if owners is None else np.asarray(owners, dtype=np.int64)
        w = self.wlen[owners]
        J0 = np.repeat(owners, w)
        start = np.repeat(self.boff[owners], w)
        K = np.arange(J0.size) - np.repeat(np.cumsum(w) - w, w)
        return start + K, J0, J0 - 1 - K


# ---- pair sums ------------------------------------------------------------------------------------------------------------
def planes(G):
    G = np.asarray(G)
    b = G != 3
    a = np.where(b, G, 0).astype(np.float32)
    return a, b.astype(np.float32), (G == 2).astype(np.float32)


def pair_sums(G, band, owners=None, col0=0):
    """Exact sums of the band entries of `owners` (all by default), in band order: dict of int64 arrays nona, xs, xxs,
    ys, yys, xy (x = owner j0, y = partner j), plus o / j0 / j.  G may hold only the columns col0 .. col0 + G.shape[1]
    of the selection, as long as they cover the windows of `owners`."""
    a, b, h = planes(G)
    if a.shape[0] >= 1 << 22:
        raise ValueError("fp32 sums are exact below 2^24 only")
    o, J0, J = band.entries(owners)
    out = {k: np.zeros(o.size, dtype=np.int64) for k in ("aa", "bb", "ab", "ba", "hb", "bh")}
    blk = J0 // TM
    starts = np.flatnonzero(np.r_[True, blk[1:] != blk[:-1]]) if o.size else np.zeros(0, dtype=np.int64)
    ends = np.r_[starts[1:], o.size]
    for s, e in zip(starts, ends):
        own = np.unique(J0[s:e])
        lo, hi = int(J[s:e].min()), int(own.max())
        assert lo >= col0 and hi <= col0 + a.shape[1], "columns outside G"
        ri = np.searchsorted(own, J0[s:e])
        ci = J[s:e] - lo
        for key, X, Y in (("aa", a, a), ("bb", b, b), ("ab", a, b), ("ba", b, a), ("hb", h, b), ("bh", b, h)):
            M = X[:, own - col0].T @ Y[:, lo - col0:hi - col0]
            out[key][s:e] = M[ri, ci].astype(np.int64)
    return {"o": o, "j0": J0, "j": J, "nona": out["bb"], "xs": out["ab"], "xxs": out["ab"] + 2 * out["hb"],
            "ys": out["ba"], "yys": out["ba"] + 2 * out["bh"], "xy": out["aa"]}


# ---- epilogues (k_cor_from_sums) ------------------------------------------------------------------------------------------
def _num_deno(S):
    nona = S["nona"]
    xs, xxs, ys, yys, xy = (S[k].astype(np.float64) for k in ("xs", "xxs", "ys", "yys", "xy"))
    with np.errstate(all="ignore"):
        num = xy - xs * ys / nona
        dx = xxs - xs * xs / nona
        dy = yys - ys * ys / nona
    return num, dx, dy


def cor_epilogue(S, thr):
    """BAND_COR: (r clamped to [-1, 1], keep = isnan(r) | |r| > thr[max(nona - 1, 0)])."""
    num, dx, dy = _num_deno(S)
    with np.errstate(all="ignore"):
        r = num / np.sqrt(dx * dy)
        keep = np.isnan(r) | (np.abs(r) > np.asarray(thr, dtype=np.float64)[np.maximum(S["nona"] - 1, 0)])
    r = np.where(r > 1, 1.0, np.where(r < -1, -1.0, r))
    return r, keep


def ld_epilogue(S):
    """BAND_LD: r^2 = num^2 / (deno_x deno_y)."""
    num, dx, dy = _num_deno(S)
    with np.errstate(all="ignore"):
        return num * num / (dx * dy)


def levels_epilogue(S, nr, sumX, denoX, levels, col_na):
    """BAND_LEVELS: how many of the sorted `levels` r^2 exceeds; 0 when either column holds a missing value."""
    j0, j = S["j0"], S["j"]
    sumX, denoX = np.asarray(sumX, dtype=np.float64), np.asarray(denoX, dtype=np.float64)
    with np.errstate(all="ignore"):
        num = S["xy"].astype(np.float64) - sumX[j] * sumX[j0] / nr
        r2 = num * num / (denoX[j] * denoX[j0])
    lev = np.zeros(j0.size, dtype=np.int64)
    for t in np.asarray(levels, dtype=np.float64):
        lev += r2 > t
    lev[np.asarray(col_na)[j0] | np.asarray(col_na)[j]] = 0
    return lev


def clump_epilogue(S, center, scale, thr_r2):
    """BAND_CLUMP: r = fma(cx*cy, nona, fma(cx, -ySum, fma(cy, -xSum, xySum))) / (s_j0 * s_j); flag = r * r > thr_r2."""
    j0, j = S["j0"], S["j"]
    center, scale = np.asarray(center, dtype=np.float64), np.asarray(scale, dtype=np.float64)
    cx, cy = center[j0], center[j]
    xs, ys, xy, nona = (S[k].astype(np.float64) for k in ("xs", "ys", "xy", "nona"))
    den = scale[j0] * scale[j]
    with np.errstate(all="ignore"):
        cxy = cx * cy
        num = xy - cy * xs - cx * ys + cxy * nona
        r = num / den
        # |num - fused chain| <= 8 ulp-sized errors of the largest term: decided where r^2 clears thr_r2 by more than that
        err = 1e-14 * (np.abs(xy) + np.abs(cy * xs) + np.abs(cx * ys) + np.abs(cxy * nona)) / np.abs(den) + 1e-300
        sure_hi = np.maximum(np.abs(r) - err, 0) ** 2 > thr_r2 * (1 + 1e-14)
        sure_lo = (np.abs(r) + err) ** 2 < thr_r2 * (1 - 1e-14)
        flag = r * r > thr_r2
    for q in np.flatnonzero(~(sure_hi | sure_lo) & np.isfinite(cxy) & np.isfinite(cx) & np.isfinite(cy)):
        n1 = fma(float(cy[q]), -float(xs[q]), float(xy[q]))
        n2 = fma(float(cx[q]), -float(ys[q]), n1)
        n3 = fma(float(cxy[q]), float(nona[q]), n2)
        with np.errstate(all="ignore"):
            rq = np.float64(n3) / np.float64(den[q])
            flag[q] = rq * rq > thr_r2
    return flag


# ---- assembly and reductions ------------------------------------------------------------------------------------------------
def csc(band, S, r, keep, fill_diag=True):
    """k_fill_csc: kept entries by ascending row index, the diagonal (1.0) last.  -> (p int64, i int32, x float64)."""
    col, row, val = S["j0"][keep], S["j"][keep], r[keep]
    if fill_diag:
        d = np.arange(band.nc)
        col, row, val = np.r_[col, d], np.r_[row, d], np.r_[val, np.ones(band.nc)]
    order = np.lexsort((row, col))
    p = np.r_[0, np.cumsum(np.bincount(col, minlength=band.nc))].astype(np.int64)
    return p, row[order].astype(np.int32), val[order].astype(np.float64)


def ld_reduce(band, r2):
    """k_ld_reduce: 1.0, then the owner's own window for k ascending, then the later owners j0 = j + 1 + k ascending,
    NaN skipped; one sequential sum per column (vectorised across columns only)."""
    nc = band.nc
    full = np.asarray(r2, dtype=np.float64)
    assert full.size == band.total
    acc = np.ones(nc)
    j = np.arange(nc)
    kmax = int(band.wlen.max()) if nc else 0
    for k in range(kmax):
        m = band.wlen > k
        v = full[band.boff[:-1][m] + k]
        idx = j[m]
        ok = ~np.isnan(v)
        acc[idx[ok]] += v[ok]
    for k in range(kmax):
        j0 = j + 1 + k
        m = (j0 <= band.reach) & (j0 < nc)
        m[m] &= k < band.wlen[j0[m]]
        v = full[band.boff[j0[m]] + k]
        idx = j[m]
        ok = ~np.isnan(v)
        acc[idx[ok]] += v[ok]
    return acc


def bed_cor(G, size, thr, pos=None, fill_diag=True):
    """Model of corMat / bed_cor: `size` and `pos` in the units of the call (bp), thr indexed by nona - 1."""
    nc = G.shape[1]
    pos = 1000.0 * np.arange(1, nc + 1) if pos is None else pos
    band = Band(pos, size)
    S = pair_sums(G, band)
    r, keep = cor_epilogue(S, thr)
    return csc(band, S, r, keep, fill_diag)


def ld_scores(G, size, pos=None):
    nc = G.shape[1]
    pos = 1000.0 * np.arange(1, nc + 1) if pos is None else pos
    band = Band(pos, size)
    return ld_reduce(band, ld_epilogue(pair_sums(G, band)))


# ---- the clumping sweep -----------------------------------------------------------------------------------------------------
def clump_sweep(band, flag, pos, size, ordInd):
    """The sequential pass of src/clumping-bed.cpp / src/clumping.cpp over per-pair conflict flags (bool per band entry):
    variants in priority order; neighbours as which_to_check lists them (right while pos[j] <= pos[j0] + size, left while
    pos[j] >= pos[j0] - size, alternating, each side stopping at its first failure); j0 is removed when a better-ranked kept
    neighbour conflicts with it.  -> keep (int32 0 / 1)."""
    pos = np.asarray(pos, dtype=np.float64)
    m = pos.size
    order = np.asarray(ordInd, dtype=np.int64) - 1
    rank = np.empty(m, dtype=np.int64)
    rank[order] = np.arange(m)
    keep = np.full(m, -1, dtype=np.int32)
    wlen, boff = band.wlen, band.boff
    flag = np.asarray(flag, dtype=bool).tolist()
    posl, rankl, wl, bo = pos.tolist(), rank.tolist(), wlen.tolist(), boff.tolist()
    for j0 in order.tolist():
        pmin, pmax = posl[j0] - size, posl[j0] + size
        kj = 1
        hi_ok = lo_ok = True
        k = 1
        while (hi_ok or lo_ok) and kj:
            if hi_ok:
                j = j0 + k
                hi_ok = j < m and posl[j] <= pmax
                if hi_ok and rankl[j0] > rankl[j] and keep[j] != 0:
                    assert j - 1 - j0 < wl[j], "pair outside the band"
                    if flag[bo[j] + j - 1 - j0]:
                        kj = 0
            if lo_ok and kj:
                j = j0 - k
                lo_ok = j >= 0 and posl[j] >= pmin
                if lo_ok and rankl[j0] > rankl[j] and keep[j] != 0:
                    assert j0 - 1 - j < wl[j0], "pair outside the band"
                    if flag[bo[j0] + j0 - 1 - j]:
                        kj = 0
            k += 1
        keep[j0] = kj
    return keep


# ---- path metadata (which code paths a case reaches; the bytes never depend on it) ---------------------------------------
class Plan:
    """pair_band's tiling: per-column NA flags, the tiles (row block, column block, mode) of every batch under the bound on
    the tile sums, and the number of B tiles per row block."""

    def __init__(self, G_or_na, band, max_sum_ints=MAX_SUM_INTS):
        na = np.asarray(G_or_na)
        if na.ndim == 2:
            na = (na == 3).any(axis=0)
        nc = band.nc
        self.col_na = na.astype(bool)
        nib, njb = (nc + TM - 1) // TM, (nc + CTN - 1) // CTN
        na_jb = np.zeros(njb, dtype=bool)
        np.logical_or.at(na_jb, np.arange(nc) // CTN, self.col_na)
        self.na_jb = na_jb
        self.batches = []  # list of (ib_start, ib_end, [(ib, jb, mode)], used)
        self.ntiles = np.zeros(nib, dtype=np.int64)
        wlen = band.wlen
        ib = 0
        while ib < nib:
            tiles, used, ib_start = [], 0, ib
            while ib < nib:
                r0, r1 = ib * TM, min(nc, ib * TM + TM)
                w = wlen[r0:r1]
                live = np.flatnonzero(w > 0)
                if live.size:
                    jb0 = int(((r0 + live) - w[live]).min()) // CTN
                    jb1 = int(r0 + live.max() - 1) // CTN
                    na_i = bool(na_jb[r0 // CTN:(r1 - 1) // CTN + 1].any())
                    modes = [int(na_i or na_jb[jb]) for jb in range(jb0, jb1 + 1)]
                    need = sum(6 if md else 1 for md in modes) * TM * CTN
                    if used + need > max_sum_ints and ib > ib_start:
                        break
                    tiles += [(ib, jb0 + q, md) for q, md in enumerate(modes)]
                    used += need
                    self.ntiles[ib] = len(modes)
                ib += 1
            self.batches.append((ib_start, ib, tiles, used))

    @property
    def nbatches(self):
        return len(self.batches)

    def boundaries(self):
        """first row block of every batch after the first"""
        return [b[0] for b in self.batches[1:]]

    def mixed_pairs(self):
        """(batch, 256-row pair, column block) where the pair's two 128-row halves both have a tile and their modes
        differ: gramt_cor runs the five NA products for one half only."""
        out = []
        for bi, (_, _, tiles, _) in enumerate(self.batches):
            mode = {(ib, jb): md for ib, jb, md in tiles}
            for (ib, jb), md in mode.items():
                if ib % 2 == 0 and (ib + 1, jb) in mode and mode[(ib + 1, jb)] != md:
                    out.append((bi, ib // 2, jb))
        return out

    def split_pairs(self):
        """256-row pairs whose halves fall in different batches (a boundary at an odd row block)."""
        return [b for b in self.boundaries() if b % 2 == 1]
