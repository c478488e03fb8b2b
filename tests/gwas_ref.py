"""CPU restatements of big_univLinReg (bigstatsr's univLinReg5 + R glue, not vendored in the reference) and an exact model
of the device arithmetic of bsg_univlinreg (bigsnpr_b200/csrc/bsg_gwas.cu).

- `univlinreg_fp64`: the literal fp64 statistic of univLinReg5 on a dense matrix (y2 = y - U U'y, x2 = x - U U'x, ...), with
  the port's intended differences: NaN for a column holding an NA value or a constant column.
- `univlinreg_model`: every step the device takes -- host scalars as sequential sums, the quantisation of y_c (60 bits,
  8 digits) and of each column of U (30 bits, 4 digits) scattered onto the sample positions, exact integer slice sums,
  the top-down fp64 combination, the epilogue in the kernel's operation order -- so that its output is byte-identical.
- `model_bound`: a per-column bound on |model - fp64 restatement| (quantisation of the vectors, plus fp64 slack).
"""
from __future__ import annotations

import numpy as np

Y_BITS, U_BITS, Y_DIG, U_DIG = 60, 30, 8, 4
SLACK = 1e-12  # fp64 rounding slack of either side, relative to the largest magnitude a difference cancels


def read_bed_codes(path, n, m):
    """n x m uint8 codes of a PLINK .bed (0 / 1 / 2, 3 = NA), the staged values of the device copy."""
    raw = np.fromfile(path, dtype=np.uint8)[3:].reshape(m, (n + 3) // 4)
    f = np.stack([(raw >> (2 * k)) & 3 for k in range(4)], axis=2).reshape(m, -1)[:, :n]
    dec = np.array([2, 3, 1, 0], dtype=np.uint8)  # .bed 00 -> 2, 01 -> NA, 10 -> 1, 11 -> 0
    return np.ascontiguousarray(dec[f].T)


def covar_basis(covar, n, thr_eigval=1e-4):
    """The R glue's U (same as bigsnpr_b200.api.univlinreg_covar_basis, restated without the package)."""
    cols = [np.ones(n)]
    if covar is not None:
        cv = np.asarray(covar, dtype=np.float64)
        cols.append(cv.reshape(n, -1) if cv.ndim == 1 else cv)
    C = np.column_stack(cols)
    u, d, _ = np.linalg.svd(C, full_matrices=False)
    return u[:, d / (np.sqrt(n) + np.sqrt(C.shape[1]) - 1) > thr_eigval]


def univlinreg_fp64(Xd, y, U):
    """Literal univLinReg5 on the dense nr x m matrix Xd of the ind.train rows (NaN = NA).  Returns estim, std_err, score."""
    Xd = np.asarray(Xd, dtype=np.float64)
    nr, K = U.shape
    na = np.isnan(Xd).any(axis=0)
    X0 = np.where(np.isnan(Xd), 0.0, Xd)
    y2 = y - U @ (U.T @ y)
    x2 = X0 - U @ (U.T @ X0)
    xx = np.einsum("ij,ij->j", x2, x2)
    xy = x2.T @ y2
    with np.errstate(invalid="ignore", divide="ignore"):
        estim = xy / xx
        rss = y2 @ y2 - estim * xy
        se = np.sqrt(rss / (nr - K - 1) / xx)
    const = np.all(X0 == X0[:1], axis=0)
    bad = na | const
    estim[bad] = np.nan
    se[bad] = np.nan
    return estim, se, estim / se


def _seqsum(a):
    """The C loop `s += a[i]` in index order."""
    a = np.asarray(a, dtype=np.float64)
    return float(np.cumsum(a)[-1]) if a.size else 0.0


def _pick_e(m, hb, bits):
    if m > 0:
        return bits - int(np.frexp(m)[1]) - hb
    return 0


def _hb_bits(maxmult):
    b = 0
    while (1 << b) < maxmult:
        b += 1
    return b + 1 if b >= 8 else b


def _digits(Q, nd):
    q = Q.copy()
    out = []
    for _ in range(nd):
        d = ((q & 0xFF).astype(np.int64) ^ 0x80) - 0x80  # low byte as int8
        q = (q - d) >> 8
        out.append(d)
    return out


def host_scalars(y, U):
    nr, K = U.shape
    ybar = _seqsum(y) / nr
    yc = y - ybar
    yy = _seqsum(yc * yc)
    u1 = np.array([_seqsum(U[:, k]) for k in range(K)])
    uy = np.array([_seqsum(U[:, k] * yc) for k in range(K)])
    yres = yy - _seqsum(uy * uy)
    return yc, yy, u1, uy, yres


def univlinreg_model(vals, na, ind_row, ind_col, U, y, D=1, with_parts=False):
    """Exact model of bsg_univlinreg.  vals: n x m value bytes (hard calls: the codes, NA = 3; dosages: D x dosage, NA
    entries arbitrary), na: n x m bool; ind_row / ind_col 0-based (repeats allowed); U nr x K; y nr.  Returns estim, std_err
    (and the intermediate quantities when with_parts)."""
    n = vals.shape[0]
    ind_row = np.asarray(ind_row, dtype=np.int64)
    ind_col = np.asarray(ind_col, dtype=np.int64)
    nr, K = U.shape
    mult = np.bincount(ind_row, minlength=n).astype(np.int64)
    hb = _hb_bits(int(mult.max()) if nr else 1)
    yc, yy, u1, uy, yres = host_scalars(y, U)
    V = K + 1
    S = np.empty((V, ind_col.size))
    es, digs = [], []
    for v in range(V):
        x = yc if v == 0 else U[:, v - 1]
        bits, nd = (Y_BITS, Y_DIG) if v == 0 else (U_BITS, U_DIG)
        e = _pick_e(float(np.max(np.abs(x))) if nr else 0.0, hb, bits)
        es.append(e)
        q = np.rint(np.ldexp(x, e)).astype(np.int64)
        Q = np.zeros(n, dtype=np.int64)
        np.add.at(Q, ind_row, q)
        digs.append(np.column_stack(_digits(Q, nd)).astype(np.float64))  # n x nd
    sx = np.empty(ind_col.size, dtype=np.int64)
    sxx = np.empty(ind_col.size, dtype=np.int64)
    nna = np.empty(ind_col.size, dtype=np.int64)
    for c0 in range(0, ind_col.size, 256):  # column blocks keep the dense copies small
        cb = ind_col[c0:c0 + 256]
        Vc = vals[:, cb].astype(np.float64)
        NAc = na[:, cb]
        for v in range(V):
            sd = digs[v].T @ Vc  # integer partial sums < 2^53: exact
            acc = np.zeros(cb.size)
            for d in range(digs[v].shape[1] - 1, -1, -1):
                acc = acc + np.ldexp(sd[d], 8 * d - es[v])
            S[v, c0:c0 + cb.size] = acc / D
        vm = np.where(NAc, 0, vals[:, cb].astype(np.int64))
        sx[c0:c0 + cb.size] = mult @ vm
        sxx[c0:c0 + cb.size] = mult @ (vm * vm)
        nna[c0:c0 + cb.size] = mult @ NAc.astype(np.int64)
    num_i = nr * sxx - sx * sx
    nd_ = float(nr) * D
    with np.errstate(invalid="ignore", divide="ignore"):
        ssx = num_i.astype(np.float64) / (nd_ * D)
        mx = sx.astype(np.float64) / nd_
        qq = np.zeros(ind_col.size)
        pp = np.zeros(ind_col.size)
        T = np.empty((K, ind_col.size))
        for k in range(K):
            t = S[1 + k] - mx * u1[k]
            T[k] = t
            qq = qq + t * t
            pp = pp + t * uy[k]
        den = ssx - qq
        num = S[0] - pp
        b = num / den
        rss = yres - b * num
        se = np.sqrt((rss / (nr - K - 1)) / den)
    bad = (nna > 0) | (num_i <= 0) | ~(den > 0)
    b[bad] = np.nan
    se[bad] = np.nan
    if not with_parts:
        return b, se
    return b, se, dict(sx=sx, sxx=sxx, ssx=ssx, mx=mx, T=T, den=den, num=num, rss=rss, es=es, u1=u1, uy=uy, yy=yy,
                       yres=yres, sum_yc=float(np.sum(yc)), D=D, nr=nr, K=K)


def model_bound(parts, estim, se):
    """Per-column bounds (on estim, on std_err) of |model - univlinreg_fp64|: each quantised entry is within half a unit of
    its last place (2^-e), so |x.v - x.v~| <= sum(x) 2^-e / 2; the fp64 steps of either side get SLACK relative to the
    largest term each difference cancels."""
    p = parts
    D, K = p["D"], p["K"]
    sxr = p["sx"] / D
    sxxr = p["sxx"] / (D * D)
    dy = 0.5 * np.ldexp(1.0, -p["es"][0]) * sxr
    dk = [0.5 * np.ldexp(1.0, -p["es"][1 + k]) * sxr for k in range(K)]
    dq = sum(2 * np.abs(p["T"][k]) * dk[k] + dk[k] ** 2 for k in range(K))
    dp = sum(np.abs(p["uy"][k]) * dk[k] for k in range(K))
    norm_y = np.sqrt(p["yy"])
    dden = dq + SLACK * sxxr
    dnum = dy + dp + np.abs(p["mx"] * p["sum_yc"]) + SLACK * np.sqrt(sxxr) * norm_y
    with np.errstate(invalid="ignore", divide="ignore"):
        room = p["den"] - dden
        be = np.where(room > 0, (dnum + np.abs(estim) * dden) / room, np.inf)
        drss = np.abs(p["num"]) * be + np.abs(estim) * dnum + SLACK * p["yy"]
        rel = 0.5 * (drss / np.abs(p["rss"]) + dden / room) * 1.01
        bs = np.where((room > 0) & (p["rss"] > drss), se * rel + 1e-15 * se, np.inf)
    return be, bs
