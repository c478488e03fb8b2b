"""Host references of the C+T scores (snp_PRS, R/PRS.R:3-76; snp_grid_PRS, R/SCT.R:201-246).

* `literal`: R's loop in fp64 -- thresholds in order(thr.list, decreasing = TRUE), the SNPs still unused whose lpS
  exceeds the threshold (strict) added as prodVecRev = G[, ind] %*% ((2 same - 1) beta) + 2 sum(beta[!same]), the
  product summed over the columns in order (big_prodVec), `last +` the previous column.  An NA code is NaN.
* `exact`: the device arithmetic of bsg_prs.cu, built on fixedpoint_ref: one exponent per keep set (pick_e over the
  set's |beta|, 60 bits, hb = 0), Q = rint(v 2^e), signed base-256 digits, per output the exact integer slice totals
  of code x digit over the entries of the steps so far plus -2 x digit over the reversed ones, then the top-down sum
  over the 8 slices of scalbn(total_s, 8 s - e) with every add rounded on its own (the kernel uses __dadd_rn).  A row
  holding an NA code in an entry of the steps so far is NaN.  Dosage tables (codes multiples of 1 / D): the value bytes
  round(D code) take the codes' place, the reversed constant is -2 D x digit, and the sum is divided by D once.

Accuracy of `exact` (DESIGN.md section 4.1 item 4): |exact - R| <= sum_j |g_ij - 2 rev_j| 2^(-e-1) + a few ulps, with
2^-e < 2^-59 max|v|, against R's own fp64 rounding of its `last +` chain.
"""
from __future__ import annotations

import numpy as np

from tests import fixedpoint_ref as fx


def steps_of(lpS, thr, n):
    """(step of each entry (-1: never used), stable decreasing order of thr).  thr None: thresholding disabled."""
    if thr is None:
        return np.zeros(n, dtype=np.int64), np.array([0])
    thr = np.asarray(thr, dtype=np.float64)
    ordr = np.argsort(-thr, kind="stable")
    st = np.full(len(lpS), -1, dtype=np.int64)
    for k in range(thr.size - 1, -1, -1):
        st[np.asarray(lpS) > thr[ordr[k]]] = k
    return st, ordr


def literal(G, ind_row, cols, beta, same, lpS, thr):
    """R's snp_PRS for one keep set: (nr x nthr) fp64, columns in the caller's threshold order."""
    G = np.asarray(G)
    X = G[np.asarray(ind_row) - 1].astype(np.float64)
    X[X == 3] = np.nan
    cols = np.asarray(cols) - 1
    beta = np.asarray(beta, dtype=np.float64)
    same = np.ones(cols.size, dtype=bool) if same is None else np.asarray(same, dtype=bool)
    st, ordr = steps_of(lpS, thr, cols.size)
    out = np.empty((X.shape[0], ordr.size))
    last = np.zeros(X.shape[0])
    for k, i in enumerate(ordr):
        ind = np.flatnonzero(st == k)
        inc = np.zeros(X.shape[0])
        with np.errstate(invalid="ignore", over="ignore"):
            for j in ind:
                inc = inc + X[:, cols[j]] * ((2 * same[j] - 1) * beta[j])
            cst = 0.0
            for j in ind[~same[ind]]:
                cst += beta[j]
            last = last + (inc + 2 * cst)
        out[:, i] = last
    return out


def set_exponent(beta, same):
    v = np.asarray(beta, dtype=np.float64) * np.where(same, 1.0, -1.0)
    m = float(np.max(np.abs(v))) if v.size else 0.0
    return v, fx.pick_e(m, 0, 60)


def dosage_bytes(raw, code256, D):
    """A dosage FBM.code256 as the device reads it: (value bytes round(D code256[raw]), NA mask)."""
    code = np.asarray(code256, dtype=np.float64)
    isna = np.isnan(code)
    vals = np.where(isna, 0, np.rint(D * np.where(isna, 0, code))).astype(np.int64)
    raw = np.asarray(raw)
    return vals[raw], isna[raw]


def exact(G, ind_row, cols, beta, same, lpS, thr, D=None, na_mask=None):
    """bsg_prs_grid for one keep set: (nr x nthr) fp64, columns in the caller's threshold order.  Hard calls: G holds the
    codes (3 = NA).  Dosages (D given): G holds the value bytes, na_mask the NA codes; the slice totals take the
    reversed-allele constant times D and the score is divided by D once."""
    G = np.asarray(G)
    rows = G[np.asarray(ind_row) - 1]
    narows = (rows == 3) if D is None else np.asarray(na_mask)[np.asarray(ind_row) - 1]
    cols = np.asarray(cols) - 1
    same = np.ones(cols.size, dtype=bool) if same is None else np.asarray(same, dtype=bool)
    v, e = set_exponent(beta, same)
    Dg = fx.digits(fx.quantise(v, e), 8)                       # (len, 8)
    st, ordr = steps_of(lpS, thr, cols.size)
    nr = rows.shape[0]
    out = np.empty((nr, ordr.size))
    tot = np.zeros((nr, 8), dtype=object)                      # Python ints: exact
    na = np.zeros(nr, dtype=bool)
    for k, i in enumerate(ordr):
        ind = np.flatnonzero(st == k)
        if ind.size:
            # repeated columns: their digits add up first (exact integers), so the product runs over distinct columns
            u, inv = np.unique(cols[ind], return_inverse=True)
            Dk = Dg[ind]
            Du = np.zeros((u.size, 8), dtype=np.int64)
            np.add.at(Du, inv, Dk)
            A = rows[:, u].astype(np.int64)
            na |= narows[:, u].any(axis=1)
            part = np.rint(fx.partials(A, Du)).astype(np.int64).astype(object)
            rev = ~same[ind]
            kc = (-2 * (D or 1) * Dk[rev].sum(axis=0)).astype(object) if rev.any() else np.zeros(8, dtype=object)
            tot = tot + part + kc[None, :]
        acc = np.zeros(nr)
        for s in range(7, -1, -1):
            acc = fx._add_scaled(acc, np.array([int(t) for t in tot[:, s]], dtype=np.int64), 8 * s - e, fused=False)
        if D is not None:
            acc = acc / D
        acc[na] = np.nan
        out[:, i] = acc
    return out


def grid(G, ind_row, all_keep, betas, lpS, thr, fn=exact):
    """snp_grid_PRS: columns (ic - 1) n_thr + t over the keep sets in chromosome-major order."""
    betas, lpS = np.asarray(betas, dtype=np.float64), np.asarray(lpS, dtype=np.float64)
    cols = []
    for chrom in all_keep:
        for s in chrom:
            s = np.asarray(s, dtype=np.int64)
            cols.append(fn(G, ind_row, s, betas[s - 1], None, lpS[s - 1], thr))
    return np.concatenate(cols, axis=1) if cols else np.zeros((len(ind_row), 0))
