"""Exact host model of the matvec engine's arithmetic (bsg_pmv.cu, bsg_pmv_shared.cuh, bsg_naell.cu).

The engine claims that X.y and Xt.y have exactly one data-dependent rounding step after quantisation: the vector is
quantised once to fixed point, every digit-slice sum is an exact integer whatever kernel, split or staging computed it,
and the fp64 work is a fixed sequence per output.  This module restates that arithmetic in NumPy and Python integers,
so a product computed on the device can be compared with it byte for byte.

Inputs are the decoded codes (n x m, values 0 / 1 / 2 and 3 for a missing value), the 1-based selections, the vector
and the optional scaling.  The steps:

* values (make_vals): z = x / s, v1 = (c - 3) z, both correctly rounded (the build does not use fast-math);
* maxima and exponent: e = pick_e(max |v|, hb, bits) = bits - frexp_exponent(max |v|) - hb (0 for a zero or non-finite
  maximum).  hb = hb_bits(largest index multiplicity) wherever duplicates of a column or row are summed before the
  digits are taken or before the missing-value lists add them up (see `prod_T`);
* quantisation: Q = rint(v 2^e), ties to even (__double2ll_rn); scatters of duplicates add as wrapping int64, so an
  overflow shows here as it does on the device;
* digits: signed base-256 digits by `peel`, 8 slices (one vector, |Q| < 2^60) or 4 + 4 (two vectors, |Q| < 2^30);
* partials: per output line and slice, the exact integer sum of code x digit (raw plane, a missing value counting 3)
  and of flag x digit (missing-value plane) or high-bit x digit.  |digit x code| <= 384, so an fp64 GEMM of the digit
  matrix is exact for any contraction shorter than 2^53 / 384;
* missing-value lists: k_corr delivers the missing-value sum of a line as the sum of the low 32-bit halves and the sum
  of the high halves of its row sums (rows of 8 entries).  The model splits every entry on its own, which equals the
  row split whenever no row's low halves carry past 2^32.  That always holds when the line has one non-zero entry
  per row, and for vectors whose quantised entries have zero low halves (dyadic vectors with few significant bits).
  With scaling the X.y result does not depend on the split at all (the missing-value combine has two non-zero slices
  and rounds once);
* combine<NS>: top-down fp64 sum of the NS scaled slice totals, scalbn(v, k) as the device inlines it (one multiply for
  |k| < 1022, two for |k| < 2044, four beyond), the multiply of the last slice fused with its add;
* finish formulas of k_finish_prod (finish_prod_value), k_finish_cprod, k_finish_prod_pair;
* the term C = sum_k c_k z_k of k_prep1 in its exact order: 128 blocks x 256 threads, a strided serial loop per thread,
  the xor butterfly of each warp, the 8 warp sums of a block in order, then the 128 block partials in order.

Where nvcc contracts a multiply and an add, the model does the same.  `cuobjdump -sass` of libbsgpu.so (sm_90a, nvcc
12.9, -O3) shows:
  * k_prep1: `DFMA R18, R22, R18, R8` in the mode-1 loop: cz = fma(center[k], z, cz); `DADD R20, R22, -3` then
    `DMUL R20, R20, R18`: v1 = (c - 3) * z, not contracted;
  * k_finish_cprod: `DFMA R6, R6, -R2, R18`: out = fma(-c, Y - N, G) / s;
  * k_finish_prod: the slice-0 term of the combine is `DFMA R4, R6, R2, R4` (2^k times the pre-scaled slice total
    plus the accumulator), the other slices are DMUL + DADD; C is summed with DADD from 0.0 in block order.
The fused slice-0 multiply and the split scalbn only change a result whose scaled slice totals are subnormal (vectors
of subnormal size); in every other range the products by powers of two are exact.

Dosage FBM.code256 handles (bsg_dosage.cu, `dosage_*`) share the vector side: X.y takes prep_T's digits (hb = 0, one
digit block per selected column), Xt.y k_prep1 + k_quantise's scatter by physical sample (hb_bits(row multiplicity)).
The matrix operand is q = nearbyint(D code256[b]) in 0..255 (an NA byte counts 0), so |digit x q| <= 32,640 and a
k-split of 65,536 contraction indices stays within int32; the partials are exact integers as above.  The same SASS shows:
  * k_finish_dprod: every slice of the combine is DMUL + DADD, slice 0 included (`/*1970*/ DADD R8, R8, R10`): no fused
    last slice (combine(..., fused0=False)); then the IEEE division by D; C summed by DADD from 0.0 in block order; and
    `/*2ad0*/ DADD R8, -R8, R2`: full = R / D - C;
  * k_finish_dcprod: the same combine (`/*1940*/ DADD R8, R8, R10`), R / D, then `/*20f0*/ DFMA R8, -R2, R8, R6`:
    out = fma(-c, Y, R / D), divided by s;
  * k_lit_prod: `/*07d0*/ DFMA R28, R30, R10, R28`: s = fma(x_t, (code256[b] - c_t) / s_t, s);
  * k_lit_cprod: `/*0700*/ DFMA R16, R16, R12, RZ` then `/*0950*/ DFMA R16, R10, R12, R16`: lane sums by fma, then the
    butterfly by DADD (`/*2730*/ DADD R10, R10, R16`);
  * k_proj_literal<false> / <true>: `/*06c0*/ DFMA R12, R16, R16, R12` / `/*0660*/ DFMA R14, R16, R16, R14`:
    rss = fma(x, x, rss); `/*08d0*/ DFMA R18, R20, R16, R18` / `/*0870*/ DFMA R18, R20, R16, R18`: XV = fma(V, x, XV).
    x = (v - c) / s is a DADD and an IEEE division (MUFU.RCP64H, DFMA refinement, slow-path CALL) in every literal loop.
(Offsets within each function of `cuobjdump -sass libbsgpu.so`.)  Accuracy of X.y: |out - exact| <= sum_t (q_t / D)
|z_t| ... as above with g = q / D: 2^(-e-1) sum_t q_t / D + a few ulps of |out| + the rounding of 1 / D and of C.

Accuracy this proves (one vector, 61-bit format): |out - exact| <= sum_t |g_t| 2^(-e-1) (quantisation, g the
codes or scaled codes the vector meets) + a few ulps of |out| (combine) + the rounding of C.  e = 60 - ex - hb with
max |v| < 2^ex, so the quantisation term is below 2^(-61+hb) max|v| sum_t |g_t|: about 4e-19 max|v| sum|g| without
duplicate indices.  Two vectors per pass: the same with 30 for 60 (about 5e-10 max|v| sum|g|).
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

SUMCZ_BLOCKS, PREP_THREADS = 128, 256
_M32 = (1 << 32) - 1


# ---- scalars ---------------------------------------------------------------------------------------------------------
def hb_bits(maxmult: int) -> int:
    """ceil(log2(maxmult)), plus one from 8 on: below 2^53 rint cannot reach 2^(60-b), above it can."""
    b = 0
    while (1 << b) < maxmult:
        b += 1
    return b + 1 if b >= 8 else b


def max_mult(idx) -> int:
    idx = np.asarray(idx)
    if idx.size == 0:
        return 1
    return int(np.max(np.unique(idx, return_counts=True)[1]))


def pick_e(m: float, hb: int, bits: int) -> int:
    if m > 0 and math.isfinite(m):
        return bits - math.frexp(m)[1] - hb
    return 0


def fma(a: float, b: float, c: float) -> float:
    """a * b + c rounded once (Fraction arithmetic; int / int true division is correctly rounded).  Non-finite operands
    give what the fp64 ops give; an exact zero keeps IEEE's sign (+0 from a cancellation, the signed sum when a b = 0);
    an overflow is an infinity."""
    a, b, c = float(a), float(b), float(c)
    if not (math.isfinite(a) and math.isfinite(b) and math.isfinite(c)):
        return a * b + c
    r = Fraction(a) * Fraction(b) + Fraction(c)
    if r == 0:
        return a * b + c if (a == 0.0 or b == 0.0) else 0.0
    try:
        return float(r)
    except OverflowError:
        return math.copysign(math.inf, r)


# ---- vector preparation ---------------------------------------------------------------------------------------------
def make_vals(mode, x, center=None, scale=None):
    x = np.asarray(x, dtype=np.float64)
    if mode == 0:
        return x.copy(), np.zeros_like(x)
    if mode == 2:
        return x.copy(), np.asarray(center, dtype=np.float64).copy()
    z = x / np.asarray(scale, dtype=np.float64)
    return z, (np.asarray(center, dtype=np.float64) - 3.0) * z


def sum_cz(center, z) -> float:
    """C = sum_k c_k z_k in k_prep1's order (grid of 128 x 256, fma in the thread loop) and the finish kernel's."""
    center, z = np.asarray(center, dtype=np.float64), np.asarray(z, dtype=np.float64)
    nt = SUMCZ_BLOCKS * PREP_THREADS
    cz = np.zeros(nt)
    for k0 in range(0, z.size, nt):
        for t in range(min(nt, z.size - k0)):
            cz[t] = fma(center[k0 + t], z[k0 + t], cz[t])
    lanes = cz.reshape(SUMCZ_BLOCKS, PREP_THREADS // 32, 32)
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, :, idx ^ o]
    cpart = np.zeros(SUMCZ_BLOCKS)
    for w in range(PREP_THREADS // 32):
        cpart = cpart + lanes[:, w, 0]
    C = 0.0
    for b in range(SUMCZ_BLOCKS):
        C += float(cpart[b])
    return C


def quantise(v, e: int) -> np.ndarray:
    """Q = rint(v 2^e), ties to even.  |v 2^e| < 2^61 by construction of e, so the double is exact in int64."""
    return np.rint(np.ldexp(np.asarray(v, dtype=np.float64), e)).astype(np.int64)


def scatter(q, idx0, length: int) -> np.ndarray:
    """Q[idx0[k]] += q[k] as wrapping int64 (the device's integer atomics)."""
    out = np.zeros(length, dtype=np.int64)
    with np.errstate(over="ignore"):
        np.add.at(out, np.asarray(idx0, dtype=np.int64), np.asarray(q, dtype=np.int64))
    return out


def digits(q, ns: int) -> np.ndarray:
    """Signed base-256 digits by `peel` (low byte as int8, then (q - d) >> 8), (len, ns) int64."""
    q = np.array(q, dtype=np.int64)
    out = np.empty((q.size, ns), dtype=np.int64)
    with np.errstate(over="ignore"):
        for s in range(ns):
            d = ((q & 0xFF) ^ 0x80) - 0x80
            out[:, s] = d
            q = (q - d) >> 8
    return out


def partials(A, D) -> np.ndarray:
    """Exact sum_t A[l, t] D[t, s]: small integers, so the fp64 product is exact."""
    A = np.asarray(A, dtype=np.float64)
    D = np.asarray(D, dtype=np.float64)
    if A.shape[1] == 0:
        return np.zeros((A.shape[0], D.shape[1]), dtype=np.int64)
    return np.rint(A @ D).astype(np.int64)


def split_lists(flags, qna) -> tuple[np.ndarray, np.ndarray]:
    """Missing-value lists: per line, sum of the low 32-bit halves and of the high halves of its entries."""
    q = np.asarray(qna, dtype=np.int64)
    lo = (q & _M32).astype(np.float64)   # < 2^32: exact; sums stay below 2^53 for any realistic line
    hi = (q >> 32).astype(np.float64)
    F = np.asarray(flags, dtype=np.float64)
    return np.rint(F @ lo).astype(np.int64), np.rint(F @ hi).astype(np.int64)


# ---- combine ----------------------------------------------------------------------------------------------------------
def _mul_pow2(t: float, k: int) -> float:
    return float(Fraction(t) * (Fraction(2) ** k))


def _add_scaled1(acc: float, v: int, k: int, fused: bool) -> float:
    t = float(v)
    if t == 0.0 or k == 0:
        return acc + t
    k = max(-2200, min(2200, k))
    a = abs(k)
    if a < 1022:
        last = k
    elif a < 2044:
        h = int(k / 2)
        t, last = _mul_pow2(t, h), k - h
    else:
        q4 = int(k / 4)
        for _ in range(3):
            t = _mul_pow2(t, q4)
        last = k - 3 * q4
    if fused:
        return float(Fraction(acc) + Fraction(t) * (Fraction(2) ** last))
    return acc + _mul_pow2(t, last)


def _add_scaled(acc: np.ndarray, v: np.ndarray, k: int, fused: bool) -> np.ndarray:
    vf = v.astype(np.float64)
    if abs(k) < 1022:
        t = np.ldexp(vf, k)
        if not np.any((t != 0) & (np.abs(t) < 2.0 ** -1022)):
            return acc + t   # products by 2^k exact: fused or not, one rounding in the add
    return np.array([_add_scaled1(float(a), int(x), k, fused) for a, x in zip(acc, v)])


def combine(raw, na, c0: int, c1: int, e: int, ns: int = 8, s0: int = 0, fused0: bool = True) -> np.ndarray:
    """combine<NS>: sum over s = NS-1 .. 0 of scalbn(c0 raw[s0+s] + c1 na[s0+s], 8 s - e), top down.  fused0: the last
    slice's multiply is fused with its add (the 2-bit finish kernels; the dosage ones keep DMUL + DADD)."""
    raw = np.asarray(raw, dtype=np.int64)
    na = np.zeros_like(raw) if na is None else np.asarray(na, dtype=np.int64)
    acc = np.zeros(raw.shape[0])
    for s in range(ns - 1, -1, -1):
        v = np.zeros(raw.shape[0], dtype=np.int64)
        if c0:
            v = v + c0 * raw[:, s0 + s]
        if c1:
            v = v + c1 * na[:, s0 + s]
        acc = _add_scaled(acc, v, 8 * s - e, fused=fused0 and s == 0)
    return acc


# ---- products ---------------------------------------------------------------------------------------------------------
def _sel(G, ir, ic):
    G = np.asarray(G)
    n, m = G.shape
    ir = np.arange(1, n + 1) if ir is None else np.asarray(ir, dtype=np.int64)
    ic = np.arange(1, m + 1) if ic is None else np.asarray(ic, dtype=np.int64)
    return G, ir - 1, ic - 1


def _scaling(center, scale):
    """None when identity (center 0, scale 1): the view then takes the unscaled path."""
    if center is None:
        return None, None
    c, s = np.asarray(center, dtype=np.float64), np.asarray(scale, dtype=np.float64)
    if np.all(c == 0.0) and np.all(s == 1.0):
        return None, None
    return c, s


def _prod_finish(raw, na, has_na, scaled, e0, e1, C, ns=8, s0=0):
    if scaled:
        R = combine(raw, None, 1, 0, e0, ns, s0)
        Nw = combine(raw * 0, na, 0, 1, e1, ns, s0) if has_na else 0.0
        return (R + Nw) - C
    return combine(raw, na, 1, -3 if has_na else 0, e0, ns, s0)


def prod_T(G, ir, iy, y, center=None, scale=None, lists=False, legacy_hb=False):
    """X.y on the SNP-major copy (prodvec_T: k_pmvT / k_pmvT_lines / k_pmvT2<1> + missing-value lists).

    Lines are all n samples, the contraction runs over the selected columns in selection order (a duplicate is a
    repeated line with its own digits).  With `lists` the missing-value vector is scattered by physical SNP and summed by
    k_corr; the exponent then leaves hb_bits(column multiplicity) of head-room.  legacy_hb: hb = 0 there, as before
    that head-room was added (the sums of duplicates then wrap)."""
    G, r0, c0 = _sel(G, ir, iy)
    n, m = G.shape
    has_na = bool(np.any(G == 3))
    c, s = _scaling(center, scale)
    scaled = c is not None
    mode = 1 if scaled else 0
    v0, v1 = make_vals(mode, y, c, s)
    if not (np.all(np.isfinite(v0)) and np.all(np.isfinite(v1))):
        return np.full(r0.size, np.nan)
    hb = hb_bits(max_mult(c0)) if (lists and has_na and not legacy_hb) else 0
    e0 = pick_e(float(np.max(np.abs(v0), initial=0.0)), hb, 60)
    e1 = pick_e(float(np.max(np.abs(v1), initial=0.0)), hb, 60)
    q0, q1 = quantise(v0, e0), quantise(v1, e1)
    Gs = G[:, c0]
    raw = partials(Gs, digits(q0, 8))
    na = np.zeros_like(raw)
    if has_na and lists:
        qna = scatter(q1 if scaled else q0, c0, m)
        lo, hi = split_lists(G == 3, qna)
        na[:, 0], na[:, 4] = lo, hi
    elif has_na:
        na = partials(Gs == 3, digits(q1 if scaled else q0, 8))
    C = sum_cz(c, v0) if scaled else 0.0
    return _prod_finish(raw, na, has_na, scaled, e0, e1, C)[r0]


def prod_pmv(G, ir, iy, y, center=None, scale=None):
    """X.y on the sample-major copy (k_pmv, lines = samples): the vector is scattered by physical SNP first, with
    hb_bits(column multiplicity) of head-room; flag plane for missing values."""
    G, r0, c0 = _sel(G, ir, iy)
    n, m = G.shape
    has_na = bool(np.any(G == 3))
    c, s = _scaling(center, scale)
    scaled = c is not None
    mode = 1 if scaled else 0
    v0, v1 = make_vals(mode, y, c, s)
    if not (np.all(np.isfinite(v0)) and np.all(np.isfinite(v1))):
        return np.full(r0.size, np.nan)
    hb = hb_bits(max_mult(c0))
    e0 = pick_e(float(np.max(np.abs(v0), initial=0.0)), hb, 60)
    e1 = pick_e(float(np.max(np.abs(v1), initial=0.0)), hb, 60)
    q0, q1 = scatter(quantise(v0, e0), c0, m), scatter(quantise(v1, e1), c0, m)
    raw = partials(G, digits(q0, 8))
    na = partials(G == 3, digits(q1 if scaled else q0, 8)) if has_na else np.zeros_like(raw)
    C = sum_cz(c, v0) if scaled else 0.0
    return _prod_finish(raw, na, has_na, scaled, e0, e1, C)[r0]


def cprod(G, ir, iy, y, center=None, scale=None, lists=False):
    """Xt.y (k_pmv over the SNP-major copy, lines = selected columns): y scattered by physical sample with
    hb_bits(row multiplicity); the missing-value sums from the flag plane or from the lists; k_finish_cprod."""
    G, r0, c0 = _sel(G, ir, iy)
    n, m = G.shape
    has_na = bool(np.any(G == 3))
    c, s = _scaling(center, scale)
    y = np.asarray(y, dtype=np.float64)
    if not np.all(np.isfinite(y)):
        return np.full(c0.size, np.nan)
    e = pick_e(float(np.max(np.abs(y), initial=0.0)), hb_bits(max_mult(r0)), 60)
    q = scatter(quantise(y, e), r0, n)
    A = G[:, c0].T
    raw = partials(A, digits(q, 8))
    na = np.zeros_like(raw)
    if has_na and lists:
        lo, hi = split_lists(A == 3, q)
        na[:, 0], na[:, 4] = lo, hi
    elif has_na:
        na = partials(A == 3, digits(q, 8))
    Gv = combine(raw, na, 1, -3 if has_na else 0, e)
    if c is None:
        return Gv
    N = combine(raw * 0, na, 0, 1, e) if has_na else np.zeros(c0.size)
    sum_hi, sum_lo = int(np.sum(q >> 32)), int(np.sum(q & _M32))
    Y = math.ldexp(float(sum_hi), 32 - e) + math.ldexp(float(sum_lo), -e)
    YN = Y - N
    return np.array([fma(-cj, d, g) for cj, d, g in zip(c, YN, Gv)]) / s


def prod_pair(G, ir, iy, ya, yb, center=None, scale=None):
    """Two vectors per pass over the SNP-major copy (prodvec_T_pair, k_quantT<2>, k_finish_prod_pair): 30-bit fixed
    point per vector, slices 0..3 and 4..7; flag plane for missing values.  yb may be None."""
    G, r0, c0 = _sel(G, ir, iy)
    n, m = G.shape
    has_na = bool(np.any(G == 3))
    c, s = _scaling(center, scale)
    scaled = c is not None
    mode = 1 if scaled else 0
    Gs = G[:, c0]
    D, Dn, scal = np.zeros((c0.size, 8), np.int64), np.zeros((c0.size, 8), np.int64), []
    for vv, y in enumerate((ya, yb)):
        if y is None:
            scal.append(None)
            continue
        v0, v1 = make_vals(mode, y, c, s)
        e0 = pick_e(float(np.max(np.abs(v0), initial=0.0)), 0, 30)
        e1 = pick_e(float(np.max(np.abs(v1), initial=0.0)), 0, 30)
        q0, q1 = quantise(v0, e0), quantise(v1, e1)
        D[:, 4 * vv:4 * vv + 4] = digits(q0, 4)
        Dn[:, 4 * vv:4 * vv + 4] = digits(q1 if scaled else q0, 4)
        scal.append((e0, e1, sum_cz(c, v0) if scaled else 0.0))
    raw = partials(Gs, D)
    na = partials(Gs == 3, Dn) if has_na else np.zeros_like(raw)
    out = []
    for vv, sc in enumerate(scal):
        out.append(None if sc is None else _prod_finish(raw, na, has_na, scaled, sc[0], sc[1], sc[2], 4, 4 * vv)[r0])
    return out


def prod_and_rowSumsSq_XV(G, ir, iy, center, scale, V, pair=True, lists=False):
    """XV of prod_and_rowSumsSq: columns of V two per pass (pair, K >= 2), else one 61-bit X.y per column."""
    V = np.asarray(V, dtype=np.float64)
    V = V.reshape(V.shape[0], -1)
    K = V.shape[1]
    cols = []
    if pair and K >= 2:
        for k in range(0, K, 2):
            a, b = prod_pair(G, ir, iy, V[:, k], V[:, k + 1] if k + 1 < K else None, center, scale)
            cols += [a] + ([b] if b is not None else [])
    else:
        cols = [prod_T(G, ir, iy, V[:, k], center, scale, lists=lists) for k in range(K)]
    return np.stack(cols, axis=1)


RSS_BLOCKS = 64


def _rss_weights(c, s):
    """k_rss_weights: w = 1 / s^2, a = (1 - 2c) w, nv = (fma(-6, c, 5) + c c) w, and T = sum c c w in the kernel's order
    (64 x 256 grid-stride threads accumulating fma(c c, w, t), xor butterfly, 8 warp sums in order, then
    k_rss_final's sum of the 64 block partials in order)."""
    w = 1.0 / (s * s)
    a = (1.0 - 2.0 * c) * w
    cc = c * c
    nv = (np.array([fma(-6.0, float(cj), 5.0) for cj in c]) + cc) * w
    nt = RSS_BLOCKS * 256
    t = np.zeros(nt)
    for k0 in range(0, c.size, nt):
        for j in range(min(nt, c.size - k0)):
            t[j] = fma(float(cc[k0 + j]), float(w[k0 + j]), float(t[j]))
    lanes = t.reshape(RSS_BLOCKS, 8, 32)
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, :, idx ^ o]
    tpart = np.zeros(RSS_BLOCKS)
    for k in range(8):
        tpart = tpart + lanes[:, k, 0]
    T = 0.0
    for b in range(RSS_BLOCKS):
        T += float(tpart[b])
    return a, w, nv, T


def _plane_sums(Gl, sel_phys, m, x1, x2, plane, pmv):
    """view_planes_dev, X side: R = sum code x1, P = sum plane x2 (plane 'hi': codes 2 and 3; 'na': code 3, with x2 = x1
    sharing one digit block), through k_finish_planes' combine.  pmv: k_pmv over the sample-major copy (vectors
    scattered by physical SNP with hb_bits(multiplicity)); else k_pmvT (one digit block per selected column, hb = 0).
    Gl: lines x physical SNPs (pmv) or lines x selected columns (k_pmvT)."""
    two = plane == "hi"
    hb = hb_bits(max_mult(sel_phys)) if pmv else 0
    e0 = pick_e(float(np.max(np.abs(x1), initial=0.0)), hb, 60)
    e1 = pick_e(float(np.max(np.abs(x2), initial=0.0)), hb, 60) if two else e0
    q1, q2 = quantise(x1, e0), quantise(x2, e1)
    if pmv:
        q1, q2 = scatter(q1, sel_phys, m), scatter(q2, sel_phys, m)
    flags = (Gl >= 2) if plane == "hi" else (Gl == 3)
    R = combine(partials(Gl, digits(q1, 8)), None, 1, 0, e0)
    P = combine(np.zeros((Gl.shape[0], 8), np.int64), partials(flags, digits(q2 if two else q1, 8)), 0, 1, e1)
    return R, P


def row_sums_sq(G, ir, iy, center, scale, pmv=False):
    """rowSumsSq of prod_and_rowSumsSq: (t1 + t2) + T with t1 = (R(a) + 2 H(w)) + 0, t2 = (-N(nv)) + 0 (missing values
    only, else 0.0).  The coefficients 1, 2, 0, -1 of k_finish_planes make its products exact, so where nvcc fuses
    them does not matter.  pmv: the sample-major kernel (a handle holding that copy and no missing value)."""
    G, r0, c0 = _sel(G, ir, iy)
    n, m = G.shape
    has_na = bool(np.any(G == 3))
    c, s = _scaling(center, scale)
    if c is None:  # identity scaling: the view keeps no center / scale; the kernel writes the constants
        c, s = np.zeros(c0.size), np.ones(c0.size)
    a, w, nv, T = _rss_weights(c, s)
    Gl = G if pmv else G[:, c0]
    R, H = _plane_sums(Gl, c0, m, a, w, "hi", pmv)
    t1 = (R + 2.0 * H) + 0.0
    t2 = 0.0
    if has_na:
        _, N = _plane_sums(Gl, c0, m, nv, nv, "na", pmv)
        t2 = (-N) + 0.0
    return ((t1 + t2) + T)[r0]


# ---- dosage FBM.code256 (bsg_dosage.cu) -------------------------------------------------------------------------------
def dosage_table(code256):
    """dosage_scale_of: the smallest D in 1..255 with D v within 1e-9 of an integer in 0..255 for every non-NaN v of the
    table (0 when none, or when an entry is infinite); the byte map q = nearbyint(D v) (NA -> 0) of the value copy; the NA
    flags.  Returns (D, q, na); q is None when D = 0."""
    code = np.asarray(code256, dtype=np.float64)
    na = np.isnan(code)
    v = code[~na]
    if not np.all(np.isfinite(v)):
        return 0, None, na
    for D in range(1, 256):
        t = D * v
        r = np.rint(t)
        if np.all((np.abs(t - r) <= 1e-9) & (r >= 0) & (r <= 255)):
            q = np.where(na, 0.0, np.rint(D * np.where(na, 0.0, code))).astype(np.uint8)
            return D, q, na
    return 0, None, na


def _dsel(raw, ir, ic):
    raw = np.asarray(raw, dtype=np.uint8)
    n, m = raw.shape
    r0 = np.arange(n) if ir is None else np.asarray(ir, dtype=np.int64) - 1
    c0 = np.arange(m) if ic is None else np.asarray(ic, dtype=np.int64) - 1
    return raw, r0, c0


def dosage_prod(raw, code256, ir, ic, y, center=None, scale=None):
    """X.y on a dosage handle (dosage_prep_cols -> prep_T, k_dmvT, k_finish_dprod, k_na_rows, k_gather_rows).

    Lines are the selected columns in selection order, each with its own digits of z = y / s (or y), so hb = 0; the
    contraction runs over q[byte] of the value copy (an NA byte counts 0); R = combine<8> of the slice totals, then R / D,
    then - C with scaling.  Every sample holding an NA byte in a selected column is NaN, then the rows are gathered.  A
    non-finite z or (c - 3) z (k_prep1's flag) makes every output NaN (the device-pointer forms; the host forms re-run
    `lit_prod` instead)."""
    D, qmap, isna = dosage_table(code256)
    raw, r0, c0 = _dsel(raw, ir, ic)
    c, s = _scaling(center, scale)
    scaled = c is not None
    with np.errstate(all="ignore"):
        v0, v1 = make_vals(1 if scaled else 0, y, c, s)
    if not (np.all(np.isfinite(v0)) and np.all(np.isfinite(v1))):
        return np.full(r0.size, np.nan)
    e = pick_e(float(np.max(np.abs(v0), initial=0.0)), 0, 60)
    part = partials(qmap[raw[:, c0]], digits(quantise(v0, e), 8))
    full = combine(part, None, 1, 0, e, fused0=False) / D
    if scaled:
        full = full - sum_cz(c, v0)
    full[isna[raw[:, c0]].any(axis=1)] = np.nan
    return full[r0]


def dosage_cprod(raw, code256, ir, ic, y, center=None, scale=None):
    """Xt.y on a dosage handle (dosage_prep_rows -> k_prep1 + k_quantise, k_digits_rows, k_dmv, k_finish_dcprod,
    k_na_lines / k_na_cols).

    y is quantised with hb_bits(row multiplicity) and scattered by physical sample; lines are the selected columns, the
    contraction runs over all n samples of the value copy; R = combine<8> / D; with scaling out = fma(-c, Y, R) / s with
    Y = scalbn(sum_hi, 32 - e) + scalbn(sum_lo, -e) from the exact sum of Q.  A line holding an NA byte in a selected row
    is NaN.  A non-finite y, center or 1 / scale makes every output NaN (k_check_scaling)."""
    D, qmap, isna = dosage_table(code256)
    raw, r0, c0 = _dsel(raw, ir, ic)
    n = raw.shape[0]
    c, s = _scaling(center, scale)
    y = np.asarray(y, dtype=np.float64)
    with np.errstate(all="ignore"):
        bad = not np.all(np.isfinite(y)) or (c is not None and not (np.all(np.isfinite(c)) and np.all(np.isfinite(1.0 / s))))
    if bad:
        return np.full(c0.size, np.nan)
    e = pick_e(float(np.max(np.abs(y), initial=0.0)), hb_bits(max_mult(r0)), 60)
    q = scatter(quantise(y, e), r0, n)
    part = partials(qmap[raw[:, c0]].T, digits(q, 8))
    R = combine(part, None, 1, 0, e, fused0=False) / D
    if c is None:
        out = R
    else:
        sum_hi, sum_lo = int(np.sum(q >> 32)), int(np.sum(q & _M32))
        Y = math.ldexp(float(sum_hi), 32 - e) + math.ldexp(float(sum_lo), -e)
        out = np.array([fma(-cj, Y, Rj) for cj, Rj in zip(c, R)]) / s
    rows = np.unique(r0)
    out[isna[raw[np.ix_(rows, c0)]].any(axis=0)] = np.nan
    return out


def _lit_terms(code, raw, r0, col, cj, sj):
    """(code256[b] - c) / s for the bytes of one column at rows r0 (one IEEE subtraction and division each)."""
    with np.errstate(all="ignore"):
        return (np.asarray(code, dtype=np.float64)[raw[r0, col]] - cj) / sj


def _fma_vec(a, b, c):
    a, b, c = np.broadcast_arrays(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64),
                                  np.asarray(c, dtype=np.float64))
    return np.array([fma(x, y, z) for x, y, z in zip(a.ravel(), b.ravel(), c.ravel())]).reshape(a.shape)


def _lit_scaling(center, scale, nc):
    c, s = _scaling(center, scale)
    return (np.zeros(nc), np.ones(nc)) if c is None else (c, s)


def lit_prod(raw, code256, ir, ic, x, center=None, scale=None):
    """k_lit_prod: one thread per selected row, a serial loop over the selected columns in order,
    s = fma(x_t, (code256[b] - c_t) / s_t, s) from 0 (non-finite values propagate as in fp64)."""
    raw, r0, c0 = _dsel(raw, ir, ic)
    c, s = _lit_scaling(center, scale, c0.size)
    x = np.asarray(x, dtype=np.float64)
    acc = np.zeros(r0.size)
    for t in range(c0.size):
        acc = _fma_vec(_lit_terms(code256, raw, r0, c0[t], c[t], s[t]), x[t], acc)
    return acc


def lit_cprod(raw, code256, ir, ic, x, center=None, scale=None):
    """k_lit_cprod: one warp per selected column; lane l sums rows l, l + 32, ... with s = fma(term, x_i, s) from 0,
    then the xor butterfly 16, 8, 4, 2, 1 (DADD) and lane 0's value."""
    raw, r0, c0 = _dsel(raw, ir, ic)
    c, s = _lit_scaling(center, scale, c0.size)
    x = np.asarray(x, dtype=np.float64)
    nr = r0.size
    out = np.empty(c0.size)
    for t in range(c0.size):
        term = _lit_terms(code256, raw, r0, c0[t], c[t], s[t])
        lanes = np.zeros(32)
        for i0 in range(0, nr, 32):
            k = min(32, nr - i0)
            lanes[:k] = _fma_vec(term[i0:i0 + k], x[i0:i0 + k], lanes[:k])
        idx = np.arange(32)
        with np.errstate(all="ignore"):
            for o in (16, 8, 4, 2, 1):
                lanes = lanes + lanes[idx ^ o]
        out[t] = lanes[0]
    return out


def proj_literal(P, code256, ir, ic, center, scale, V=None):
    """k_proj_literal<BYTES> (prod_and_rowSumsSq2's literal pass): one thread per selected row, a serial loop over the
    selected columns in order.  code256 given: P is the n x m code bytes, v = code256[b]; code256 None: P holds hard calls
    0 / 1 / 2 / 3 (3 = NA -> NaN).  x = (v - c) / s, rss = fma(x, x, rss), XV[:, k] = fma(V[j, k], x, XV[:, k]) from 0.
    Returns (XV, rss, na) with na = the rows where a selected column holds an NA."""
    P, r0, c0 = _dsel(P, ir, ic)
    c, s = _lit_scaling(center, scale, c0.size)
    code = np.r_[0.0, 1.0, 2.0, np.nan] if code256 is None else np.asarray(code256, dtype=np.float64)
    V = np.zeros((c0.size, 0)) if V is None else np.asarray(V, dtype=np.float64).reshape(c0.size, -1)
    rss, XV = np.zeros(r0.size), np.zeros((r0.size, V.shape[1]))
    na = np.zeros(r0.size, dtype=bool)
    for j in range(c0.size):
        x = _lit_terms(code, P, r0, c0[j], c[j], s[j])
        na |= np.isnan(code[P[r0, c0[j]]])
        rss = _fma_vec(x, x, rss)
        for k in range(V.shape[1]):
            XV[:, k] = _fma_vec(V[j, k], x, XV[:, k])
    return XV, rss, na


def exact_dosage_prod(raw, code256, ir, ic, y, center=None, scale=None):
    """X~ y over a dosage table in rationals: sum over the selected columns of (q / D - c) / s y; None where an NA byte
    meets the row."""
    D, qmap, isna = dosage_table(code256)
    raw, r0, c0 = _dsel(raw, ir, ic)
    c, s = _lit_scaling(center, scale, c0.size)
    w = [Fraction(float(yk)) / Fraction(float(sk)) for yk, sk in zip(y, s)]
    out = []
    for i in r0:
        b = raw[i, c0]
        if isna[b].any():
            out.append(None)
            continue
        out.append(sum(((Fraction(int(qmap[bb]), D) - Fraction(float(c[t]))) * w[t] for t, bb in enumerate(b)),
                       Fraction(0)))
    return out


# ---- exact references -------------------------------------------------------------------------------------------------
def exact_prod(G, ir, iy, y, center=None, scale=None):
    """X~ y in rationals: (g - c) / s over non-missing entries, 0 for a missing one (bedAccScaled)."""
    G, r0, c0 = _sel(G, ir, iy)
    c = np.zeros(c0.size) if center is None else np.asarray(center, dtype=np.float64)
    s = np.ones(c0.size) if scale is None else np.asarray(scale, dtype=np.float64)
    w = [Fraction(float(yk)) / Fraction(float(sk)) for yk, sk in zip(y, s)]
    out = []
    for i in r0:
        acc = Fraction(0)
        for t, j in enumerate(c0):
            g = int(G[i, j])
            if g != 3:
                acc += (g - Fraction(float(c[t]))) * w[t]
        out.append(acc)
    return out
