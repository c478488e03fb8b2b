"""The exact host model of the matvec arithmetic (tests/fixedpoint_ref.py) checked on its own, without a GPU: integer
totals of the digit slices, the accuracy bound it proves against rational arithmetic, agreement with the CPU oracle,
and the head-room rule for duplicate columns summed by the missing-value lists."""
import math
import os
from fractions import Fraction

import numpy as np
import pytest

from tests import fixedpoint_ref as fx

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _codes(rng, n, m, na_rate):
    G = rng.integers(0, 3, size=(n, m)).astype(np.uint8)
    G[rng.random((n, m)) < na_rate] = 3
    return G


@pytest.mark.parametrize("ns,bits", [(8, 60), (4, 30)])
def test_digit_slices_sum_to_the_exact_integer_total(rng, ns, bits):
    G = _codes(rng, 37, 101, 0.1)
    y = rng.normal(size=101) * 3.7
    e = fx.pick_e(float(np.max(np.abs(y))), 0, bits)
    q = fx.quantise(y, e)
    assert np.max(np.abs(q)) < 2 ** bits
    D = fx.digits(q, ns)
    assert np.all((D >= -128) & (D <= 127))
    assert all(sum(int(D[k, s]) << (8 * s) for s in range(ns)) == int(q[k]) for k in range(q.size))
    part = fx.partials(G, D)
    want = [sum(int(G[i, j]) * int(q[j]) for j in range(101)) for i in range(37)]
    assert [sum(int(part[i, s]) * 256 ** s for s in range(ns)) for i in range(37)] == want


def test_pick_e_edges():
    assert fx.pick_e(0.0, 0, 60) == 0 and fx.pick_e(float("inf"), 0, 60) == 0 and fx.pick_e(float("nan"), 3, 60) == 0
    assert fx.pick_e(1.0, 0, 60) == 59                    # frexp(1) = 0.5 * 2^1
    assert fx.pick_e(np.nextafter(1.0, 0), 0, 60) == 60   # just below one
    assert fx.pick_e(2.0 ** -1074, 0, 60) == 60 + 1073    # smallest subnormal
    for hb, mult in ((0, 1), (1, 2), (2, 3), (4, 16), (5, 17)):
        assert fx.hb_bits(mult) == hb
    # ties to even at 2^-e
    e = fx.pick_e(1.0, 0, 60)
    half = 2.0 ** (-e - 1)
    assert list(fx.quantise([half, 3 * half, -half, -3 * half], e)) == [0, 2, 0, -2]


def _bound(G, ir, ic, y, center, scale, bits, hb=0):
    """Quantisation + combine + C bound of one output vector (see the model's docstring)."""
    G, r0, c0 = fx._sel(G, ir, ic)
    s = np.ones(c0.size) if scale is None else np.asarray(scale)
    c = np.zeros(c0.size) if center is None else np.asarray(center)
    v = np.asarray(y) / s
    e = fx.pick_e(float(np.max(np.abs(v))), hb, bits)
    g = np.abs(np.where(G[np.ix_(r0, c0)] == 3, 0.0, G[np.ix_(r0, c0)] - c))  # |scaled code| each value meets
    gq = np.abs(G[np.ix_(r0, c0)]).astype(float) + 3 * np.abs(c - 3) * (G[np.ix_(r0, c0)] == 3)
    quant = (gq + g).sum(1) * 2.0 ** (-e - 1)
    if center is not None:  # v1 = (c - 3) z has its own exponent; bound it by the same formula
        e1 = fx.pick_e(float(np.max(np.abs((c - 3) * v))), hb, bits)
        quant = quant + 3 * (G[np.ix_(r0, c0)] == 3).sum(1) * 2.0 ** (-e1 - 1)
    mag = (g * np.abs(v)).sum(1) + np.abs(c * v).sum()
    return quant + 8 * 2.0 ** -52 * mag + 1e-300


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("na_rate", [0.0, 0.1])
def test_model_within_its_bound_of_the_exact_product(rng, scaled, na_rate):
    n, m = 23, 57
    G = _codes(rng, n, m, na_rate)
    ic = rng.integers(1, m + 1, 40)
    y = rng.normal(size=40)
    c, s = (rng.normal(size=40), rng.uniform(0.3, 2.0, size=40)) if scaled else (None, None)
    exact = fx.exact_prod(G, None, ic, y, c, s)
    for lists in (False, True):
        got = fx.prod_T(G, None, ic, y, c, s, lists=lists)
        hb = fx.hb_bits(fx.max_mult(ic - 1)) if lists and na_rate else 0
        err = np.array([abs(Fraction(float(a)) - b) for a, b in zip(got, exact)], dtype=float)
        assert np.all(err <= _bound(G, None, ic, y, c, s, 60, hb)), err
    got = fx.prod_pmv(G, None, ic, y, c, s)
    err = np.array([abs(Fraction(float(a)) - b) for a, b in zip(got, exact)], dtype=float)
    assert np.all(err <= _bound(G, None, ic, y, c, s, 60, fx.hb_bits(fx.max_mult(ic - 1))))
    # two vectors per pass: 30 bits each
    yb = rng.normal(size=40)
    a, b = fx.prod_pair(G, None, ic, y, yb, c, s)
    for got, yy in ((a, y), (b, yb)):
        exact = fx.exact_prod(G, None, ic, yy, c, s)
        err = np.array([abs(Fraction(float(x)) - w) for x, w in zip(got, exact)], dtype=float)
        assert np.all(err <= _bound(G, None, ic, yy, c, s, 30)), err


def test_cprod_model_within_its_bound(rng):
    n, m = 41, 29
    G = _codes(rng, n, m, 0.1)
    ir = rng.integers(1, n + 1, 50)
    y = rng.normal(size=50)
    c, s = rng.normal(size=m), rng.uniform(0.3, 2.0, size=m)
    for lists in (False, True):
        for cs in ((None, None), (c, s)):
            got = fx.cprod(G, ir, None, y, *cs, lists=lists)
            ex = fx.exact_prod(G[ir - 1].T, None, None, y)  # t(X) y over the codes, missing -> 0
            cc = np.zeros(m) if cs[0] is None else cs[0]
            ss = np.ones(m) if cs[1] is None else cs[1]
            nona = [Fraction(0)] * m
            for j in range(m):
                nona[j] = sum((Fraction(float(y[k])) for k in range(ir.size) if G[ir[k] - 1, j] != 3), Fraction(0))
            want = [(ex[j] - Fraction(float(cc[j])) * nona[j]) / Fraction(float(ss[j])) for j in range(m)]
            e = fx.pick_e(float(np.max(np.abs(y))), fx.hb_bits(fx.max_mult(ir - 1)), 60)
            quant = 2.0 ** (-e - 1) * ir.size * (3 + 3 + np.abs(cc)) / ss
            mag = np.array([float(abs(w)) for w in want]) + (np.abs(y).sum() * (2 + np.abs(cc))) / ss
            err = np.array([abs(Fraction(float(a)) - w) for a, w in zip(got, want)], dtype=float)
            assert np.all(err <= quant + 8 * 2.0 ** -52 * mag), err


def test_model_agrees_with_the_oracle_on_the_golden_files(oracle, obed, obed_na, rng):
    for o in (obed_na, obed):
        G = oracle.decode_dense(o)
        n, m = G.shape
        ir = rng.integers(1, n + 1, min(n, 150))
        ic = rng.integers(1, m + 1, 400)
        sc = oracle.bed_scaleBinom(o, ir, ic)
        c, s = sc["center"], sc["scale"]
        y_col, y_row = rng.normal(size=ic.size), rng.normal(size=ir.size)
        lists = bool(np.any(G == 3))
        for cs in ((None, None), (c, s)):
            a = fx.prod_T(G, ir, ic, y_col, *cs, lists=lists)
            want = oracle.bed_prodVec(o, y_col, ir, ic, *cs)
            sc_ = 1.0 if cs[1] is None else cs[1]
            tol = 1e-14 * (np.abs(y_col / sc_).sum() * 5)
            assert np.max(np.abs(a - want)) < tol
            b = fx.cprod(G, ir, ic, y_row, *cs, lists=lists)
            want = oracle.bed_cprodVec(o, y_row, ir, ic, *cs)
            tol = 1e-14 * np.abs(y_row).sum() * 5 / np.min(sc_)
            assert np.max(np.abs(b - want)) < tol


def test_row_sums_sq_model_agrees_with_the_oracle(oracle, obed, obed_na, rng):
    """rowSumsSq from the raw, high-bit and missing-value plane sums: (x - c)^2 / s^2 summed over present entries."""
    for o in (obed_na, obed):
        G = oracle.decode_dense(o)
        n, m = G.shape
        sc = oracle.bed_scaleBinom(o)
        for ir, ic in ((None, None), (rng.integers(1, n + 1, 60), rng.integers(1, m + 1, 333))):
            sel = np.arange(m) if ic is None else ic - 1
            c, s = sc["center"][sel], sc["scale"][sel]
            irr = np.arange(1, n + 1) if ir is None else ir
            icc = np.arange(1, m + 1) if ic is None else ic
            _, want = oracle.prod_and_rowSumsSq(o, irr, icc, c, s, np.zeros((sel.size, 1)))
            for pmv in (False, True):
                got = fx.row_sums_sq(G, ir, ic, c, s, pmv=pmv)
                assert np.max(np.abs(got - want)) < 1e-13 * np.max(want)


def test_sum_cz_follows_the_block_order(rng):
    """C = sum c z in k_prep1's order: equal to a plain sum up to rounding, and exactly its own order."""
    for n in (1, 300, 32768 + 5):
        c, z = rng.normal(size=n), rng.normal(size=n)
        C = fx.sum_cz(c, z)
        exact = sum((Fraction(float(a)) * Fraction(float(b)) for a, b in zip(c, z)), Fraction(0))
        assert abs(Fraction(C) - exact) <= 2.0 ** -50 * float(np.abs(c * z).sum())
    c, z = np.array([1.0, 3.0]), np.array([0.1, 1.0 / 3.0])
    assert fx.sum_cz(c, z) == math.fsum([fx.fma(1.0, 0.1, 0.0), fx.fma(3.0, 1.0 / 3.0, 0.0)])


def test_duplicate_columns_need_head_room_in_the_list_scatter(oracle, obed_na):
    """A missing-value column selected 16 times with y = 1: without head-room the physical-SNP sum of the quantised
    vector is 16 x 2^59 = 2^63 and wraps; with hb_bits(16) = 4 it stays below 2^60 and the product is right."""
    G = oracle.decode_dense(obed_na)
    j = int(np.nonzero((G == 3).any(axis=0))[0][0])
    ic = np.full(16, j + 1)
    y = np.ones(16)
    e_legacy = fx.pick_e(1.0, 0, 60)
    assert fx.scatter(fx.quantise(y, e_legacy), ic - 1, G.shape[1])[j] == -(2 ** 63)  # wrapped
    e_fixed = fx.pick_e(1.0, fx.hb_bits(16), 60)
    assert fx.scatter(fx.quantise(y, e_fixed), ic - 1, G.shape[1])[j] == 2 ** 59
    want = oracle.bed_prodVec(obed_na, y, None, ic)
    good = fx.prod_T(G, None, ic, y, lists=True)
    bad = fx.prod_T(G, None, ic, y, lists=True, legacy_hb=True)
    hit = G[:, j] == 3
    assert np.array_equal(good, want)  # integer-valued: exact
    assert np.array_equal(bad[~hit], want[~hit]) and np.all(np.abs(bad[hit] - want[hit]) > 1)
    # the flag plane has per-line digits and no scatter: no head-room needed
    assert np.array_equal(fx.prod_T(G, None, ic, y, lists=False), want)


def test_head_room_covers_rounding_up_to_the_binade():
    """From 2^8 duplicates on, rint(v 2^e) of an entry just below the binade reaches 2^(60 - hb) itself: 256 copies of
    nextafter(1, 0) with hb = 8 would sum to exactly 2^60, and 8 such sums in one k_corr row to 2^63.  hb_bits gives one
    bit more there; below 2^8 the double v 2^e is already an integer and cannot round up."""
    y = np.full(256, np.nextafter(1.0, 0.0))
    assert fx.scatter(fx.quantise(y, fx.pick_e(y[0], 8, 60)), np.zeros(256, int), 1)[0] == 2 ** 60
    for mult in (2, 3, 100, 128, 129, 256, 257, 5000):
        yy = np.full(mult, np.nextafter(1.0, 0.0))
        tot = int(fx.scatter(fx.quantise(yy, fx.pick_e(yy[0], fx.hb_bits(mult), 60)), np.zeros(mult, int), 1)[0])
        assert 0 < tot < 2 ** 60 and 8 * tot < 2 ** 63


# ---- dosage FBM.code256 (bsg_dosage.cu) -------------------------------------------------------------------------------
CODE_DOSAGE = np.concatenate([[0, 1, 2, np.nan, 0, 1, 2], np.arange(201) * 0.01, np.full(48, np.nan)])


def dosage_tables():
    """Tables of every scale the dosage kernels serve: CODE_DOSAGE (D = 100), bytes as values (D = 1, up to 255), k / 255
    (D = 255, byte 255 -> q = 255), and D = 4 / D = 2 tables holding NA entries."""
    d4 = np.arange(256) / 4.0
    d4[[3, 77, 200]] = np.nan
    d2 = np.arange(256) / 2.0
    d2[[5, 254]] = np.nan
    return {"dosage": (CODE_DOSAGE, 100), "d1": (np.arange(256.0), 1), "d255": (np.arange(256) / 255.0, 255),
            "d4": (d4, 4), "d2": (d2, 2)}


def worst_case_vector(k, e=60):
    """k copies of y = Q 2^-e with Q = -(9 2^56 + sum_{s<7} 128 256^s): digits -128 in slices 0..6 and -9 in slice 7."""
    Q = -(9 * 2 ** 56 + sum(128 * 256 ** s for s in range(7)))
    return np.full(k, math.ldexp(float(Q), -e)), Q


def test_dosage_table_rule():
    for name, (code, D) in dosage_tables().items():
        got, q, na = fx.dosage_table(code)
        assert got == D, name
        ok = ~np.isnan(code)
        assert np.array_equal(na, ~ok) and np.all(q[~ok] == 0)
        assert np.array_equal(q[ok].astype(float), np.rint(D * code[ok])) and np.max(q) <= 255
    D, q, na = fx.dosage_table(CODE_DOSAGE)
    assert list(q[:7]) == [0, 100, 200, 0, 0, 100, 200] and q[7 + 137] == 137 and q[207] == 200 and na[3] and na[230]
    assert fx.dosage_table(np.linspace(0, 2, 256))[0] == 0                     # no D makes every value an integer
    assert fx.dosage_table(np.r_[np.inf, np.arange(255.0)])[0] == 0           # an infinite entry
    assert fx.dosage_table(np.r_[256.0, np.arange(255.0)])[0] == 0            # q would exceed 255
    assert fx.dosage_table(np.arange(256) / 255.0)[1][255] == 255


def _dosage_bound(Dq, ir, ic, y, center, scale, D, hb=0, cprod=False):
    """Quantisation + combine + 1 / D + C bound of one dosage product (as the 2-bit model's bound): each vector entry is
    off by at most 2^(-e-1) after rint, and meets q / D in every value of its line."""
    n, m = Dq.shape
    r0 = np.arange(n) if ir is None else ir - 1
    c0 = np.arange(m) if ic is None else ic - 1
    c = np.zeros(c0.size) if center is None else np.asarray(center)
    s = np.ones(c0.size) if scale is None else np.asarray(scale)
    val = Dq[np.ix_(r0, c0)] / D
    if not cprod:
        v = np.asarray(y) / s
        e = fx.pick_e(float(np.max(np.abs(v))), 0, 60)
        quant = val.sum(1) * 2.0 ** (-e - 1)
        mag = ((val + np.abs(c)) * np.abs(v)).sum(1) + np.abs(c * v).sum()
    else:
        e = fx.pick_e(float(np.max(np.abs(y))), hb, 60)
        quant = ((val + np.abs(c)) / s).sum(0) * 2.0 ** (-e - 1)
        mag = ((val + np.abs(c)) / s * np.abs(np.asarray(y))[:, None]).sum(0)
    return quant + 8 * 2.0 ** -52 * mag + 1e-300


@pytest.mark.parametrize("table", ["dosage", "d1", "d255", "d4", "d2"])
@pytest.mark.parametrize("scaled", [False, True])
def test_dosage_model_within_its_bound_of_the_exact_product(rng, table, scaled):
    code, D = dosage_tables()[table]
    n, m = 29, 43
    raw = rng.integers(0, 256, size=(n, m)).astype(np.uint8)
    _, qmap, isna = fx.dosage_table(code)
    ic = np.r_[np.repeat(rng.choice(m, 2, replace=False) + 1, 5), rng.integers(1, m + 1, 20)]   # a multiset
    ir = np.r_[np.repeat(rng.choice(n, 2, replace=False) + 1, 17), rng.integers(1, n + 1, 12)]
    c, s = (rng.uniform(0, 2, size=ic.size), rng.uniform(0.3, 2.0, size=ic.size)) if scaled else (None, None)
    y = rng.normal(size=ic.size)
    got = fx.dosage_prod(raw, code, None, ic, y, c, s)
    exact = fx.exact_dosage_prod(raw, code, None, ic, y, c, s)
    hit = np.array([w is None for w in exact])
    assert np.array_equal(np.isnan(got), hit) and (not isna.any() or hit.any())
    bound = _dosage_bound(qmap[raw].astype(float), None, ic, y, c, s, D)
    for a, w, b in zip(got, exact, bound):
        assert w is None or abs(Fraction(float(a)) - w) <= b
    # Xt.y: the exact product over the transposed selection, NaN on the lines an NA byte meets
    yr = rng.normal(size=ir.size)
    cc = None if c is None else rng.uniform(0, 2, size=ic.size)
    got = fx.dosage_cprod(raw, code, ir, ic, yr, cc, s)
    cz = np.zeros(ic.size) if cc is None else cc
    sz = np.ones(ic.size) if s is None else s
    bound = _dosage_bound(qmap[raw].astype(float), ir, ic, yr, cc, s, D, fx.hb_bits(fx.max_mult(ir - 1)), cprod=True)
    for t, j in enumerate(ic - 1):
        b = raw[ir - 1, j]
        if isna[b].any():
            assert np.isnan(got[t])
            continue
        w = sum(((Fraction(int(qmap[bb]), D) - Fraction(float(cz[t]))) / Fraction(float(sz[t])) * Fraction(float(yy))
                 for bb, yy in zip(b, yr)), Fraction(0))
        assert abs(Fraction(float(got[t])) - w) <= bound[t]


def test_worst_case_vector_reaches_the_int32_cap():
    """The vector that drives every digit slice to -128: |Q| in [2^59, 2^60), set bits 7..59 (an exact double), so
    pick_e returns e; 65,536 lines of q = 255 put -2,139,095,040 in each accumulator, 65,794 lines would pass -2^31."""
    y, Q = worst_case_vector(4)
    assert 2 ** 59 <= -Q < 2 ** 60 and int(math.ldexp(y[0], 60)) == Q
    assert fx.pick_e(float(np.max(np.abs(y))), 0, 60) == 60
    q = fx.quantise(y, 60)
    assert np.all(q == Q)
    d = fx.digits(q, 8)
    assert np.all(d[:, :7] == -128) and np.all(d[:, 7] == -9)
    one = fx.partials(np.full((1, 1), 255), d[:1])[0]
    assert np.all(one[:7] * 65536 == -2139095040) and -2139095040 >= -(2 ** 31)
    assert one[0] * 65793 >= -(2 ** 31) > one[0] * 65794


def test_literal_models_within_rounding_of_the_exact_sums(rng):
    """lit_prod / lit_cprod / proj_literal against rationals (finite input) and fp64 NumPy (NaN / Inf pattern)."""
    n, m = 45, 37
    raw = rng.integers(0, 208, size=(n, m)).astype(np.uint8)
    raw[rng.random((n, m)) < 0.01] = 230
    raw[0, :] = 3
    ir, ic = rng.integers(1, n + 1, 40), rng.integers(1, m + 1, 35)
    c, s = rng.uniform(0, 2, size=35), rng.uniform(0.3, 2.0, size=35)
    x, yr = rng.normal(size=35), rng.normal(size=40)
    X = (CODE_DOSAGE[raw[np.ix_(ir - 1, ic - 1)]] - c) / s
    ok = ~np.isnan(X)
    for got, want, mag in ((fx.lit_prod(raw, CODE_DOSAGE, ir, ic, x, c, s), X @ x, np.abs(X) @ np.abs(x)),
                           (fx.lit_cprod(raw, CODE_DOSAGE, ir, ic, yr, c, s), yr @ X, np.abs(yr) @ np.abs(X))):
        assert np.array_equal(np.isnan(got), np.isnan(want)) and np.isnan(want).any()
        fin = ~np.isnan(want)
        assert np.all(np.abs(got[fin] - want[fin]) <= 64 * 2.0 ** -52 * mag[fin])
    V = rng.normal(size=(35, 2))
    XV, rss, na = fx.proj_literal(raw, CODE_DOSAGE, ir, ic, c, s, V)
    assert np.array_equal(na, ~ok.all(axis=1)) and np.array_equal(np.isnan(rss), na)
    Xz = np.where(ok, X, 0.0)
    assert np.all(np.abs(rss[~na] - (Xz * Xz).sum(1)[~na]) <= 64 * 2.0 ** -52 * (Xz * Xz).sum(1)[~na])
    assert np.allclose(XV[~na], (Xz @ V)[~na], rtol=0, atol=1e-12)
    # exact in rationals for one row: the serial fma loop rounds once per column
    i = int(np.nonzero(~na)[0][0])
    acc = 0.0
    for j in range(35):
        acc = float(Fraction(float(X[i, j])) * Fraction(float(X[i, j])) + Fraction(acc))
    assert rss[i] == acc
    # non-finite input: Inf / NaN propagate as in fp64
    s0 = s.copy()
    s0[3] = 0.0
    with np.errstate(all="ignore"):
        want = (((CODE_DOSAGE[raw[np.ix_(ir - 1, ic - 1)]] - c) / s0) * x).sum(1)  # one infinite column
    got = fx.lit_prod(raw, CODE_DOSAGE, ir, ic, x, c, s0)
    assert np.array_equal(np.isinf(got), np.isinf(want)) and np.array_equal(np.isnan(got), np.isnan(want))
    assert np.isinf(got).any() and np.all(got[np.isfinite(want)] == want[np.isfinite(want)])
    # hard calls: code 3 is NA
    G = rng.integers(0, 4, size=(n, m)).astype(np.uint8)
    XV, rss, na = fx.proj_literal(G, None, ir, ic, c, s, V)
    assert np.array_equal(na, (G[np.ix_(ir - 1, ic - 1)] == 3).any(axis=1)) and np.array_equal(np.isnan(XV[:, 0]), na)
