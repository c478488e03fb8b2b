"""The dosage X.y / Xt.y kernels (k_dmvT, k_dmv), their literal fallbacks (k_lit_prod, k_lit_cprod) and
prod_and_rowSumsSq2 (k_proj_literal) against the exact host model (tests/fixedpoint_ref.py), byte for byte.

The byte-operand kernels quantise the vector once, sum digit slices as exact integers and finish with a fixed fp64
sequence, like the 2-bit kernels, so any lost or doubled slice, a split that wraps its int32 accumulator, a missing
head-room bit or a change of rounding changes the bytes here.  Tables of every scale (D = 1, 2, 4, 100, 255, bytes up to
255), shapes around the value-copy stride (128), k_dmv's 64-sample chunks and k_dmvT's 512-byte segments and 32-line
steps, forced k-splits, the int32 cap of one split, multisets, special vectors, the NA rule and empty selections.

NaN payloads are not part of the comparison (an NA result is any NaN); every other output is compared by its bytes.
"""
import numpy as np
import pytest

from tests import fixedpoint_ref as fx
from tests.test_fixedpoint_model import dosage_tables, worst_case_vector
from tests.test_gpu_fixedpoint import _same, _special_vectors

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def B():
    import bigsnpr_b200 as b

    from bigsnpr_b200 import build

    build.build()
    return b


def _same_na(got, want, what=""):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, what
    assert np.array_equal(np.isnan(got), np.isnan(want)), "%s: NaN pattern differs" % what
    _same(np.where(np.isnan(got), np.nan, got), np.where(np.isnan(want), np.nan, want), what)


def _handle(B, raw, table):
    code, D = dosage_tables()[table]
    g = B.Bed.from_fbm(raw, code256=code)
    assert g.dosage_scale == D and fx.dosage_table(code)[0] == D
    return g, code


def _raw(rng, n, m, table, na_rate=0.0):
    """Bytes 0..255 for the D = 1 / 255 tables (every byte finite), the finite bytes of the others, plus NA bytes."""
    code, _ = dosage_tables()[table]
    fin = np.nonzero(~np.isnan(code))[0]
    raw = fin[rng.integers(0, fin.size, size=(n, m))].astype(np.uint8)
    raw[rng.random((n, m)) < 0.05] = fin[-1]  # the largest byte value of the table
    nas = np.nonzero(np.isnan(code))[0]
    if na_rate and nas.size:
        hit = rng.random((n, m)) < na_rate
        raw[hit] = nas[rng.integers(0, nas.size, size=int(hit.sum()))]
    return raw


def _xy(B, g, y, ir, ic, c=None, s=None):
    return B.bed_prodVec(g, y, ... if ir is None else ir, ... if ic is None else ic, c, s)


def _xty(B, g, y, ir, ic, c=None, s=None):
    return B.bed_cprodVec(g, y, ... if ir is None else ir, ... if ic is None else ic, c, s)


def _check(B, g, raw, code, rng, ir, ic, what, y=None, yr=None):
    """X.y and Xt.y on (ir, ic), unscaled and scaled, against the model."""
    n, m = raw.shape
    nr, nc = (n if ir is None else ir.size), (m if ic is None else ic.size)
    c, s = rng.uniform(0.05, 1.95, size=nc), rng.uniform(0.3, 2.0, size=nc)
    for cs in ((None, None), (c, s)):
        yy = rng.normal(size=nc) if y is None else y
        _same_na(_xy(B, g, yy, ir, ic, *cs), fx.dosage_prod(raw, code, ir, ic, yy, *cs),
                 "X.y %s scaled=%s" % (what, cs[0] is not None))
        yyr = rng.normal(size=nr) if yr is None else yr
        cc = None if cs[0] is None else rng.uniform(0.05, 1.95, size=nc)
        _same_na(_xty(B, g, yyr, ir, ic, cc, cs[1]), fx.dosage_cprod(raw, code, ir, ic, yyr, cc, cs[1]),
                 "Xt.y %s scaled=%s" % (what, cs[0] is not None))


# ---- shapes at the layout boundaries ------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 127, 128, 129, 511, 512, 513, 1025])
def test_shapes_match_the_model(B, rng, n):
    """Value-copy stride round_up(n, 128), k_dmv's 64-sample chunks, k_dmvT's 512-byte segments (n around 512 / 1024) and
    32-line steps (1 / 31 / 32 / 33 / 65 lines): identity columns (TMA stage), permutations and multisets (bulk-copy
    stage, whose 512-byte loads run past a line into the next one or the slack), row subsets; every table."""
    names = list(dosage_tables())
    for k, nc in enumerate((1, 31, 32, 33, 65)):
        table = names[(k + n) % len(names)]
        raw = _raw(rng, n, nc, table, na_rate=0.002)
        g, code = _handle(B, raw, table)
        ir = rng.integers(1, n + 1, size=max(1, n // 2))
        cases = [(None, None), (None, rng.permutation(nc) + 1), (ir, rng.permutation(nc) + 1),
                 (None, rng.integers(1, nc + 1, size=nc)), (rng.permutation(n) + 1, np.array([nc]))]
        for ir_, ic_ in cases:
            _check(B, g, raw, code, rng, ir_, ic_, "%s n=%d nc=%d" % (table, n, nc))
        g.close()


@pytest.mark.parametrize("ks", ["1", "2", "3", "7"])
def test_forced_ksplits_give_the_models_bytes(B, rng, monkeypatch, ks):
    """BSG_DMV_KS (read on every call): 1, 2, 3 and 7 splits of the lines (X.y) and of the 64-sample chunks (Xt.y) each
    give the model's bytes."""
    monkeypatch.setenv("BSG_DMV_KS", ks)
    for table, (n, m) in (("d255", (1153, 300)), ("dosage", (2049, 97)), ("d4", (700, 161))):
        raw = _raw(rng, n, m, table, na_rate=0.001)
        g, code = _handle(B, raw, table)
        _check(B, g, raw, code, rng, None, None, "%s ks=%s" % (table, ks))
        _check(B, g, raw, code, rng, rng.integers(1, n + 1, n // 3), rng.integers(1, m + 1, m + 9), "%s ks=%s" % (table, ks))
        g.close()


# ---- int32 cap of one k-split ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lines", [65536, 65537, 65794])
def test_xy_int32_cap_of_one_split(B, monkeypatch, lines):
    """X.y over `lines` selected lines, all byte 255 (q = 255), with the vector whose digits are -128 in slices 0..6.
    BSG_DMV_KS=1: at 65,536 lines one split holds every line and each accumulator reaches -2,139,095,040; 65,537 lines
    need a second split; 65,794 lines in one split would pass -2^31."""
    monkeypatch.setenv("BSG_DMV_KS", "1")
    n = 129
    raw = np.full((n, 2), 255, dtype=np.uint8)
    g, code = _handle(B, raw, "d1")
    y, _ = worst_case_vector(lines)
    ic = np.ones(lines, dtype=np.int32)  # one column selected `lines` times: the lines of one split
    for cs in ((None, None), (np.full(lines, 0.7), np.ones(lines))):
        want = fx.dosage_prod(raw, code, None, ic, y, *cs)
        assert np.all(np.isfinite(want))
        _same(_xy(B, g, y, None, ic, *cs), want, "X.y %d lines scaled=%s" % (lines, cs[0] is not None))
    g.close()


@pytest.mark.parametrize("n", [65536, 65537, 131073])
def test_xty_int32_cap_of_one_split(B, monkeypatch, n):
    """Xt.y over n samples of byte 255 with the worst-case vector, BSG_DMV_KS=1: one, two and three splits of 1,024
    chunks of 64 samples."""
    monkeypatch.setenv("BSG_DMV_KS", "1")
    raw = np.full((n, 3), 255, dtype=np.uint8)
    raw[::7, 1] = 0
    g, code = _handle(B, raw, "d255")
    y, _ = worst_case_vector(n)
    c, s = np.array([0.5, 1.5, 0.25]), np.array([1.0, 0.75, 2.0])
    for cs in ((None, None), (c, s)):
        _same(_xty(B, g, y, None, None, *cs), fx.dosage_cprod(raw, code, None, None, y, *cs), "Xt.y n=%d" % n)
    g.close()


# ---- multisets -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mult", [1, 2, 3, 16, 17, 255, 256, 257])
def test_multisets_match_the_model(B, rng, mult):
    """Row multiplicities for Xt.y (scattered into Q with hb_bits(multiplicity) of head-room: 0 .. 9 bits) and column
    multiplicities for X.y (each duplicate its own line), the repeated entries at the vector's largest magnitude."""
    n, m = 600, 120
    for table in ("d255", "dosage"):
        raw = _raw(rng, n, m, table, na_rate=0.0005)
        g, code = _handle(B, raw, table)
        rows = np.repeat(rng.choice(n, 3, replace=False) + 1, mult)
        ir = np.r_[rows, rng.integers(1, n + 1, 50)]
        perm = rng.permutation(ir.size)
        ir = ir[perm]
        yr = np.r_[np.full(rows.size, np.nextafter(1.0, 0.0)), rng.uniform(-1, 1, 50)][perm]
        cols = np.repeat(rng.choice(m, 3, replace=False) + 1, mult)
        ic = np.r_[cols, rng.integers(1, m + 1, 40)]
        y = np.r_[np.full(cols.size, -1.0), rng.uniform(-1, 1, 40)]
        _check(B, g, raw, code, rng, ir, ic, "%s mult=%d" % (table, mult), y=y, yr=yr)
        _check(B, g, raw, code, rng, None, ic, "%s mult=%d" % (table, mult), y=y)
        _check(B, g, raw, code, rng, ir, None, "%s mult=%d" % (table, mult), yr=yr)
        g.close()


# ---- vectors -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("table", ["dosage", "d1", "d255"])
def test_special_vectors_match_the_model(B, rng, table):
    n, m = 1025, 97
    raw = _raw(rng, n, m, table, na_rate=0.001)
    g, code = _handle(B, raw, table)
    c, s = rng.uniform(0.1, 1.9, size=m), rng.uniform(0.3, 2, size=m)
    with np.errstate(over="ignore", under="ignore"):
        for name, y in _special_vectors(rng, m).items():
            scalings = [(None, None)]
            if name not in ("subnormal", "huge_tiny"):  # scaled: z = y / s leaves the tested range
                scalings += [(np.zeros(m), s), (c, s)]
            for cs in scalings:
                _same_na(_xy(B, g, y, None, None, *cs), fx.dosage_prod(raw, code, None, None, y, *cs),
                         "X.y %s scaled=%s" % (name, cs[0] is not None))
            yr = _special_vectors(rng, n)[name]
            for cs in scalings:
                _same_na(_xty(B, g, yr, None, None, *cs), fx.dosage_cprod(raw, code, None, None, yr, *cs),
                         "Xt.y %s scaled=%s" % (name, cs[0] is not None))
    g.close()


# ---- NA rule -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("table", ["dosage", "d4", "d2"])
def test_na_codes_outside_the_selection_poison_nothing(B, rng, table):
    """NA bytes only in unselected rows and unselected columns: every output is finite and the model's bytes."""
    n, m = 513, 70
    code, _ = dosage_tables()[table]
    nas = np.nonzero(np.isnan(code))[0]
    raw = _raw(rng, n, m, table)
    bad_rows, bad_cols = rng.choice(n, 20, replace=False), rng.choice(m, 6, replace=False)
    raw[np.ix_(bad_rows, rng.choice(m, 30, replace=False))] = nas[0]
    raw[np.ix_(rng.choice(n, 100, replace=False), bad_cols)] = nas[-1]
    g, _ = _handle(B, raw, table)
    ir = np.setdiff1d(np.arange(n), bad_rows)[rng.permutation(n - 20)] + 1
    ic = rng.permutation(np.setdiff1d(np.arange(m), bad_cols)) + 1
    y, yr = rng.normal(size=ic.size), rng.normal(size=ir.size)
    c, s = rng.uniform(0.1, 1.9, size=ic.size), rng.uniform(0.3, 2, size=ic.size)
    for cs in ((None, None), (c, s)):
        a, b = _xy(B, g, y, ir, ic, *cs), _xty(B, g, yr, ir, ic, *cs)
        assert np.all(np.isfinite(a)) and np.all(np.isfinite(b))
        _same(a, fx.dosage_prod(raw, code, ir, ic, y, *cs), "X.y")
        _same(b, fx.dosage_cprod(raw, code, ir, ic, yr, *cs), "Xt.y")
    g.close()


@pytest.mark.parametrize("table", ["dosage", "d4", "d2"])
def test_na_codes_in_the_selection_give_nan_even_against_zero_weights(B, rng, table):
    """An NA byte in a selected row and column makes its output row (X.y) or line (Xt.y) NaN even where the vector's
    entry is 0; CODE_DOSAGE's byte 230 maps to NA like byte 3."""
    n, m = 300, 50
    code, _ = dosage_tables()[table]
    nas = np.nonzero(np.isnan(code))[0]
    raw = _raw(rng, n, m, table)
    raw[10, 4], raw[20, 7], raw[30, 7] = nas[0], nas[-1], nas[nas.size // 2]
    if table == "dosage":
        raw[40, 9] = 230
    g, _ = _handle(B, raw, table)
    ic = np.r_[5, 8, 10, rng.integers(1, m + 1, 30)]
    ir = np.r_[11, 21, 31, 41, rng.integers(1, n + 1, 60)]
    y = rng.normal(size=ic.size)
    y[:3] = 0.0
    yr = rng.normal(size=ir.size)
    yr[:4] = 0.0
    for cs in ((None, None), (rng.uniform(0.1, 1.9, size=ic.size), rng.uniform(0.3, 2, size=ic.size))):
        a, b = _xy(B, g, y, ir, ic, *cs), _xty(B, g, yr, ir, ic, *cs)
        assert np.all(np.isnan(a[:3 + (table == "dosage")])) and np.all(np.isnan(b[:2 + (table == "dosage")]))
        _same_na(a, fx.dosage_prod(raw, code, ir, ic, y, *cs), "X.y")
        _same_na(b, fx.dosage_cprod(raw, code, ir, ic, yr, *cs), "Xt.y")
        _same_na(_xy(B, g, y, None, ic, *cs), fx.dosage_prod(raw, code, None, ic, y, *cs), "X.y all rows")
    g.close()


def test_empty_selections_give_the_models_zeros(B, rng):
    n, m = 200, 40
    raw = _raw(rng, n, m, "dosage", na_rate=0.01)
    g, code = _handle(B, raw, "dosage")
    e = np.array([], dtype=np.int32)
    ir, ic = rng.integers(1, n + 1, 30), rng.integers(1, m + 1, 12)
    c, s = rng.uniform(0.1, 1.9, size=12), rng.uniform(0.3, 2, size=12)
    for cs in ((None, None), (c, s)):
        _same_na(_xty(B, g, np.zeros(0), e, ic, *cs), fx.dosage_cprod(raw, code, e, ic, np.zeros(0), *cs), "Xt.y nr=0")
        assert _xy(B, g, rng.normal(size=12), e, ic, *cs).size == 0
    got = _xy(B, g, np.zeros(0), ir, e)
    _same(got, fx.dosage_prod(raw, code, ir, e, np.zeros(0)), "X.y nc=0")
    assert not np.any(got) and _xty(B, g, rng.normal(size=30), ir, e).size == 0
    g.close()


# ---- device-pointer forms and the literal fallbacks --------------------------------------------------------------------------
def test_device_pointer_forms_match_the_host_forms_and_the_model(B, rng):
    import torch

    n, m = 1025, 300
    raw = _raw(rng, n, m, "d4", na_rate=0.001)
    g, code = _handle(B, raw, "d4")
    ir, ic = rng.integers(1, n + 1, 700), rng.integers(1, m + 1, 333)
    c, s = rng.uniform(0.1, 1.9, size=ic.size), rng.uniform(0.3, 2, size=ic.size)
    v = B.View(g, ir, ic, center=c, scale=s)
    try:
        dev = torch.device("cuda", 0)
        y, yr = rng.normal(size=ic.size), rng.normal(size=ir.size)
        o_d = torch.empty(ir.size, dtype=torch.float64, device=dev)
        v.prodvec_dev(torch.tensor(y, device=dev).data_ptr(), o_d.data_ptr())
        or_d = torch.empty(ic.size, dtype=torch.float64, device=dev)
        xr_d = torch.tensor(yr, device=dev)
        v.cprodvec_dev(xr_d.data_ptr(), or_d.data_ptr())
        torch.cuda.synchronize()
        want, wantr = fx.dosage_prod(raw, code, ir, ic, y, c, s), fx.dosage_cprod(raw, code, ir, ic, yr, c, s)
        _same_na(o_d.cpu().numpy(), want, "prodvec_dev")
        _same_na(or_d.cpu().numpy(), wantr, "cprodvec_dev")
        _same_na(v.prodvec(y), want, "view prodvec")
        _same_na(v.cprodvec(yr), wantr, "view cprodvec")
        _same_na(_xy(B, g, y, ir, ic, c, s), want, "bed_prodVec")
    finally:
        v.close()
        g.close()


def test_non_finite_host_forms_give_the_literal_loops_bytes(B, rng):
    """Inf / NaN in x, a zero scale, an infinite center: the host forms re-run k_lit_prod / k_lit_cprod."""
    n, m = 150, 70
    raw = _raw(rng, n, m, "dosage", na_rate=0.005)
    g, code = _handle(B, raw, "dosage")
    ir, ic = rng.integers(1, n + 1, 120), rng.integers(1, m + 1, 60)
    c, s = rng.uniform(0.1, 1.9, size=60), rng.uniform(0.3, 2, size=60)
    s0 = s.copy()
    s0[7] = 0.0
    cinf = c.copy()
    cinf[3] = np.inf
    y, yr = rng.normal(size=60), rng.normal(size=120)
    yi, yn = y.copy(), yr.copy()
    yi[5], yn[9] = np.inf, np.nan
    with np.errstate(all="ignore"):
        for what, x, cs in (("Inf in x", yi, (None, None)), ("Inf in x, scaled", yi, (c, s)), ("zero scale", y, (c, s0)),
                            ("Inf center", y, (cinf, s))):
            _same_na(_xy(B, g, x, ir, ic, *cs), fx.lit_prod(raw, code, ir, ic, x, *cs), "X.y %s" % what)
        for what, x, cs in (("NaN in y", yn, (None, None)), ("NaN in y, scaled", yn, (c, s)), ("zero scale", yr, (c, s0)),
                            ("Inf center", yr, (cinf, s))):
            _same_na(_xty(B, g, x, ir, ic, *cs), fx.lit_cprod(raw, code, ir, ic, x, *cs), "Xt.y %s" % what)
    g.close()


# ---- prod_and_rowSumsSq2 ---------------------------------------------------------------------------------------------------
CODE_012 = np.r_[[0.0, 1.0, 2.0], np.full(253, np.nan)]


def _xv_model(g, kind, P, code, ir, ic, c, s, v):
    """One column of XV: the dosage model, or the 2-bit model of the path the hard-call handle takes, then NaN rows."""
    if not kind.startswith("hard"):
        return fx.dosage_prod(P, code, ir, ic, v, c, s)
    G = P
    if (g.layouts & 2) and not np.any(G == 3):
        out = fx.prod_pmv(G, ir, ic, v, c, s)
    else:
        out = fx.prod_T(G, ir, ic, v, c, s, lists=False)
    out[(G[np.ix_(ir - 1, ic - 1)] == 3).any(axis=1)] = np.nan
    return out


@pytest.mark.parametrize("K", [1, 2, 3])
def test_prod_and_rowSumsSq2_matches_the_model(B, rng, K):
    """XV column by column equals the single-vector X.y model with NaN rows; rowSumsSq equals k_proj_literal's serial fma
    loop; with a zero scale XV is that loop's too."""
    n, m = 257, 131
    for kind in ("dosage", "d4", "hard", "hard_na"):
        if kind.startswith("hard"):
            G = rng.integers(0, 3, size=(n, m)).astype(np.uint8)
            if kind == "hard_na":
                G[rng.random((n, m)) < 0.1] = 3
            P, code, g = G, None, B.Bed.from_fbm(G, code256=CODE_012)
            assert g.dosage_scale == 0
        else:
            P = _raw(rng, n, m, kind, na_rate=0.002)
            g, code = _handle(B, P, kind)
        ir = rng.integers(1, n + 1, 200)
        ic = rng.permutation(m)[:100] + 1
        c, s = rng.uniform(0.2, 1.8, size=ic.size), rng.uniform(0.3, 1.2, size=ic.size)
        V = rng.normal(size=(ic.size, K))
        XV, rss = B.prod_and_rowSumsSq2(g, ir, ic, c, s, V)
        for k in range(K):
            _same_na(XV[:, k], _xv_model(g, kind, P, code, ir, ic, c, s, V[:, k]), "%s XV[, %d]" % (kind, k))
        _, rss0, _ = fx.proj_literal(P, code, ir, ic, c, s)
        _same_na(rss, rss0, "%s rowSumsSq" % kind)
        s0 = s.copy()
        s0[11] = 0.0
        XV, rss = B.prod_and_rowSumsSq2(g, ir, ic, c, s0, V)
        XV0, rss0, _ = fx.proj_literal(P, code, ir, ic, c, s0, V)
        _same_na(XV, XV0, "%s XV, zero scale" % kind)
        _same_na(rss, rss0, "%s rowSumsSq, zero scale" % kind)
        g.close()
