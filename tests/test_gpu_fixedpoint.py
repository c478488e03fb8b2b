"""Every X.y / Xt.y kernel path against the exact host model of its arithmetic (tests/fixedpoint_ref.py), byte for byte.

The products are sums of exact integers (digit slices of a fixed-point vector) followed by one fixed fp64 sequence per
output, so a kernel, split, staging or missing-value mode that changes any integer partial changes the bytes here.
Paths: k_pmv (sample-major copy for X.y, SNP-major copy for Xt.y), k_pmvT (TMA staging, identity columns),
k_pmvT_lines (column lists), k_pmvT2<1> (flag plane), k_pmvT2<2> and k_pmv<3> (high-bit plane, through rowSumsSq), the
missing-value lists, two vectors per pass, the device-pointer entry points, and the process-wide switches (k-split,
waves, k_pmv variant, kernel choice, pair modes) in subprocesses.  multLinReg's t-scores are compared across the switch
settings, not with the model: the regression formula on top of its plane sums is not restated.

Where the lists deliver a missing-value sum without scaling, its split into 32-bit halves follows the row layout built
on the device; those cases use dyadic vectors (quantised entries with zero low halves), for which every layout gives the
same halves (see the model's docstring).
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import fixedpoint_ref as fx

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def B():
    import bigsnpr_b200 as b

    from bigsnpr_b200 import build

    build.build()
    return b


def _same(got, want, what=""):
    got, want = np.ascontiguousarray(got, dtype=np.float64), np.ascontiguousarray(want, dtype=np.float64)
    assert got.shape == want.shape, what
    if got.tobytes() != want.tobytes():
        bad = np.nonzero(got.view(np.int64) != want.view(np.int64))[0]
        k = bad[0]
        raise AssertionError("%s: %d of %d differ, first at %d: %r vs model %r (max |diff| %.3g)"
                             % (what, bad.size, got.size, k, got[k], want[k], np.max(np.abs(got - want))))


def _sel(ind):
    return ... if ind is None else ind  # the API's "every row / column"


def _xy(B, g, y, ir=None, ic=None, center=None, scale=None):
    return B.bed_prodVec(g, y, _sel(ir), _sel(ic), center, scale)


def _xty(B, g, y, ir=None, ic=None, center=None, scale=None):
    return B.bed_cprodVec(g, y, _sel(ir), _sel(ic), center, scale)


def _codes(rng, n, m, na_rate):
    G = rng.integers(0, 3, size=(n, m)).astype(np.uint8)
    if na_rate:
        G[rng.random((n, m)) < na_rate] = 3
        G[0, 0] = 3
    return G


def _handle(B, G, layouts=None):
    from oracle import ref

    n, m = G.shape
    return B.Bed.from_packed(ref.write_bed_bytes(G), n, m, layouts=B.LAYOUT_SNP_MAJOR if layouts is None else layouts)


def _vec(rng, k, dyadic):
    if dyadic:  # quantised entries are multiples of 2^32 (see the module docstring)
        return rng.integers(-(1 << 20), 1 << 20, size=k) / float(1 << 20)
    return rng.normal(size=k)


def _uses_lists(G, env_off=False):
    rate = float(np.mean(G == 3))
    return 0 < rate <= 0.04 and not env_off


def _check_handle(B, g, G, rng, cases, lists, pmv_x=False):
    """X.y and Xt.y of handle g on every (ir, ic) of `cases`, unscaled and scaled, against the model."""
    n, m = G.shape
    for ir, ic in cases:
        nr, nc = (n if ir is None else ir.size), (m if ic is None else ic.size)
        c = rng.uniform(0.05, 1.95, size=nc)
        s = rng.uniform(0.3, 2.0, size=nc)
        for cs in ((None, None), (c, s)):
            y = _vec(rng, nc, dyadic=lists and cs[0] is None)
            got = _xy(B, g, y, ir, ic, *cs)
            want = (fx.prod_pmv(G, ir, ic, y, *cs) if pmv_x else fx.prod_T(G, ir, ic, y, *cs, lists=lists))
            _same(got, want, "X.y n=%d nc=%d scaled=%s" % (n, nc, cs[0] is not None))
            yr = _vec(rng, nr, dyadic=lists)
            cc, ss = (None, None) if cs[0] is None else (rng.uniform(0.05, 1.95, size=nc), s)
            got = _xty(B, g, yr, ir, ic, cc, ss)
            _same(got, fx.cprod(G, ir, ic, yr, cc, ss, lists=lists), "Xt.y n=%d nc=%d" % (nr, nc))


# ---- shapes at the kernels' boundaries --------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1023, 1025, 2046, 2047, 2048, 2049])
@pytest.mark.parametrize("na", ["none", "lists", "plane", "lists_off"])
def test_snp_major_paths_match_the_model(B, rng, monkeypatch, n, na):
    """k_pmvT (identity columns: TMA), k_pmvT_lines (column lists), k_pmvT2<1> (flag plane), the missing-value lists
    and Xt.y on k_pmv, for 1 / 31 / 32 / 33 lines (32 per step) and sample counts around the 2048 / 1024 blocks."""
    rate = {"none": 0.0, "lists": 0.005, "plane": 0.1, "lists_off": 0.005}[na]
    G = _codes(rng, n, 33, rate)
    monkeypatch.setenv("BSG_NA_LISTS", "0" if na == "lists_off" else "1")
    g = _handle(B, G)
    lists = _uses_lists(G, env_off=na == "lists_off")
    ir = rng.choice(n, n // 3, replace=False) + 1
    cases = [(None, None), (None, np.arange(1, 32)), (ir, np.array([7])), (None, np.arange(1, 33)),
             (ir, rng.permutation(33)[:33] + 1)]
    _check_handle(B, g, G, rng, cases, lists)
    g.close()


@pytest.mark.parametrize("L", [511, 512, 513])
def test_sample_major_and_xty_chunks_match_the_model(B, rng, L):
    """k_pmv around its 512-code chunks (contraction length L) and its 352 / 480-line groups: X.y on the sample-major
    copy (no missing value) and Xt.y on the SNP-major copy (with and without missing values)."""
    for nlines in (352, 353, 480, 481):
        G = _codes(rng, nlines, L, 0.0)
        g = _handle(B, G, B.LAYOUT_SNP_MAJOR | B.LAYOUT_SAMPLE_MAJOR)
        _check_handle(B, g, G, rng, [(None, None), (None, rng.integers(1, L + 1, L // 2))], False, pmv_x=True)
        g.close()
    for na_rate in (0.0, 0.1):
        G = _codes(rng, L, 481, na_rate)
        g = _handle(B, G)
        _check_handle(B, g, G, rng, [(None, None), (rng.integers(1, L + 1, 300), rng.integers(1, 482, 353))], False)
        g.close()


def test_sample_and_snp_major_x_products_are_bit_identical(B, rng):
    """Without duplicate columns both X.y kernels quantise with the same exponent and produce the same integers."""
    G = _codes(rng, 2049, 700, 0.0)
    g3 = _handle(B, G, B.LAYOUT_SNP_MAJOR | B.LAYOUT_SAMPLE_MAJOR)
    g1 = _handle(B, G)
    for ir, ic in ((None, None), (rng.choice(2049, 999, replace=False) + 1, rng.choice(700, 333, replace=False) + 1)):
        nc = 700 if ic is None else ic.size
        y, c, s = rng.normal(size=nc), rng.uniform(0.1, 1.9, size=nc), rng.uniform(0.3, 2, size=nc)
        for cs in ((None, None), (c, s)):
            a, b = _xy(B, g3, y, ir, ic, *cs), _xy(B, g1, y, ir, ic, *cs)
            _same(a, b, "k_pmv vs k_pmvT")
            _same(a, fx.prod_pmv(G, ir, ic, y, *cs), "k_pmv")
    g3.close()
    g1.close()


def test_int32_caps_force_splits(B, rng):
    """More lines than one k_pmvT item may hold (65,537 columns) and more codes than one k_pmv item (262,145 samples):
    the forced splits add the same integers."""
    G = _codes(rng, 40, 65537, 0.0)
    g = _handle(B, G)
    y, c, s = rng.normal(size=65537), rng.uniform(0.1, 1.9, size=65537), rng.uniform(0.3, 2, size=65537)
    _same(_xy(B, g, y), fx.prod_T(G, None, None, y), "k_pmvT 65537 lines")
    _same(_xy(B, g, y, None, None, c, s), fx.prod_T(G, None, None, y, c, s), "k_pmvT 65537 lines, scaled")
    g.close()
    G = _codes(rng, 262145, 3, 0.01)
    g = _handle(B, G)
    yr = _vec(rng, 262145, dyadic=True)
    _same(_xty(B, g, yr), fx.cprod(G, None, None, yr, lists=True), "k_pmv 262145 codes")
    g.close()
    G = _codes(rng, 8, 262145, 0.0)
    g = _handle(B, G, B.LAYOUT_SNP_MAJOR | B.LAYOUT_SAMPLE_MAJOR)
    y = rng.normal(size=262145)
    _same(_xy(B, g, y), fx.prod_pmv(G, None, None, y), "k_pmv X.y 262145 codes")
    g.close()


# ---- vectors ------------------------------------------------------------------------------------------------------------
def _special_vectors(rng, k):
    e = 59  # exponent of a vector whose largest entry is 1
    out = {
        "zero": np.zeros(k),
        "one_nonzero": np.where(np.arange(k) == k // 2, -2.5, 0.0),
        "negative_zero": np.where(np.arange(k) % 3 == 0, -0.0, rng.normal(size=k)),
        "max_power_of_two": np.r_[4.0, rng.uniform(-4, 4, size=k - 1)],
        "max_below_one": np.r_[np.nextafter(1.0, 0), rng.uniform(-1, 1, size=k - 1)],
        "ties": np.r_[1.0, (2 * rng.integers(-1000, 1000, size=k - 1) + 1) * 2.0 ** (-e - 1)],
        "huge_tiny": np.where(np.arange(k) % 2 == 0, 1e300 * rng.uniform(0.5, 1, size=k), 1e-300),
        "subnormal": rng.integers(1, 1 << 20, size=k) * 2.0 ** -1074,
    }
    return out


@pytest.mark.parametrize("na_rate", [0.0, 0.1])
def test_special_vectors_match_the_model(B, rng, na_rate):
    n, m = 1025, 97
    G = _codes(rng, n, m, na_rate)
    handles = [(_handle(B, G), False)]
    if na_rate == 0.0:
        handles.append((_handle(B, G, B.LAYOUT_SNP_MAJOR | B.LAYOUT_SAMPLE_MAJOR), True))
    c, s = rng.uniform(0.1, 1.9, size=m), rng.uniform(0.3, 2, size=m)
    with np.errstate(over="ignore", under="ignore"):
        for g, pmv_x in handles:
            for name, y in _special_vectors(rng, m).items():
                scalings = [(None, None)]
                if name not in ("subnormal", "huge_tiny"):  # scaled: z = y / s leaves the tested range
                    scalings += [(np.zeros(m), s), (c, s)]
                for cs in scalings:
                    want = fx.prod_pmv(G, None, None, y, *cs) if pmv_x else fx.prod_T(G, None, None, y, *cs)
                    _same(_xy(B, g, y, None, None, *cs), want, "X.y %s scaled=%s" % (name, cs[0] is not None))
                yr = _special_vectors(rng, n)[name]
                _same(_xty(B, g, yr), fx.cprod(G, None, None, yr), "Xt.y %s" % name)
                if name not in ("subnormal", "huge_tiny"):
                    _same(_xty(B, g, yr, None, None, c, s), fx.cprod(G, None, None, yr, c, s), "Xt.y %s" % name)
            g.close()


@pytest.mark.parametrize("mult", [1, 2, 3, 16, 17])
def test_multisets_match_each_paths_model(B, rng, monkeypatch, mult):
    """Column and row multiplicities 1, 2, 3, 16, 17 (head-room bits 0 .. 5) on every missing-value mode."""
    n, m = 600, 120
    for rate, layouts, env in ((0.0, None, "1"), (0.0, 3, "1"), (0.005, None, "1"), (0.1, None, "1"), (0.005, None, "0")):
        G = _codes(rng, n, m, rate)
        monkeypatch.setenv("BSG_NA_LISTS", env)
        g = _handle(B, G, layouts)
        lists = _uses_lists(G, env_off=env == "0")
        ic = np.r_[np.repeat(rng.choice(m, 3, replace=False) + 1, mult), rng.integers(1, m + 1, 40)]
        ir = np.r_[np.repeat(rng.choice(n, 3, replace=False) + 1, mult), rng.integers(1, n + 1, 50)]
        _check_handle(B, g, G, rng, [(None, rng.permutation(ic)), (rng.permutation(ir), None), (ir, ic)], lists,
                      pmv_x=layouts == 3)
        g.close()


def test_repeated_missing_value_columns_do_not_overflow(B, oracle, obed_na):
    """A column holding missing values selected 16 times with y = 1 (16 x 2^59 = 2^63 before the exponent left
    head-room for duplicates), 9 times with y = 0.99, the eight missing-value columns of one sample twice each with the
    same large weight, and the same eight columns 256 times each with y just below one (where rint rounds every entry up
    to the binade, so the head-room needs its extra bit): the samples with a missing value there must still get the
    right sum."""
    G = oracle.decode_dense(obed_na)
    g = B.Bed(os.path.join(GOLDEN, "example-missing.bed"))
    assert _uses_lists(G)
    na_cols = np.nonzero((G == 3).any(axis=0))[0]
    i8 = int(np.argmax((G == 3).sum(axis=1)))
    cols8 = np.nonzero(G[i8] == 3)[0][:8]
    assert cols8.size == 8
    report = []
    for name, ic, y in (("16 x 1.0", np.full(16, na_cols[0] + 1), np.ones(16)),
                        ("9 x 0.99", np.full(9, na_cols[1] + 1), np.full(9, 0.99)),
                        ("8 columns x 2", np.repeat(cols8 + 1, 2), np.full(16, 1.0)),
                        ("8 columns x 256", np.repeat(cols8 + 1, 256), np.full(2048, np.nextafter(1.0, 0.0)))):
        got = _xy(B, g, y, None, ic)
        want = oracle.bed_prodVec(obed_na, y, None, ic)
        hit = (G[:, ic - 1] == 3).any(axis=1)
        err = np.abs(got - want)
        if np.max(err) >= 1e-12 * ic.size:
            report.append("%s: max error %.3g on the %d samples with a missing value, %.3g elsewhere"
                          % (name, np.max(err[hit]), hit.sum(), np.max(err[~hit], initial=0.0)))
        elif got.tobytes() != fx.prod_T(G, None, ic, y, lists=True).tobytes():
            report.append("%s: differs from the model" % name)
    g.close()
    assert not report, "; ".join(report)


def test_two_vectors_per_pass_match_the_model(B, oracle, obed, obed_na, rng):
    """prod_and_rowSumsSq: XV with the columns of V two per pass (30-bit fixed point each, slices 0..3 and 4..7), the
    odd one alone in slices 0..3, missing values on the flag plane; rowSumsSq from the raw, high-bit (k_pmvT2<2>) and
    missing-value plane sums."""
    for o in (obed_na, obed):
        G = oracle.decode_dense(o)
        n, m = G.shape
        g = B.Bed(o.bedfile)
        sc = oracle.bed_scaleBinom(o)
        for ir, ic in ((None, None), (rng.integers(1, n + 1, 77), rng.integers(1, m + 1, 301))):
            sel = np.arange(m) if ic is None else ic - 1
            irr = np.arange(1, n + 1) if ir is None else ir
            icc = np.arange(1, m + 1) if ic is None else ic
            c, s = sc["center"][sel], sc["scale"][sel]
            V = rng.normal(size=(sel.size, 3))
            XV, rss = B.prod_and_rowSumsSq(g, irr, icc, c, s, V)
            _same(XV, fx.prod_and_rowSumsSq_XV(G, ir, ic, c, s, V), "XV pair")
            _same(rss, fx.row_sums_sq(G, ir, ic, c, s), "rowSumsSq")
        g.close()


def test_device_pointer_entry_points_match_the_model(B, rng):
    """bsg_view_prodvec_dev / bsg_view_cprodvec_dev on device vectors: the same bytes as the model."""
    import torch

    G = _codes(rng, 3001, 515, 0.1)
    g = _handle(B, G)
    ir, ic = rng.integers(1, 3002, 1000), rng.integers(1, 516, 700)
    c, s = rng.uniform(0.1, 1.9, size=700), rng.uniform(0.3, 2, size=700)
    v = B.View(g, ir, ic, center=c, scale=s)
    try:  # the view goes before its handle, whatever the outcome
        dev = torch.device("cuda", 0)
        y, yr = rng.normal(size=700), rng.normal(size=1000)
        x_d, o_d = torch.tensor(y, device=dev), torch.empty(1000, dtype=torch.float64, device=dev)
        v.prodvec_dev(x_d.data_ptr(), o_d.data_ptr())
        xr_d, or_d = torch.tensor(yr, device=dev), torch.empty(700, dtype=torch.float64, device=dev)
        v.cprodvec_dev(xr_d.data_ptr(), or_d.data_ptr())
        torch.cuda.synchronize()
        _same(o_d.cpu().numpy(), fx.prod_T(G, ir, ic, y, c, s), "view prodvec_dev")
        _same(or_d.cpu().numpy(), fx.cprod(G, ir, ic, yr, c, s), "view cprodvec_dev")
    finally:
        v.close()
        g.close()


def test_identity_scaling_after_a_scaled_call_takes_the_unscaled_path(B, rng):
    """The 9-argument calls cache their view.  center = 0, scale = 1 after a scaled call on the same selection must give
    the unscaled path's bytes, as a first call does, not those of the cached scaled view."""
    G = _codes(rng, 1025, 97, 0.1)
    g = _handle(B, G)
    ir, ic = rng.integers(1, 1026, 500), rng.integers(1, 98, 60)
    y = rng.normal(size=60)
    want = fx.prod_T(G, ir, ic, y)
    c, s = rng.uniform(0.1, 1.9, size=60), rng.uniform(0.3, 2, size=60)
    _same(_xy(B, g, y, ir, ic, c, s), fx.prod_T(G, ir, ic, y, c, s), "scaled call")
    _same(_xy(B, g, y, ir, ic, np.zeros(60), np.ones(60)), want, "identity scaling after a scaled call")
    _same(_xy(B, g, y, ir, ic), want, "no scaling")
    g.close()


# ---- process-wide switches ----------------------------------------------------------------------------------------------
def _knob_inputs():
    """Seeded inputs of the switch runs (the child process and the parent build the same ones)."""
    rng = np.random.default_rng(77)
    out = []
    for name, n, m, rate, layouts in (("pmv", 3001, 2500, 0.0, 3), ("pmvt", 3001, 2500, 0.0, 1),
                                      ("plane", 2049, 1500, 0.1, 1), ("lists", 2049, 1500, 0.005, 1)):
        G = _codes(rng, n, m, rate)
        ir, ic = rng.integers(1, n + 1, n // 2), rng.integers(1, m + 1, m - 7)
        c, s = rng.uniform(0.1, 1.9, size=m), rng.uniform(0.3, 2, size=m)
        dy = rate > 0
        out.append(dict(name=name, G=G, layouts=layouts, ir=ir, ic=ic, c=c, s=s, y=_vec(rng, m, dy),
                        yc=_vec(rng, ic.size, dy), yr=_vec(rng, n, dy), V=rng.normal(size=(m, 3))))
    return out


def _knob_products(B, inputs):
    res = {}
    for d in inputs:
        g = _handle(B, d["G"], d["layouts"])
        k = d["name"]
        res[k + "_xy"] = _xy(B, g, d["y"])
        res[k + "_xy_sc"] = _xy(B, g, d["y"], None, None, d["c"], d["s"])
        res[k + "_xy_sel"] = _xy(B, g, d["yc"], d["ir"], d["ic"])
        res[k + "_xty"] = _xty(B, g, d["yr"])
        res[k + "_xty_sc"] = _xty(B, g, d["yr"], None, None, d["c"], d["s"])
        n, m = d["G"].shape
        res[k + "_xv"], res[k + "_rss"] = B.prod_and_rowSumsSq(g, np.arange(1, n + 1), np.arange(1, m + 1), d["c"], d["s"],
                                                               d["V"])
        U = np.linalg.qr(np.random.default_rng(5).normal(size=(n, 2)))[0]
        res[k + "_mlr"] = B.multLinReg(g, np.arange(1, n + 1), np.arange(1, m + 1), U)
        g.close()
    return res


_KNOB_RUN = r"""
import sys
sys.path.insert(0, sys.argv[1])
import numpy as np
import bigsnpr_b200 as B
from tests import test_gpu_fixedpoint as t
np.savez(sys.argv[2], **t._knob_products(B, t._knob_inputs()))
"""

_KNOBS = [{}, {"BSG_PMVT_KS": "1"}, {"BSG_PMVT_KS": "2"}, {"BSG_PMVT_KS": "5"}, {"BSG_PMVT_WAVES": "1"},
          {"BSG_PMVT_WAVES": "64"}, {"BSG_PMVT": "1"}, {"BSG_PROJ_PAIR": "0"}, {"BSG_MLR_PAIR": "0"}] + \
         [{"BSG_PMV_VARIANT": v} for v in ("11x2s0", "11x2s1", "11x2s2", "11x3s0", "11x3s1", "15x2s1")]


@pytest.fixture(scope="module")
def knob_model():
    inputs = _knob_inputs()
    want = {}
    for d in inputs:
        G, k, lists = d["G"], d["name"], d["name"] == "lists"
        n, m = G.shape
        pmv = d["layouts"] == 3
        prod = fx.prod_pmv if pmv else (lambda *a: fx.prod_T(*a, lists=lists))
        want[k + "_xy"] = prod(G, None, None, d["y"])
        want[k + "_xy_sc"] = prod(G, None, None, d["y"], d["c"], d["s"])
        want[k + "_xy_sel"] = prod(G, d["ir"], d["ic"], d["yc"])
        want[k + "_xty"] = fx.cprod(G, None, None, d["yr"], lists=lists)
        want[k + "_xty_sc"] = fx.cprod(G, None, None, d["yr"], d["c"], d["s"], lists=lists)
        want[k + "_xv"] = fx.prod_and_rowSumsSq_XV(G, None, None, d["c"], d["s"], d["V"])
        want[k + "_xv_single"] = (np.stack([fx.prod_pmv(G, None, None, d["V"][:, j], d["c"], d["s"]) for j in range(3)], 1)
                                  if pmv else fx.prod_and_rowSumsSq_XV(G, None, None, d["c"], d["s"], d["V"], pair=False,
                                                                       lists=lists))
        want[k + "_rss"] = fx.row_sums_sq(G, None, None, d["c"], d["s"], pmv=pmv)
        want[k + "_rss_T"] = fx.row_sums_sq(G, None, None, d["c"], d["s"])
        want[k + "_xy_T"] = fx.prod_T(G, None, None, d["y"], lists=lists)
        want[k + "_xy_sc_T"] = fx.prod_T(G, None, None, d["y"], d["c"], d["s"], lists=lists)
        want[k + "_xy_sel_T"] = fx.prod_T(G, d["ir"], d["ic"], d["yc"], lists=lists)
    return want


@pytest.fixture(scope="module")
def knob_default(B):
    """The switch runs' products in this process (default settings)."""
    return _knob_products(B, _knob_inputs())


@pytest.mark.parametrize("env", _KNOBS, ids=lambda e: ",".join("%s=%s" % kv for kv in e.items()) or "default")
def test_process_switches_give_the_models_bytes(B, knob_model, knob_default, env, tmp_path):
    """Each switch is read once per process, hence one subprocess per setting: k-split counts 1 / 2 / 5, 1 and 64 waves,
    every compiled k_pmv variant, X.y forced onto the SNP-major kernel, and the one-vector-per-pass projection and
    multLinReg.  Products and prod_and_rowSumsSq's rowSumsSq (high-bit and missing-value planes) must equal the model's
    bytes.  multLinReg's t-scores (its fp64 regression formula is not
    modelled) must equal the default settings' bytes, except with one column of U per pass: 61-bit sums instead of
    30-bit ones change the last bits, so those agree to the 30-bit format's accuracy."""
    res = tmp_path / "knob.npz"
    r = subprocess.run([sys.executable, "-c", _KNOB_RUN, ROOT, str(res)], capture_output=True, text=True,
                       env=dict(os.environ, **env), timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = np.load(res)
    forced_t = env.get("BSG_PMVT") == "1"
    for k in ("pmv", "pmvt", "plane", "lists"):
        for p in ("_xy", "_xy_sc", "_xy_sel"):
            key = k + p + ("_T" if forced_t and k == "pmv" else "")
            _same(got[k + p], knob_model[key], "%s %s" % (env, k + p))
        for p in ("_xty", "_xty_sc"):
            _same(got[k + p], knob_model[k + p], "%s %s" % (env, k + p))
        _same(got[k + "_rss"], knob_model[k + "_rss" + ("_T" if forced_t and k == "pmv" else "")], "%s %s_rss" % (env, k))
        xv = knob_model[k + ("_xv_single" if env.get("BSG_PROJ_PAIR") == "0" else "_xv")]
        _same(got[k + "_xv"], xv, "%s %s_xv" % (env, k))
    for k in ("pmv", "pmvt", "plane", "lists"):
        a, b = got[k + "_mlr"], knob_default[k + "_mlr"]
        assert np.array_equal(np.isnan(a), np.isnan(b)) and np.isfinite(b).any()
        if env.get("BSG_MLR_PAIR") == "0":
            ok = np.isfinite(b)
            assert np.max(np.abs(a[ok] - b[ok]) / (1.0 + np.abs(b[ok]))) < 1e-7
        else:
            _same(a, b, "%s %s_mlr" % (env, k))
