"""The exact model of the GRM's arithmetic (tests/grm_ref.py) against the oracle, on the CPU.

* at 9 digit slices the quantisation is far below fp64 noise, so the model must agree with oracle.bed_tcrossprodSelf to
  about 1e-13 of max|K|: this checks the weights, the missing-value decomposition and the vector terms;
* at the library's 4 slices, one exponent per weight vector (the quantisation before weight classes) loses bits on
  every column whose W1 is far below the maximum: a single MAC-1 or MAC-2 column, or a caller's scaling with a cohort
  allele frequency near 0 or 1, pushes the error of K past 1e-8 of max|K|.  With the weight classes it stays below;
* an input whose weights form one class is computed exactly as before the classes existed.

The device is held to the model byte for byte in tests/test_gpu_grm.py, so these errors are the device's.
"""
import os

import numpy as np
import pytest

from tests import grm_ref as gr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _codes(rng, n, m, na_rate=0.0, maf_lo=0.02):
    p = rng.uniform(maf_lo, 0.5, size=m)
    G = rng.binomial(2, p[None, :], size=(n, m)).astype(np.uint8)
    if na_rate:
        G[rng.random((n, m)) < na_rate] = 3
    return G


def _binom(G, ir=None, ic=None):
    r0 = np.arange(G.shape[0]) if ir is None else np.asarray(ir) - 1
    c0 = np.arange(G.shape[1]) if ic is None else np.asarray(ic) - 1
    Gs = G[np.ix_(r0, c0)]
    nona = (Gs != 3).sum(axis=0)
    af = np.where(Gs == 3, 0, Gs).sum(axis=0) / (2.0 * nona)
    return 2 * af, np.sqrt(2 * af * (1 - af))


def _oracle_K(oracle, G, center, scale, ir=None, ic=None):
    n, m = G.shape
    o = oracle.OracleBed.from_packed(oracle.write_bed_bytes(G), n, m)
    fun = lambda *_a, **_k: {"center": center, "scale": scale}  # noqa: E731
    return oracle.bed_tcrossprodSelf(o, fun, ir, ic, block_size=max(1, m if ic is None else len(ic)))[0]


def _rel(K, K0):
    return float(np.max(np.abs(K - K0)) / np.max(np.abs(K0)))


def _cohort(center, scale, cols, p):
    """Caller's scaling with a cohort allele frequency p on the given columns."""
    c, s = center.copy(), scale.copy()
    c[cols] = 2 * p
    s[cols] = np.sqrt(2 * p * (1 - p))
    return c, s


def _mac(G, col, mac):
    """Column `col` holds exactly `mac` copies of the minor allele (hard calls, no missing value)."""
    G[:, col] = 0
    G[:mac, col] = 1


# ---- the algebra: 9 slices against the oracle ---------------------------------------------------------------------------
@pytest.mark.parametrize("na_rate", [0.0, 0.01, 0.1])
@pytest.mark.parametrize("sel", ["all", "subset", "multiset"])
def test_model_matches_the_oracle_at_nine_slices(oracle, rng, na_rate, sel):
    G = _codes(rng, 160, 700, na_rate)
    n, m = G.shape
    ir = ic = None
    if sel == "subset":
        ir, ic = np.sort(rng.choice(n, 97, replace=False)) + 1, np.sort(rng.choice(m, 401, replace=False)) + 1
    elif sel == "multiset":
        ir, ic = rng.integers(1, n + 1, 131), rng.integers(1, m + 1, 523)
    c, s = _binom(G, ir, ic)
    if na_rate:
        c, s = _cohort(c, s, [3, 5], 1 - 2e-6)  # W2' and W3 as large as W1 on these columns
    K0 = _oracle_K(oracle, G, c, s, ir, ic)
    lists = 0 < np.mean(G == 3) <= 0.04
    K = gr.tcrossprod(G, c, s, ir, ic, nslices=9, path="wgram", lists=lists)  # more than 4 slices: k_wgram5's order
    assert _rel(K, K0) < 1e-13, _rel(K, K0)
    assert np.array_equal(K, K.T)


def test_example_bed_matches_the_oracle(oracle, obed_na):
    G = oracle.decode_dense(obed_na)
    c, s = _binom(G)
    K0 = oracle.bed_tcrossprodSelf(obed_na)[0]
    assert _rel(gr.tcrossprod(G, c, s, nslices=9, path="wgram", lists=True), K0) < 1e-13
    assert _rel(gr.tcrossprod(G, c, s, lists=True), K0) < 1e-8


# ---- precision of the 4-slice quantisation ----------------------------------------------------------------------------------
def _skewed_cases(rng):
    """(name, G, center, scale, na): inputs whose W1 spans orders of magnitude."""
    out = []
    for mac in (1, 2):
        G = _codes(rng, 1000, 2000)
        _mac(G, 17, mac)
        out.append(("MAC-%d" % mac, G) + _binom(G))
    for p in (2e-6, 1 - 2e-6):
        for na in (0.0, 0.01):
            G = _codes(rng, 600, 1500, na)
            c, s = _cohort(*_binom(G), [0, 700, 1499], p)
            out.append(("cohort p=%g na=%g" % (p, na), G, c, s))
    return out


def test_one_exponent_per_weight_loses_precision_and_weight_classes_keep_it(oracle, rng):
    report = []
    for name, G, c, s in _skewed_cases(rng):
        K0 = _oracle_K(oracle, G, c, s)
        lists = 0 < np.mean(G == 3) <= 0.04
        old = _rel(gr.tcrossprod(G, c, s, lists=lists, old_classes=True), K0)
        new = _rel(gr.tcrossprod(G, c, s, lists=lists), K0)
        new5 = _rel(gr.tcrossprod(G, c, s, path="wgram", lists=lists), K0)
        assert gr.n_classes(c, s) > 1, name
        report.append((name, old, new, new5))
    msg = "\n".join("%s: one exponent %.2g, classes %.2g (k_wgram5 order %.2g)" % r for r in report)
    assert all(r[1] > 1e-8 for r in report), msg
    assert all(r[2] < 1e-8 and r[3] < 1e-8 for r in report), msg


def test_unskewed_inputs_stay_inside_the_design_bound(oracle, rng):
    """MAF U(0.02, 0.5), the synthetic generator's range: K within 1e-8 of max|K| either way."""
    G = _codes(rng, 500, 4000, 0.01)
    c, s = _binom(G)
    K0 = _oracle_K(oracle, G, c, s)
    assert _rel(gr.tcrossprod(G, c, s, lists=True), K0) < 1e-8


# ---- the class rule -----------------------------------------------------------------------------------------------------------
def test_weight_classes_bound_the_spread_inside_each_class(rng):
    W1 = np.exp(rng.uniform(-40, 3.4, size=5000))
    W1[:3] = [0.0, 2.0 ** 5, np.nextafter(2.0 ** 1, np.inf)]
    cls = gr.weight_classes(W1)
    assert cls[0] == 0 and cls[1] == 0 and cls[2] == 0  # W1 in (max / 16, max]: one class across four binades
    for c in np.unique(cls):
        w = W1[(cls == c) & (W1 > 0)]
        if w.size:
            assert w.min() * 16 > w.max(), c
    # the boundaries are exact: class c holds max / 16^(c+1) < W1 <= max / 16^c
    m = W1.max()
    pos = W1 > 0
    assert np.all(W1[pos] * 16.0 ** cls[pos] <= m) and np.all(W1[pos] * 16.0 ** (cls[pos] + 1) > m)
    edge = np.r_[m, m / 16, np.nextafter(m / 16, np.inf), np.nextafter(m / 16, 0), m / 256, np.nextafter(m / 256, 0)]
    assert gr.weight_classes(np.r_[W1, edge])[-6:].tolist() == [0, 1, 0, 1, 2, 2]


def test_one_class_inputs_are_computed_as_before(oracle, rng, obed):
    """The synthetic data of the benchmarks (allele frequencies in U(0.02, 0.5): W1 in [2, 25.5]) and the golden
    example.bed form one class, and one class gives the bytes of the single-exponent quantisation."""
    assert gr.n_classes(np.r_[0.04, 1.0], np.sqrt([2 * 0.02 * 0.98, 0.5])) == 1
    G0 = oracle.decode_dense(obed)
    assert gr.n_classes(*_binom(G0)) == 1
    for na in (0.0, 0.01):
        G = _codes(rng, 300, 1200, na, maf_lo=0.1)
        c, s = _binom(G)
        assert gr.n_classes(c, s) == 1
        for path, ns in (("gramt", 4), ("gramt", 3), ("wgram", 5)):
            a = gr.tcrossprod(G, c, s, nslices=ns, path=path, lists=na > 0)
            b = gr.tcrossprod(G, c, s, nslices=ns, path=path, lists=na > 0, old_classes=True)
            assert a.tobytes() == b.tobytes()


def test_degenerate_scaling_is_left_to_dsyrk():
    W = gr.grm_weights(np.r_[1.0, -0.5], np.r_[1.0, 1.0])
    assert gr.degenerate(*W[:3])  # negative center: W2' < 0
    W = gr.grm_weights(np.r_[1.0, 1.0], np.r_[1.0, 0.0])
    assert gr.degenerate(*W[:3])  # zero scale
    W = gr.grm_weights(np.r_[1.0, 1.0], np.r_[1.0, -2.0])
    assert not gr.degenerate(*W[:3])  # a negative scale changes no weight's sign: W2' = c / s^2
