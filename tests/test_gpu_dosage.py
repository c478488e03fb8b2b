"""Dosage FBM.code256 handles (CODE_DOSAGE, R/bigSNP-class.R:13) on the byte-operand tensor-pipe kernels: X.y, Xt.y and
bed_randomSVD against literal per-element fp64 loops over code256[byte] (SubBMCode256Acc with bigstatsr's scaling,
(code256[b] - c) / s, NA code = NA_real), written out here in NumPy.

Tolerance: 1e-12 of max |ref| (the kernels sum exactly in 61-bit fixed point and apply 1/D once; the literal loop rounds
after every fp64 add).  NaN patterns must match exactly.
"""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# CODE_DOSAGE: 0, 1, 2, NA, 0, 1, 2, seq(0, 2, by = 0.01), NA x 48
CODE_DOSAGE = np.concatenate([[0, 1, 2, np.nan, 0, 1, 2], 0 + np.arange(201) * 0.01, np.full(48, np.nan)])


@pytest.fixture(scope="module")
def B():
    import bigsnpr_b200 as b

    from bigsnpr_b200 import build

    build.build()
    return b


def _mean2(G):
    """src/impute-simple.cpp, method "mean2": a missing call (code 3) becomes the column mean of the observed calls rounded
    to 2 decimals, stored as code 7 + 100 * value of CODE_DOSAGE (ties at exact .5 may round differently from R)."""
    G = G.astype(np.uint8).copy()
    for j in range(G.shape[1]):
        na = G[:, j] == 3
        if na.any():
            mu = G[~na, j].mean() if (~na).any() else 0.0
            G[na, j] = 7 + int(np.rint(100 * mu))
    return G


def _mixed(rng, n, m, na_rate=0.0):
    """Codes 0-2, 4-6 and 7-207 mixed (several bytes map to the same value) with LD-like column blocks."""
    lat = rng.normal(size=(n, (m + 19) // 20))
    prob = 1 / (1 + np.exp(-(0.9 * lat[:, np.arange(m) // 20] + 0.6 * rng.normal(size=(n, m)))))
    val = np.clip(np.rint(200 * prob), 0, 200).astype(np.int64)  # dosage x 100
    G = (7 + val).astype(np.uint8)
    hard = rng.random(size=(n, m)) < 0.3
    hv = np.clip(np.rint(val / 100.0), 0, 2).astype(np.int64)
    alt = rng.random(size=(n, m)) < 0.5
    G[hard] = (hv + np.where(alt, 4, 0))[hard].astype(np.uint8)
    if na_rate > 0:
        na = rng.random(size=(n, m)) < na_rate
        G[na] = np.where(rng.random(size=(n, m)) < 0.5, 3, 230)[na].astype(np.uint8)
    return G


def _X(G, ir, ic, center, scale):
    with np.errstate(all="ignore"):
        return (CODE_DOSAGE[G[np.ix_(ir - 1, ic - 1)]] - center) / scale


def _lit_prod(G, ir, ic, center, scale, x):
    with np.errstate(all="ignore"):
        return (_X(G, ir, ic, center, scale) * x[None, :]).sum(axis=1)


def _lit_cprod(G, ir, ic, center, scale, y):
    with np.errstate(all="ignore"):
        return (_X(G, ir, ic, center, scale) * y[:, None]).sum(axis=0)


def _check(got, want, tol=1e-12):
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    if ok.any():
        s = max(np.max(np.abs(want[ok])), 1e-300)
        assert np.max(np.abs(got[ok] - want[ok])) / s < tol


def _products(B, G, rng, with_na):
    n, m = G.shape
    g = B.Bed.from_fbm(G, code256=CODE_DOSAGE)
    assert g.dosage_scale == 100
    try:
        sels = [(np.arange(1, n + 1, dtype=np.int32), np.arange(1, m + 1, dtype=np.int32))]
        # tests/testthat/test-5-bed-prod-vec.R:18-41: subsets with replacement, unsorted
        sels.append((rng.integers(1, n + 1, size=n // 2).astype(np.int32), rng.integers(1, m + 1, size=m // 2).astype(np.int32)))
        sels.append((np.arange(1, n + 1, dtype=np.int32), rng.permutation(m)[: m // 3].astype(np.int32) + 1))  # column list
        for ir, ic in sels:
            for scaled in (False, True):
                if scaled:
                    c, s = rng.uniform(0, 2, size=ic.size), rng.uniform(0.2, 1.5, size=ic.size)
                else:
                    c, s = np.zeros(ic.size), np.ones(ic.size)
                x, y = rng.normal(size=ic.size), rng.normal(size=ir.size)
                a = B.bed_prodVec(g, x, ir, ic, c, s)
                b = B.bed_cprodVec(g, y, ir, ic, c, s)
                _check(a, _lit_prod(G, ir, ic, c, s, x))
                _check(b, _lit_cprod(G, ir, ic, c, s, y))
                if with_na:
                    assert np.isnan(a).any() and np.isnan(b).any()
    finally:
        g.close()


def test_dosage_products_synthetic(B):
    rng = np.random.default_rng(1)
    _products(B, _mixed(rng, 1303, 1117), rng, with_na=False)


def test_dosage_products_with_na_codes(B):
    rng = np.random.default_rng(2)
    _products(B, _mixed(rng, 777, 901, na_rate=0.002), rng, with_na=True)


def test_dosage_products_mean2_imputed_example(B):
    rng = np.random.default_rng(3)
    gb = B.Bed(os.path.join(GOLDEN, "example-missing.bed"))
    codes = gb[None, None]
    gb.close()
    codes = np.where(codes == B.NA_INTEGER, 3, codes)
    G = _mean2(codes)
    assert (G >= 7).any() and not (G == 3).any()
    _products(B, G, rng, with_na=False)


def test_dosage_zero_scale_host_and_dev(B):
    import torch

    rng = np.random.default_rng(4)
    G = _mixed(rng, 401, 333)
    n, m = G.shape
    g = B.Bed.from_fbm(G, code256=CODE_DOSAGE)
    ir, ic = np.arange(1, n + 1, dtype=np.int32), np.arange(1, m + 1, dtype=np.int32)
    c, s = rng.uniform(0, 2, size=m), rng.uniform(0.2, 1.5, size=m)
    s[17] = 0.0
    x, y = rng.normal(size=m), rng.normal(size=n)
    # host forms: the literal loop, element for element
    a, b = B.bed_prodVec(g, x, ir, ic, c, s), B.bed_cprodVec(g, y, ir, ic, c, s)
    with np.errstate(all="ignore"):
        a0, b0 = _lit_prod(G, ir, ic, c, s, x), _lit_cprod(G, ir, ic, c, s, y)
    assert np.array_equal(np.isnan(a), np.isnan(a0)) and np.array_equal(np.isinf(a), np.isinf(a0))
    assert np.array_equal(np.isnan(b), np.isnan(b0)) and np.array_equal(np.isinf(b), np.isinf(b0))
    fin = np.isfinite(b0)
    assert fin.sum() == m - 1 and np.max(np.abs(b[fin] - b0[fin])) / np.max(np.abs(b0[fin])) < 1e-12
    # device forms: all NaN
    v = B.View(g, ir, ic, c, s)
    xd, yd = torch.tensor(x, device="cuda"), torch.tensor(y, device="cuda")
    od, oc = torch.empty(n, dtype=torch.float64, device="cuda"), torch.empty(m, dtype=torch.float64, device="cuda")
    v.prodvec_dev(xd.data_ptr(), od.data_ptr())
    v.cprodvec_dev(yd.data_ptr(), oc.data_ptr())
    torch.cuda.synchronize()
    assert torch.isnan(od).all() and torch.isnan(oc).all()
    v.close()
    g.close()


@pytest.mark.parametrize("shape", [(300, 70000), (70000, 300)])
def test_dosage_forced_ksplit_is_bit_identical(B, shape):
    rng = np.random.default_rng(5)
    n, m = shape
    G = (7 + rng.integers(0, 201, size=(n, m))).astype(np.uint8)
    G[:, -10:][rng.random(size=(n, 10)) < 0.2] = 255  # 255: NA in CODE_DOSAGE, only in the 10 unselected columns
    g = B.Bed.from_fbm(G, code256=CODE_DOSAGE)
    ic = np.arange(1, m - 10 + 1, dtype=np.int32)  # X.y at 300 x 70,000 contracts over 69,990 > 65,536 lines
    c, s = rng.uniform(0, 2, size=ic.size), rng.uniform(0.2, 1.5, size=ic.size)
    x, y = rng.normal(size=ic.size), rng.normal(size=n)
    outs = []
    old = os.environ.get("BSG_DMV_KS")
    try:
        for ks in ("1", "3", "0"):
            os.environ["BSG_DMV_KS"] = ks
            outs.append((B.bed_prodVec(g, x, ind_col=ic, center=c, scale=s),
                         B.bed_cprodVec(g, y, ind_col=ic, center=c, scale=s),
                         B.bed_prodVec(g, x[: ic.size], ind_col=ic[::-1].copy(), center=c, scale=s)))
    finally:
        if old is None:
            os.environ.pop("BSG_DMV_KS", None)
        else:
            os.environ["BSG_DMV_KS"] = old
    for o in outs[1:]:
        for u, w in zip(o, outs[0]):
            assert u.tobytes() == w.tobytes()
    ir = np.arange(1, n + 1, dtype=np.int32)
    _check(outs[0][0], _lit_prod(G, ir, ic, c, s, x))
    _check(outs[0][1], _lit_cprod(G, ir, ic, c, s, y))
    g.close()


def test_dosage_randomsvd_vs_dense(B):
    rng = np.random.default_rng(6)
    G = _mixed(rng, 600, 900)
    g = B.Bed.from_fbm(G, code256=CODE_DOSAGE)
    k = 5
    svd = B.bed_randomSVD(g, fun_scaling=B.snp_scaleBinom(), k=k)
    ir, ic = np.arange(1, 601, dtype=np.int32), np.arange(1, 901, dtype=np.int32)
    st = B.snp_scaleBinom()(g)
    X = _X(G, ir, ic, st["center"], st["scale"])
    U, d, Vt = np.linalg.svd(X, full_matrices=False)
    assert np.max(np.abs(svd["d"] - d[:k]) / d[:k]) < 1e-7
    assert np.min(np.abs(np.sum(svd["u"] * U[:, :k], axis=0))) > 1 - 1e-6
    assert np.min(np.abs(np.sum(svd["v"] * Vt[:k].T, axis=0))) > 1 - 1e-6
    with pytest.raises(B.BsgError, match="needs hard calls"):  # the NULL default is bed_scaleBinom: counts of hard calls
        B.bed_randomSVD(g, k=k)
    g.close()


def test_non_dosage_tables_keep_their_refusal(B):
    G = np.zeros((20, 10), dtype=np.uint8)
    g = B.Bed.from_fbm(G, code256=np.linspace(0, 2, 256))
    assert g.dosage_scale == 0
    with pytest.raises(B.BsgError, match="needs hard calls"):
        B.bed_prodVec(g, np.ones(10))
    g.close()
    g = B.Bed.from_fbm(G, code256=CODE_DOSAGE)
    with pytest.raises(B.BsgError, match="needs hard calls"):
        B.prod_and_rowSumsSq(g, np.arange(1, 21), np.arange(1, 11), np.zeros(10), np.ones(10), np.ones((10, 2)))
    g.close()
