"""CPU checks of the C+T score references (tests/prs_ref.py) and of snp_PRS's argument checks: the exact model of the
device arithmetic against R's literal loop, the step rule (unsorted and tied thresholds, a threshold equal to an lpS,
empty steps, thresholding disabled), reversed alleles, and the new kernels' PTX having no fused multiply-add."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import bigsnpr_b200 as B
from tests import prs_ref as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def codes(rng, n, m, na_rate=0.0):
    G = rng.integers(0, 3, size=(n, m))
    if na_rate:
        G[rng.random((n, m)) < na_rate] = 3
    return G


def bound(G, ind_row, cols, beta, same):
    """sum_j |g_ij - 2 rev_j| 2^(-e-1) (quantisation) + 64 ulps of the largest score (fp64 chains)."""
    v, e = P.set_exponent(beta, same)
    X = np.asarray(G)[np.asarray(ind_row) - 1][:, np.asarray(cols) - 1].astype(np.float64)
    w = np.abs(X - 2 * (~np.asarray(same, dtype=bool)))
    return w.sum(axis=1) * 2.0 ** (-e - 1)


@pytest.mark.parametrize("na_rate", [0.0, 0.05])
def test_exact_model_within_bound_of_literal(na_rate):
    rng = np.random.default_rng(3)
    G = codes(rng, 150, 400, na_rate)
    ir = rng.integers(1, 151, size=90)
    cols = rng.choice(400, 250, replace=True) + 1
    beta = rng.normal(size=cols.size) * 10.0 ** rng.integers(-3, 2, size=cols.size)
    same = rng.random(cols.size) < 0.7
    lpS = rng.exponential(2.0, size=cols.size)
    thr = rng.permutation(np.linspace(0, 5, 11))
    a = P.exact(G, ir, cols, beta, same, lpS, thr)
    b = P.literal(G, ir, cols, beta, same, lpS, thr)
    assert np.array_equal(np.isnan(a), np.isnan(b))
    ok = ~np.isnan(a)
    tol = bound(G, ir, cols, beta, same)[:, None] + 64 * np.finfo(float).eps * np.nanmax(np.abs(b))
    assert np.all(np.abs(a - b)[ok] <= np.broadcast_to(tol, a.shape)[ok])
    if na_rate:
        assert np.isnan(a).any() and not np.isnan(a).all()


def test_steps_strict_ties_unsorted_empty():
    lpS = np.array([0.5, 2.0, 1.0, 3.0, 1.0, 0.0])
    thr = np.array([1.0, 3.0, 0.0, 1.0, 10.0])
    st, ordr = P.steps_of(lpS, thr, lpS.size)
    assert list(ordr) == [4, 1, 0, 3, 2]                 # stable decreasing: the first 1.0 before the second
    # 10: none; 3: none (strict, 3.0 is not > 3); first 1.0: 2.0 and 3.0; second 1.0: none left; 0: 0.5, 1.0, 1.0
    assert list(st) == [4, 2, 4, 2, 4, -1]
    rng = np.random.default_rng(0)
    G = codes(rng, 40, 6)
    beta = rng.normal(size=6)
    for f in (P.literal, P.exact):
        s = f(G, np.arange(1, 41), np.arange(1, 7), beta, None, lpS, thr)
        assert np.array_equal(s[:, 0], s[:, 3])           # tied thresholds: equal columns
        assert np.all(s[:, 4] == 0) and np.all(s[:, 1] == 0)  # empty steps add 0
        # unsorted thresholds: the same columns as sorted ones, permuted
        s2 = f(G, np.arange(1, 41), np.arange(1, 7), beta, None, lpS, np.sort(thr))
        assert np.array_equal(s[:, np.argsort(thr, kind="stable")], s2)


def test_thresholding_disabled_is_one_column_over_all():
    rng = np.random.default_rng(1)
    G = codes(rng, 30, 20)
    beta = rng.normal(size=20)
    a = P.literal(G, np.arange(1, 31), np.arange(1, 21), beta, None, None, None)
    assert a.shape == (30, 1)
    assert np.allclose(a[:, 0], G.astype(float) @ beta, rtol=1e-13, atol=1e-13)
    e = P.exact(G, np.arange(1, 31), np.arange(1, 21), beta, None, None, None)
    assert np.abs(e - a).max() <= 1e-13


def test_reversed_alleles():
    """prodVecRev: g (-beta) + 2 beta = (2 - g) beta for a SNP whose reference allele is swapped."""
    rng = np.random.default_rng(2)
    G = codes(rng, 25, 10)
    beta = rng.normal(size=10)
    same = np.array([True, False] * 5)
    want = (np.where(same, G, 2 - G).astype(float) @ beta)
    for f in (P.literal, P.exact):
        got = f(G, np.arange(1, 26), np.arange(1, 11), beta, same, None, None)[:, 0]
        assert np.allclose(got, want, rtol=1e-13, atol=1e-12)


def _fake_bed(n, m):
    return B.Bed(_handle=ctypes.c_void_p(), _shape=(n, m))


def test_snp_PRS_argument_checks():
    G = _fake_bed(10, 5)
    b = np.ones(5)
    with pytest.raises(TypeError, match="logical"):
        B.snp_PRS(G, b, same_keep=np.ones(5))
    with pytest.raises(ValueError, match="missing value"):
        B.snp_PRS(G, b, same_keep=np.array([True, None, True, True, True], dtype=object))
    with pytest.raises(ValueError, match="dimensions"):
        B.snp_PRS(G, b, same_keep=np.ones(4, dtype=bool))
    with pytest.raises(ValueError, match="dimensions"):
        B.snp_PRS(G, np.ones(4))
    with pytest.raises(ValueError, match="dimensions"):
        B.snp_PRS(G, b, lpS_keep=np.ones(4), thr_list=[1.0])
    with pytest.raises(ValueError, match="non-negative"):
        B.snp_PRS(G, b, lpS_keep=np.array([1, 2, -1, 0, 0.0]), thr_list=[1.0])
    with pytest.raises(ValueError, match="missing values"):
        B.snp_PRS(G, b, lpS_keep=np.array([1, 2, np.nan, 0, 0.0]), thr_list=[1.0])
    with pytest.raises(TypeError):
        B.snp_PRS(np.zeros((10, 5)), b)
    with pytest.raises(ValueError, match="type"):
        B.snp_grid_PRS(G, [[np.arange(1, 6)]], b, b, type="int")


def test_prs_kernels_ptx_have_no_fma(tmp_path):
    """Every fp64 add of the score combine, the literal loop and the constant rounds on its own (no contraction)."""
    ptx = tmp_path / "prs.ptx"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-ptx", "-arch=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-I",
                           os.path.join(ROOT, "bigsnpr_b200", "csrc"),
                           os.path.join(ROOT, "bigsnpr_b200", "csrc", "bsg_prs.cu"), "-o", str(ptx)])
    bodies = [(n.split("ILb")[0], b) for n, b in re.findall(r"\.entry \w*?(k_prs\w*?)E\w*\((.*?)\n}\n", ptx.read_text(), re.S)]
    names = {n for n, _ in bodies}
    assert names == {"k_prs", "k_prs_dos", "k_prs_const", "k_prs_literal", "k_prs_gather"}, names
    for name, body in bodies:
        assert "fma.rn.f64" not in body, name
    k = [b for n, b in bodies if n == "k_prs"]
    assert len(k) == 2 and all("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32" in b and "add.rn.f64" in b for b in k)


GOLD = os.path.join(ROOT, "tests", "golden")


def reference_fixture(G):
    """snp_PRS of tests/testthat/test-6-PRS.R:34-44 (tests/golden/prs_scores.npz, 517 x 11 at thresholds 0, 0.5, .., 5)
    with the keep set of clumping.rds and lpS = -log10(pval.rds) (tests/golden/prs_clumping.npz).  The GWAS betas are not
    stored, so they are recovered: under the strict > rule, the increment of column t (threshold 0.5 t) over column
    t + 1 is G[, S_t] beta[S_t] with S_t the kept SNPs whose lpS lies in (0.5 t, 0.5 (t + 1)] (above 5 for the last
    column), and beta[S_t] is its least-squares solution.  Columns 4-11 (thresholds 1.5 .. 5) fit to <= 4e-14; the
    columns at 1.0 and below were made with a slightly different keep set (the 1.0 step fits only with 360 SNPs instead
    of 355), so they cannot pin anything and the betas of SNPs at lpS <= 1.5 stay 0.  Returns (keep, lpS, beta, scores,
    thresholds, selection sizes, largest relative residual)."""
    gold = np.load(os.path.join(GOLD, "prs_scores.npz"))
    cl = np.load(os.path.join(GOLD, "prs_clumping.npz"))
    keep = np.asarray(cl["keep"], dtype=np.int64)
    lpS = -np.log10(cl["pval"][keep - 1])
    scores, thr = gold["scores"], gold["thr"]
    X = np.asarray(G, dtype=np.float64)[:, keep - 1]
    beta = np.zeros(keep.size)
    sizes, resid = [], 0.0
    for t in range(3, 11):
        sel = (lpS > thr[t]) & ((lpS <= thr[t + 1]) if t < 10 else True)
        inc = scores[:, t] - (scores[:, t + 1] if t < 10 else 0.0)
        b, *_ = np.linalg.lstsq(X[:, sel], inc, rcond=None)
        beta[sel] = b
        sizes.append(int(sel.sum()))
        resid = max(resid, np.max(np.abs(X[:, sel] @ b - inc)) / np.max(np.abs(inc)))
    return keep, lpS, beta, scores, thr, sizes, resid


def test_reference_scores_reproduced(obed, oracle):
    """R's own snp_PRS output, thresholds 1.5 .. 5: the step rule (strict >, cumulative over decreasing thresholds) must
    reproduce it from the recovered betas, in the literal restatement and in the exact model of the device."""
    G = oracle.decode_dense(obed)
    keep, lpS, beta, scores, thr, sizes, resid = reference_fixture(G)
    assert sizes == [92, 28, 10, 1, 1, 2, 2, 3] and resid <= 4e-14
    ir = np.arange(1, G.shape[0] + 1)
    for f in (P.literal, P.exact):
        got = f(G, ir, keep, beta, None, lpS, thr)
        assert np.max(np.abs(got[:, 3:] - scores[:, 3:])) <= 1e-12
        # unsorted thresholds give the same columns
        perm = np.random.default_rng(0).permutation(thr.size)
        assert np.array_equal(f(G, ir, keep, beta, None, lpS, thr[perm]), got[:, perm])
