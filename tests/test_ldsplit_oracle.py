"""The snp_ldsplit oracle (tests/ldsplit_oracle.c + tests/ldsplit_ref.py) against facts that do not depend on it: every
expectation of tests/testthat/test-4-split-LD.R, the costs of the reference's split_before.rds fixture, costs recomputed
by brute force from the blocks, and an exhaustive search over every split of small matrices.  Also the host side of
api.snp_ldsplit (argument checks, the lower triangle from each input form) and the kernels' PTX.  No GPU needed."""
import itertools
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from bigsnpr_b200 import api
from tests import ldsplit_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NA = R.NA_INTEGER
INF = np.inf


def outer4():
    """tests/testthat/test-4-split-LD.R:9-10: outer(1:4 / 10, 1:4 / 10, '+') with a unit diagonal."""
    c = np.add.outer(np.arange(1, 5) / 10, np.arange(1, 5) / 10)
    np.fill_diagonal(c, 1)
    return c


def spmat():
    """spMat.rds and split_before.rds, parsed into tests/golden/ldsplit.npz by tests/golden/make_ldsplit_golden.py."""
    d = np.load(os.path.join(ROOT, "tests", "golden", "ldsplit.npz"))
    assert str(d["uplo"][0]) == "U"
    A = sp.csc_matrix((d["x"], d["i"], d["p"]), shape=tuple(d["Dim"]))
    return A, d["before_cost"], d["before_n_block"]


def r_equal(target, current, tol=1.5e-8):
    """testthat's expect_equal on numbers (all.equal): mean relative difference below tol."""
    target, current = np.asarray(target, dtype=float), np.asarray(current, dtype=float)
    return target.shape == current.shape and np.mean(np.abs(target - current)) / np.mean(np.abs(target)) < tol


def L_of(lower, thr_r2, max_r2):
    return R.L_csc(R.get_L(lower, thr_r2, max_r2), len(lower[0]) - 1)


def test_get_L_and_get_C_on_outer4():
    c = outer4()
    low = api.ldsplit_lower(sp.csc_matrix(c))
    L = L_of(low, 0, 1)
    dense = sp.csc_matrix((L[2], L[1], L[0]), shape=(4, 5)).toarray()
    want = np.zeros((4, 4))
    for a in range(3):
        for b in range(a + 1, 4):
            want[a, b] = np.sum(c[a, b:4] ** 2)
    assert np.allclose(dense[:, :4], want, rtol=1.5e-8) and not dense[:, 4].any()

    C1, b = R.get_C(L, 4, 1, 4, 5, INF, np.zeros(4))
    assert np.array_equal(b[:, 0], [4] * 4) and np.array_equal(C1[:, 0], [0] * 4)
    assert np.array_equal(b[:, 1], [1, 2, 3, NA]) and np.allclose(C1[:, 1], [0.5, 0.61, 0.49, INF], rtol=1.5e-8)
    assert np.array_equal(b[:, 2], [1, 2, NA, NA]) and np.allclose(C1[:, 2], [1.11, 1.1, INF, INF], rtol=1e-6)
    assert np.array_equal(b[:, 3], [1, NA, NA, NA]) and np.allclose(C1[:, 3], [1.6, INF, INF, INF], rtol=1.5e-8)
    assert np.array_equal(b[:, 4], [NA] * 4) and np.array_equal(C1[:, 4], [INF] * 4)

    C1, b = R.get_C(L, 4, 2, 2, 3, INF, np.ones(4))
    assert np.array_equal(b[:, 0], [NA, NA, 4, NA]) and np.array_equal(C1[:, 0], [INF, INF, 0, INF])
    assert np.array_equal(b[:, 1], [2, NA, NA, NA]) and np.allclose(C1[:, 1], [1.02, INF, INF, INF], rtol=1e-6)
    assert np.array_equal(b[:, 2], [NA] * 4) and np.array_equal(C1[:, 2], [INF] * 4)

    C1, b = R.get_C(L, 4, 1, 3, 3, INF, np.linspace(0, 1, 4))
    assert np.array_equal(b[:, 0], [NA, 4, 4, 4]) and np.array_equal(C1[:, 0], [INF, 0, 0, 0])
    assert np.array_equal(b[:, 1], [1, 2, 3, NA]) and np.allclose(C1[:, 1], [0.5, 0.61, 0.49, INF], rtol=1.5e-8)
    assert np.array_equal(b[:, 2], [1, 2, NA, NA]) and np.allclose(C1[:, 2], [1.11, 1.10, INF, INF], rtol=1e-6)

    pos = np.arange(1, 5) * 2.0
    assert R.snp_ldsplit(low, 0, 1, 3, max_K=3, max_r2=1, max_cost=INF, pos_scaled=pos) is None
    assert R.snp_ldsplit(low, 0, 1, 3, max_K=4, max_r2=1, max_cost=INF, pos_scaled=pos)["n_block"].size == 1
    C1, b = R.get_C(L, 4, 1, 3, 4, INF, pos)
    err = c[2, 3] ** 2
    assert np.array_equal(b[:, 0], [NA, NA, NA, 4]) and np.array_equal(C1[:, 0], [INF, INF, INF, 0])
    assert np.array_equal(b[:, 1], [NA, NA, 3, NA]) and np.allclose(C1[:, 1], [INF, INF, err, INF], rtol=1.5e-8)
    err += np.sum(c[1, 2:4] ** 2)
    assert np.array_equal(b[:, 2], [NA, 2, NA, NA]) and np.allclose(C1[:, 2], [INF, err, INF, INF], rtol=1e-6)
    err += np.sum(c[0, 1:4] ** 2)
    assert np.array_equal(b[:, 3], [1, NA, NA, NA]) and np.allclose(C1[:, 3], [err, INF, INF, INF], rtol=1e-6)


def test_last_snp_block_never_wins_a_later_layer():
    """max_size == m: at col = m - 1 the reference reads C1(m, k - 1), i.e. C1(0, k), still +Inf; a block ending at the
    last SNP is never chosen for k >= 1 (it is only layer 0's)."""
    low = api.ldsplit_lower(sp.csc_matrix(outer4()))
    C1, b = R.get_C(L_of(low, 0, 1), 4, 1, 4, 4, INF, np.zeros(4))
    assert not np.any(b[:, 1:] == 4)


def test_perc_kept_is_exact():
    low = api.ldsplit_lower(sp.csc_matrix(outer4()))
    t = R.snp_ldsplit(low, 0, 1, 2, 4, max_r2=1, max_cost=INF)
    assert np.array_equal(t["n_block"], [2, 3, 4])
    assert np.array_equal(t["perc_kept"], np.array([8, 6, 4]) / 16)


def block_num(sizes):
    return np.repeat(np.arange(len(sizes)), sizes)


def brute_cost(A, nums, thr_r2):
    """tests/testthat/test-4-split-LD.R:82-88 (compute_cost)"""
    T = sp.tril(A).tocoo()
    r2 = T.data[nums[T.row] != nums[T.col]] ** 2
    return np.sum(r2[r2 >= thr_r2])


def max_out(A, nums):
    T = sp.tril(A).tocoo()
    return np.max(T.data[nums[T.row] != nums[T.col]] ** 2)


@pytest.fixture(scope="module")
def spm():
    A, before, nb = spmat()
    A = A + sp.triu(A, 1).T  # the dsCMatrix as the full symmetric matrix
    return A.tocsc(), api.ldsplit_lower(A.tocsc()), before, nb


def test_spmat_consistent(spm):
    A, low, before, nb = spm
    res1 = R.snp_ldsplit(low, 0.02, 10, 30, max_K=50, max_r2=1, max_cost=INF)
    assert np.array_equal(res1["n_block"], np.arange(14, 41)) and np.array_equal(nb, res1["n_block"])
    costs = [brute_cost(A, block_num(s), 0.02) for s in res1["all_size"]]
    assert r_equal(costs, res1["cost"])
    assert r_equal(before, res1["cost"])

    res2 = R.snp_ldsplit(low, 0.1, 20, 40, max_K=50, max_r2=1, max_cost=INF)
    assert np.array_equal(res2["n_block"], np.arange(11, 21))
    res3 = R.snp_ldsplit(low, 0.05, 20, 40, max_K=15, max_r2=1, max_cost=INF)
    assert np.array_equal(res3["n_block"], np.arange(11, 16))

    mc = 0.5 * (res1["cost"].min() + res1["cost"].max())
    res4 = R.snp_ldsplit(low, 0.02, 10, 30, max_K=50, max_r2=1, max_cost=mc)
    assert np.all(res4["cost"] <= mc)
    assert np.all(res1["cost"][~np.isin(res1["n_block"], res4["n_block"])] > mc)

    res5 = R.snp_ldsplit(low, 0.02, 10, 50, max_K=100, max_r2=0.25, max_cost=INF)
    assert all(max_out(A, block_num(s)) <= 0.25 for s in res5["all_size"])


def rows_of(t, drop_max_size=True):
    if t is None:
        return []
    return [tuple([] if drop_max_size else [int(t["max_size"][r])]) + (int(t["n_block"][r]), t["cost"][r], t["cost2"][r],
            t["perc_kept"][r], tuple(t["all_last"][r])) for r in range(t["n_block"].size)]


def test_multiple_max_size_is_the_unique_union(spm):
    A, low, _, _ = spm
    res6 = R.snp_ldsplit(low, 0.02, 10, 30, max_K=50, max_r2=0.6, max_cost=INF)
    res7 = R.snp_ldsplit(low, 0.02, 10, 40, max_K=50, max_r2=0.6, max_cost=INF)
    res67 = R.snp_ldsplit(low, 0.02, 10, [40, 30], max_K=50, max_r2=0.6, max_cost=INF)
    union = []
    for r in rows_of(res6) + rows_of(res7):
        if r not in union:
            union.append(r)
    assert rows_of(res67) == union


def all_splits(m, min_size, max_size):
    for cuts in itertools.product((0, 1), repeat=m - 1):
        last = [j + 1 for j in range(m - 1) if cuts[j]] + [m]
        size = np.diff([0] + last)
        if np.all((size >= min_size) & (size <= max_size)):
            yield last, size


@pytest.mark.parametrize("seed", range(6))
def test_exhaustive_small(seed):
    """Dyadic r^2 (x = k / 8) make every sum exact in float and double: per K, the oracle's split is the (cost,
    cost2)-optimal one, ties going to the lexicographically largest all_last."""
    rng = np.random.default_rng(seed)
    m = int(rng.integers(6, 13))
    c = np.eye(m)
    for a in range(m):
        for b in range(a + 1, min(m, a + 5)):
            c[a, b] = c[b, a] = rng.choice([0, 1, 2, 3, 4]) / 8
    A = sp.csc_matrix(c)
    A.eliminate_zeros()
    low = api.ldsplit_lower(A)
    thr_r2, max_r2 = (0, 1) if seed % 2 == 0 else (2 / 64, 9 / 64)
    min_size, max_size = (1, m) if seed < 3 else (2, 4)
    t = R.snp_ldsplit(low, thr_r2, min_size, max_size, max_K=m, max_r2=max_r2, max_cost=INF)
    T = sp.tril(A, -1).tocoo()
    r2 = T.data ** 2
    best = {}
    for last, size in all_splits(m, min_size, max_size):
        nums = block_num(size)
        out = r2[nums[T.row] != nums[T.col]]
        cost = INF if np.any(out[out >= thr_r2] > max_r2) else float(np.sum(out[out >= thr_r2]))
        key = (cost, float(np.sum(size.astype(float) ** 2)), [-v for v in last])
        K = len(last)
        if K not in best or key < best[K]:
            best[K] = key
    got = {} if t is None else {int(k): r for k, r in zip(t["n_block"], range(t["n_block"].size))}
    cap = 2 * float(np.sum(low[2] ** 2))
    for K, (cost, cost2, neg_last) in best.items():
        if cost == INF or cost > cap:
            assert K not in got
            continue
        r = got[K]
        assert t["cost"][r] == cost and t["cost2"][r] == cost2
        assert list(t["all_last"][r]) == [-v for v in neg_last]
    assert set(got) <= set(best)


def test_lower_triangle_from_each_form():
    A, _, _ = spmat()
    full = (A + sp.triu(A, 1).T).tocsc()
    a = api.ldsplit_lower(A, upper=True)
    b = api.ldsplit_lower(full)
    up = A.tocsc()
    c = api.ldsplit_lower((up.indptr, up.indices, up.data))
    for u, v in ((a, b), (a, c)):
        assert all(np.array_equal(s, t) for s, t in zip(u, v))
    p, i, x = a
    assert np.all(np.diff(p) > 0) and np.all(i[p[:-1]] == np.arange(p.size - 1))
    # an unsorted tuple with a repeated entry is put in canonical order (summed)
    t = (np.array([0, 1, 3]), np.array([0, 1, 0]), np.array([1.0, 1.0, 0.25]))
    t2 = (np.array([0, 1, 4]), np.array([0, 1, 0, 0]), np.array([1.0, 1.0, 0.125, 0.125]))
    for u, v in zip(api.ldsplit_lower(t), api.ldsplit_lower(t2)):
        assert np.array_equal(u, v)


def test_argument_checks():
    low4 = sp.csc_matrix(outer4())
    for kw, msg in (({"min_size": 0, "max_size": 2}, "min_size"), ({"min_size": 1, "max_size": 5}, "max_size <= m"),
                    ({"min_size": 3, "max_size": 2}, "at least 'min_size'"), ({"min_size": 1, "max_size": 2, "max_K": 0}, "max_K"),
                    ({"min_size": 1, "max_size": 2, "pos_scaled": np.zeros(3)}, "dimensions")):
        with pytest.raises(ValueError, match=msg):
            api.snp_ldsplit(low4, 0, **kw)
    z = outer4()
    z[2, 2] = 0
    with pytest.raises(ValueError, match="diag"):
        api.snp_ldsplit(sp.csc_matrix(z), 0, 1, 2)
    with pytest.raises(TypeError):
        api.snp_ldsplit(np.eye(3), 0, 1, 2)


def test_kernels_have_no_fma(tmp_path):
    ptx = tmp_path / "ldsplit.ptx"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-ptx", "-arch=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-I",
                           os.path.join(ROOT, "bigsnpr_b200", "csrc"),
                           os.path.join(ROOT, "bigsnpr_b200", "csrc", "bsg_ldsplit.cu"), "-o", str(ptx)])
    text = ptx.read_text()
    bodies = text.split(".entry ")
    names = ("k_build_E", "k_suffix", "k_layer", "k_paths")
    seen = set()
    for body in bodies[1:]:
        for n in names:
            if n in body.split("(")[0]:
                seen.add(n)
                assert "fma.rn.f64" not in body and "fma.rn.f32" not in body, n
    assert seen == set(names)
