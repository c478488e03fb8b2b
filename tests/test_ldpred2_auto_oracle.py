"""CPU checks of LDpred2-auto's shared sampler header (bigsnpr_b200/csrc/bsg_ldpred2_auto.cuh) and of its CPU oracle
(tests/ldpred2_auto_oracle.c) against independent facts: Python-integer MRG32k3a, SciPy / NumPy math, SciPy's
L-BFGS-B, a pure-Python restatement of the chain loop and the sampler's statistical behaviour."""
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.special
import scipy.stats

from bigsnpr_b200 import api
from tests import ldpred2_auto_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M1, M2 = 4294967087, 4294944443
S0 = np.array([12345, 67890, 13579, 24680, 11223, 44556], dtype=np.uint32)


def py_mrg(state, n):
    """R's L'Ecuyer-CMRG unif_rand in Python integers."""
    s = [int(v) for v in state]
    out = []
    for _ in range(n):
        p1 = (1403580 * s[1] - 810728 * s[0]) % M1
        s = [s[1], s[2], p1] + s[3:]
        p2 = (527612 * s[5] - 1370589 * s[3]) % M2
        s = s[:3] + [s[4], s[5], p2]
        out.append((p1 - p2 if p1 > p2 else p1 - p2 + M1) * 2.328306549295727688e-10)
    return np.array(out), np.array(s, dtype=np.uint32)


def ulps(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    ia, ib = a.view(np.int64), b.view(np.int64)
    ia = np.where(ia < 0, np.int64(-2 ** 63) - ia, ia)
    ib = np.where(ib < 0, np.int64(-2 ** 63) - ib, ib)
    return np.abs(ia - ib)


# ---- MRG32k3a -------------------------------------------------------------------------------------------------------------

def test_mrg_matches_python_integers():
    got, s = R.unif(S0, 100_000)
    want, ws = py_mrg(S0, 100_000)
    assert got.tobytes() == want.tobytes() and np.array_equal(s, ws)
    assert got.min() > 0 and got.max() < 1


@pytest.mark.parametrize("k", [1, 5, 31, 32, 33, 255, 1000, 65537, 1_000_000])
def test_skip_ahead_equals_single_steps(k):
    _, s = R.unif(S0, k)
    assert np.array_equal(R.skip(S0, k), s)


def test_jump127_matches_big_int_matrix_powers():
    def matpow(A, e, m):  # square-and-multiply in Python integers, row-major lists
        Rm = [[int(i == j) for j in range(3)] for i in range(3)]
        mul = lambda X, Y: [[sum(X[i][k] * Y[k][j] for k in range(3)) % m for j in range(3)] for i in range(3)]
        while e:
            if e & 1:
                Rm = mul(Rm, A)
            A, e = mul(A, A), e >> 1
        return Rm

    A1 = [[0, 1, 0], [0, 0, 1], [-810728 % M1, 1403580, 0]]
    A2 = [[0, 1, 0], [0, 0, 1], [-1370589 % M2, 0, 527612]]
    J1, J2 = matpow(A1, 2 ** 127, M1), matpow(A2, 2 ** 127, M2)
    s = [int(v) for v in S0]
    want = [sum(J1[i][k] * s[k] for k in range(3)) % M1 for i in range(3)]
    want += [sum(J2[i][k] * s[3 + k] for k in range(3)) % M2 for i in range(3)]
    assert R.jump127(S0).tolist() == want
    assert api.mrg32k3a_next_stream(S0).tolist() == want
    # the published first row of A1^(2^127) (RngStreams' A1p127)
    assert J1[0] == [2427906178, 3580155704, 949770784]


def test_uniforms_inside_open_interval():
    u, _ = R.unif(api.mrg32k3a_seed(7), 1_000_000)
    assert u.min() > 0 and u.max() < 1
    assert abs(u.mean() - 0.5) < 2e-3


def test_seed_map():
    s = api.mrg32k3a_seed(42)
    assert s.dtype == np.uint32 and np.all(s[:3] < M1) and np.all(s[3:] < M2)
    assert not np.array_equal(s, api.mrg32k3a_seed(43))


# ---- math -----------------------------------------------------------------------------------------------------------------

def test_qnorm_against_ndtri():
    rng = np.random.default_rng(1)
    p = np.concatenate([10.0 ** -rng.uniform(0, 300, 200_000), rng.uniform(0, 1, 200_000),
                        1 - 10.0 ** -rng.uniform(1, 15.9, 50_000), [1e-300, 0.5, 1 - 2.0 ** -53, 0.075, 0.925]])
    p = p[(p > 0) & (p < 1)]
    got, want = R.qnorm(p), scipy.special.ndtri(p)
    near0 = np.abs(want) < 1e-3
    assert ulps(got[~near0], want[~near0]).max() <= 8
    assert np.max(np.abs(got[near0] - want[near0])) <= 1e-18 + 8 * np.spacing(np.abs(want[near0])).max()
    assert R.qnorm(np.array([0.0, 1.0]))[0] == -np.inf and R.qnorm(np.array([1.0]))[0] == np.inf


def test_exp_log_against_numpy():
    rng = np.random.default_rng(2)
    x = np.concatenate([rng.uniform(-745, 709.7, 400_000), rng.normal(0, 3, 400_000), rng.uniform(-1e-8, 1e-8, 200_000)])
    assert ulps(R.exp(x), np.exp(x)).max() <= 2
    y = np.concatenate([10.0 ** rng.uniform(-307, 308, 500_000), rng.uniform(0.5, 2, 400_000),
                        1 + rng.uniform(-1e-6, 1e-6, 100_000), 5e-324 * rng.integers(1, 2 ** 40, 1000)])
    assert ulps(R.log(y), np.log(y)).max() <= 2
    with np.errstate(all="ignore"):
        sx = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 709.8, -745.2, 1e-300])
        ex = R.exp(sx)
        assert ex[0] == 1 and ex[1] == 1 and ex[2] == np.inf and ex[3] == 0 and np.isnan(ex[4])
        assert ex[5] == np.inf and ex[6] == 0 and ex[7] == 1
        sy = np.array([0.0, -0.0, np.inf, -1.0, np.nan, 1.0, 5e-324, -np.inf])
        ly = R.log(sy)
        assert ly[0] == -np.inf and ly[1] == -np.inf and ly[2] == np.inf and np.isnan(ly[3]) and np.isnan(ly[4])
        assert ly[5] == 0 and ly[6] == np.log(5e-324) and np.isnan(ly[7])


@pytest.mark.parametrize("a,b", [(1.0, 1.0), (1.0, 200.0), (200.0, 1.0), (1.0, 1.5), (300.0, 2.0), (2.0, 300.0),
                                 (5.0, 5.0), (1.0 + 3 / 2.5, 1.0 + 9997 / 2.5), (0.5, 3.0), (3.0, 0.4)])
def test_rbeta_ks(a, b):
    x, _ = R.rbeta(a, b, api.mrg32k3a_seed(int(a * 1000 + b)), 20_000)
    assert np.all((x >= 0) & (x <= 1))
    assert scipy.stats.kstest(x, scipy.stats.beta(a, b).cdf).pvalue > 1e-3


def test_rnorm_moments_and_sigma_zero():
    z, s = R.rnorm(1.5, 2.0, S0, 200_000)
    assert abs(z.mean() - 1.5) < 0.02 and abs(z.std() - 2.0) < 0.02
    assert scipy.stats.kstest((z - 1.5) / 2, "norm").pvalue > 1e-3
    v, s2 = R.rnorm(0.3, 0.0, S0, 3)  # no draw
    assert np.all(v == 0.3) and np.array_equal(s2, S0)


def test_oracle_is_uncontracted():
    out = subprocess.run(["objdump", "-d", R.object_file()], capture_output=True, text=True).stdout
    assert "vfmadd" not in out
    assert "-ffp-contract=off" in R.FLAGS


def test_kernel_ptx_has_no_fma(tmp_path):
    ptx = tmp_path / "sparse.ptx"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-ptx", "-arch=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-I",
                           os.path.join(ROOT, "bigsnpr_b200", "csrc"),
                           os.path.join(ROOT, "bigsnpr_b200", "csrc", "bsg_sparse.cu"), "-o", str(ptx)])
    text = ptx.read_text()
    bodies = re.findall(r"\.entry \w*?k_ldpred2_auto\w*\((.*?)\n}\n", text, re.S)
    assert len(bodies) == 1
    assert "fma.rn.f64" not in bodies[0] and "div.rn.f64" in bodies[0] and "sqrt.rn.f64" in bodies[0]


# ---- MLE ------------------------------------------------------------------------------------------------------------------

def objective(a, b, t, s2):
    """src/optim-MLE-alpha.h:38-48 in NumPy"""
    return t * a.sum() + a.size * np.log(s2) + np.sum(b * np.exp(-t * a)) / s2


def test_profile_minimiser_beats_lbfgsb():
    from scipy.optimize import minimize

    rng = np.random.default_rng(4)
    for trial in range(40):
        nb = int(rng.integers(1, 400))
        a = 2 * np.log(rng.uniform(0.02, 0.7, nb))          # log_var = 2 log sd
        b = (rng.normal(size=nb) * 10 ** rng.uniform(-3, -1)) ** 2
        if trial % 4 == 0:  # a bootstrap resample, with repeats
            idx = rng.integers(0, nb, nb)
            a, b = a[idx], b[idx]
        s2 = float(np.mean(b)) * rng.uniform(0.3, 3)
        lo, hi = -0.5, 1.5
        par = R.mle_fit(a, b, lo, hi, [0.7, s2])
        assert lo <= par[0] <= hi and s2 / 2 <= par[1] <= 2 * s2
        res = minimize(lambda v: objective(a, b, v[0], v[1]), [min(max(0.0, lo), hi), s2], method="L-BFGS-B",
                       bounds=[(lo, hi), (s2 / 2, 2 * s2)])
        f_ours, f_lb = objective(a, b, par[0], par[1]), objective(a, b, *res.x)
        assert f_ours <= f_lb + 1e-12 * max(1.0, abs(f_lb)), (trial, f_ours, f_lb)
        f_h, s2h = R.mle_objective(a, b, par[0], s2 / 2, 2 * s2)
        assert s2h == par[1] and np.isclose(f_h, f_ours, rtol=1e-12, atol=1e-9)


def test_mle_fixed_alpha_and_empty_set():
    a, b = np.log(np.array([0.1, 0.2, 0.3])), np.array([1e-4, 2e-4, 5e-5])
    par = R.mle_fit(a, b, 0.0, 0.0, [0.5, 1e-4])
    assert par[0] == 0.0
    assert R.mle_fit(np.empty(0), np.empty(0), -0.5, 1.5, [0.25, 3e-5]).tolist() == [0.25, 3e-5]


# ---- chains ---------------------------------------------------------------------------------------------------------------

def banded_ld(m, rho=0.8, width=30, seed=0):
    """An AR(1) correlation matrix cut to a band (positive definite enough for the sampler), as CSC."""
    idx = np.arange(m)
    rows, cols, vals = [], [], []
    for d in range(-width, width + 1):
        j = idx[(idx + d >= 0) & (idx + d < m)]
        rows.append(j + d), cols.append(j), vals.append(np.full(j.size, rho ** abs(d)))
    return sp.csc_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(m, m))


def sim_sumstats(Rm, h2=0.4, p=0.02, N=20_000, seed=1):
    rng = np.random.default_rng(seed)
    m = Rm.shape[0]
    beta = np.zeros(m)
    c = rng.choice(m, max(1, int(p * m)), replace=False)
    beta[c] = rng.normal(size=c.size)
    beta *= np.sqrt(h2 / (beta @ (Rm @ beta)))
    L = np.linalg.cholesky(Rm.toarray() + 1e-10 * np.eye(m))
    bh = Rm @ beta + (L @ rng.normal(size=m)) / np.sqrt(N)
    n = np.round(N * rng.uniform(0.8, 1.0, m))
    sd = rng.uniform(0.05, 0.7, m)
    return bh, n, 2 * np.log(sd)


def run(storage, bh, n, lv, ind=None, p_init=(0.1,), seeds=None, **kw):
    m = bh.size
    ind = np.arange(m) if ind is None else ind
    rng = [api.mrg32k3a_seed(100 + i) for i in range(len(p_init))] if seeds is None else seeds
    kw.setdefault("h2_init", 0.3)
    kw.setdefault("mean_ld", 3.0)
    return R.ldpred2_auto(storage, bh, n, lv, ind, np.array(p_init), rng=np.array(rng), **kw)


def same(a, b):
    for k in ("beta_est", "postp_est", "corr_est", "path_p_est", "path_h2_est", "path_alpha_est", "sample_beta"):
        x, y = a[k], b[k]
        if x is None or y is None:
            assert x is None and y is None
            continue
        assert x.shape == y.shape, k
        nx, ny = np.isnan(x), np.isnan(y)
        assert np.array_equal(nx, ny) and x[~nx].tobytes() == y[~ny].tobytes(), k


def py_chain(storage, bh, n, lv, ind, p_init, h2_init, state, burn_in, num_iter, report_step, no_jump_sign, shrink,
             use_mle, p_bounds, alpha_bounds, mean_ld):
    """src/ldpred2-auto.cpp:56-202 restated in Python, the draws and math through the oracle's exports of the header."""
    nn, p_, data, first_i = storage
    cols = []
    for j in range(nn):
        lo, up = int(p_[j]), int(p_[j + 1])
        if first_i is None:
            cols.append((data[2 * lo:2 * up:2].astype(int), data[2 * lo + 1:2 * up:2]))
        else:
            cols.append((first_i[j] + np.arange(up - lo), data[lo:up]))
    m = bh.size
    s = np.array(state, dtype=np.uint32)
    dot, cb = [0.0] * nn, [0.0] * m
    avg_b, avg_p, avg_bh = [0.0] * m, [0.0] * m, [0.0] * m
    T = burn_in + num_iter
    na = np.nan
    path_p, path_h2, path_a = [na] * T, [na] * T, [na] * T
    nrep = num_iter // report_step
    sample = np.zeros((m, nrep))
    cur_h2 = 0.0
    h2 = max(h2_init, 1e-3)
    p = min(max(p_bounds[0], p_init), p_bounds[1])
    par = [0.0, h2 / (m * p)]
    gap0 = 0.0
    for v in bh:
        gap0 = gap0 + v * v
    gap0 = 2 * gap0
    rep, next_k = 0, burn_in + report_step - 1
    diverged = False
    for k in range(T):
        inv_odd_p = (1 - p) / p
        gap, causal = 0.0, []
        for j in range(m):
            j2 = int(ind[j])
            postp, C3, C4, dps = R.coord(bh[j], dot[j2], cb[j], n[j], lv[j], shrink, use_mle, par[0], par[1], inv_odd_p)
            prev = cb[j]
            if k >= burn_in:
                avg_p[j] += postp
                avg_b[j] += C3 * postp
                avg_bh[j] += dps
            diff = -prev
            u, s = R.unif(s, 1)
            if postp > u[0]:
                z, s = R.rnorm(C3, np.sqrt(C4), s)
                samp = float(z[0])
                if no_jump_sign and samp * prev < 0:
                    cb[j] = 0.0
                else:
                    cb[j] = samp
                    diff += samp
                    causal.append(j)
                    gap += samp * samp
            else:
                cb[j] = 0.0
            if diff != 0:
                cur_h2 += diff * (2 * dps + diff)
                rows, vals = cols[j2]
                for r, v in zip(rows, vals):
                    dot[r] += v * diff
        if gap > gap0:
            diverged = True
            break
        p, s = R.draw_p(len(causal), m, mean_ld, p_bounds[0], p_bounds[1], s)
        h2 = 1e-3 if cur_h2 < 1e-3 else cur_h2
        if use_mle:
            nb = len(causal)
            u, s = R.unif(s, nb)
            pick = [causal[int(nb * v)] for v in u]
            a = np.array([lv[i] for i in pick])
            b = np.array([cb[i] * cb[i] for i in pick])
            par = list(R.mle_fit(a, b, alpha_bounds[0], alpha_bounds[1], par))
        else:
            par[1] = h2 / (m * p)
        path_p[k], path_h2[k] = p, h2
        if use_mle:
            path_a[k] = par[0] - 1
        if k == next_k:
            for i in causal:
                sample[i, rep] = cb[i]
            rep += 1
            next_k += report_step
    f = (lambda v: np.nan) if diverged else (lambda v: v / num_iter)
    return {"beta_est": np.array([f(v) for v in avg_b]), "postp_est": np.array([f(v) for v in avg_p]),
            "corr_est": np.array([f(v) for v in avg_bh]), "path_p_est": np.array(path_p),
            "path_h2_est": np.array(path_h2), "path_alpha_est": np.array(path_a), "sample_beta": sample}


@pytest.mark.parametrize("case", ["default", "no_mle", "no_jump", "shrink", "compact_subset"])
def test_oracle_equals_python_restatement(case):
    Rm = banded_ld(40, 0.7, 5)
    bh, n, lv = sim_sumstats(Rm, h2=0.5, p=0.2, N=5000, seed=3)
    kw = dict(burn_in=4, num_iter=6, report_step=2, no_jump_sign=False, shrink_corr=1.0, use_mle=True,
              p_bounds=(1e-5, 1.0), alpha_bounds=(-0.5, 1.5), mean_ld=2.5, h2_init=0.2)
    compact, ind = False, np.arange(40)
    if case == "no_mle":
        kw["use_mle"] = False
    elif case == "no_jump":
        kw["no_jump_sign"] = True
    elif case == "shrink":
        kw["shrink_corr"] = 0.95
    elif case == "compact_subset":
        compact, ind = True, np.array([5, 3, 3, 20, 39, 0, 12, 11, 10, 30] * 2)
        bh, n, lv = bh[ind], n[ind], lv[ind]
    st = api.sfbm_storage(Rm, compact=compact)
    state = api.mrg32k3a_seed(9)
    got = R.ldpred2_auto(st, bh, n, lv, ind, np.array([0.3]), rng=state[None], **kw)
    want = py_chain(st, bh, n, lv, ind, 0.3, kw["h2_init"], state, kw["burn_in"], kw["num_iter"], kw["report_step"],
                    kw["no_jump_sign"], kw["shrink_corr"], kw["use_mle"], kw["p_bounds"], kw["alpha_bounds"],
                    kw["mean_ld"])
    for k in want:
        x, y = got[k][..., 0] if got[k].ndim == 3 else got[k][:, 0], want[k]
        nx = np.isnan(y)
        assert np.array_equal(np.isnan(x), nx) and x[~nx].tobytes() == y[~nx].tobytes(), k


@pytest.fixture(scope="module")
def medium():
    Rm = banded_ld(600, 0.8, 40)
    bh, n, lv = sim_sumstats(Rm, h2=0.3, p=0.05, N=20_000, seed=5)
    return Rm, bh, n, lv


def test_threads_batch_and_chain_independence(medium):
    Rm, bh, n, lv = medium
    st = api.sfbm_storage(Rm)
    seeds = [api.mrg32k3a_seed(i) for i in range(6)]
    kw = dict(burn_in=20, num_iter=20, report_step=5)
    a = run(st, bh, n, lv, p_init=(0.2, 0.1, 0.05, 0.01, 0.001, 0.1), seeds=seeds, nthreads=1, **kw)
    b = run(st, bh, n, lv, p_init=(0.2, 0.1, 0.05, 0.01, 0.001, 0.1), seeds=seeds, nthreads=4, **kw)
    same(a, b)
    one = run(st, bh, n, lv, p_init=(0.01,), seeds=[seeds[3]], **kw)
    sub = {k: (v[..., 3:4] if v.ndim == 3 else v[:, 3:4]) for k, v in a.items()}
    same(one, sub)
    assert not np.array_equal(a["beta_est"][:, 1], a["beta_est"][:, 5])  # same p_init, other stream


def test_ind_corr_equals_subset_matrix(medium):
    """test-8:289-298: running on a subset through ind_corr == running on the subset matrix."""
    Rm, bh, n, lv = medium
    ind = np.sort(np.random.default_rng(1).choice(600, 250, replace=False))
    kw = dict(burn_in=10, num_iter=10, report_step=3)
    a = run(api.sfbm_storage(Rm), bh[ind], n[ind], lv[ind], ind=ind, **kw)
    b = run(api.sfbm_storage(sp.csc_matrix(Rm[ind][:, ind])), bh[ind], n[ind], lv[ind], **kw)
    same(a, b)


def test_divergence_gives_na():
    """A matrix that is not a correlation matrix (off-diagonal 1.5) makes the sampler blow up: NA averages, NA paths
    after the diverging sweep."""
    m = 60
    A = np.full((m, m), 0.0)
    for d in (-1, 1):
        A += np.diag(np.full(m - 1, -0.9), d)
    A += np.eye(m)
    Rm = sp.csc_matrix(A)
    rng = np.random.default_rng(0)
    bh, n, lv = rng.normal(0, 0.05, m), np.full(m, 1e5), np.full(m, -2.0)
    r = run(api.sfbm_storage(Rm), bh, n, lv, p_init=(0.9,), burn_in=30, num_iter=10, p_bounds=(0.9, 0.9), use_mle=False)
    assert np.all(np.isnan(r["beta_est"])) and np.all(np.isnan(r["postp_est"]))
    assert r["beta_est"].view(np.uint64)[0, 0] == 0x7FF00000000007A2
    k = np.flatnonzero(np.isnan(r["path_p_est"][:, 0]))
    assert k.size > 0 and np.all(np.isnan(r["path_p_est"][k[0]:, 0]))


# ---- statistics -----------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def big():
    Rm = banded_ld(5000, 0.9, 60)
    bh, n, lv = sim_sumstats(Rm, h2=0.3, p=0.01, N=50_000, seed=8)
    return Rm, bh, n, lv


def test_statistics_of_the_chain(big):
    Rm, bh, n, lv = big
    st = api.sfbm_storage(Rm)
    r = run(st, bh, n, lv, p_init=(0.01, 0.05), burn_in=150, num_iter=100, report_step=10, h2_init=0.2)
    for c in range(2):
        path_p, path_h2 = r["path_p_est"][:, c], r["path_h2_est"][:, c]
        p_est, h2_est = path_p[-100:].mean(), path_h2[-100:].mean()
        assert abs(r["postp_est"][:, c].mean() - p_est) < 0.01
        assert 0.15 < h2_est < 0.45
        S = r["sample_beta"][:, :, c]
        assert S.shape == (5000, 10)
        for i in range(10):  # test-8:105-106: the h2 of each sampled beta is the path's h2 at that sweep
            b = S[:, i]
            assert np.isclose(b @ (Rm @ b), path_h2[150 + 10 * i + 9], rtol=1e-6)
    # fixed alpha: path_alpha_est == -1 everywhere (test-8:112)
    f = run(st, bh, n, lv, burn_in=5, num_iter=5, alpha_bounds=(0.0, 0.0))
    assert np.all(f["path_alpha_est"] == -1)


def test_no_jump_sign_from_p_one(big):
    Rm, bh, n, lv = big
    r = run(api.sfbm_storage(Rm), bh, n, lv, p_init=(1.0,), burn_in=100, num_iter=50, no_jump_sign=True, h2_init=0.2)
    assert r["path_p_est"][-50:, 0].mean() < 0.1


def test_identity_ld_recovers_h2_and_p():
    m, N, h2, p = 20_000, 100_000, 0.4, 0.02
    rng = np.random.default_rng(12)
    beta = np.zeros(m)
    c = rng.choice(m, int(p * m), replace=False)
    beta[c] = rng.normal(size=c.size)
    beta *= np.sqrt(h2 / (beta @ beta))
    bh = beta + rng.normal(size=m) / np.sqrt(N)
    Rm = sp.identity(m, format="csc")
    r = run(api.sfbm_storage(Rm), bh, np.full(m, float(N)), np.zeros(m), p_init=(0.1,), burn_in=200, num_iter=100,
            h2_init=0.1, mean_ld=1.0, alpha_bounds=(0.0, 0.0))
    assert abs(r["path_h2_est"][-100:, 0].mean() - h2) < 0.05
    assert 0.5 * p < r["path_p_est"][-100:, 0].mean() < 2 * p
