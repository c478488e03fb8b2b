"""LDpred2-grid's CPU oracle (tests/ldpred2_grid_oracle.c) against a pure-Python restatement of src/ldpred2.cpp:9-69 and
src/ldpred2-sampling.cpp:9-59, its draw count, exact and statistical properties, launch independence, and
snp_ldpred2_grid's host logic (checks, order, seeding, scaling) with the device call replaced by the oracle."""
import math
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from bigsnpr_b200 import api
from tests import ldpred2_auto_ref as AR
from tests import ldpred2_grid_ref as G
from tests.test_ldpred2_auto_oracle import ROOT, banded_ld, sim_sumstats

NA_BITS = 0x7FF00000000007A2


def same(x, y):
    nx, ny = np.isnan(x), np.isnan(y)
    return x.shape == y.shape and np.array_equal(nx, ny) and x[~nx].tobytes() == y[~ny].tobytes()


def py_gibbs(storage, bh, n, ind, h2, p, sparse, state, burn_in, num_iter, sampling=False):
    """src/ldpred2.cpp:9-69 (or src/ldpred2-sampling.cpp:9-59) in Python floats, exp and the draws through the oracle's
    exports of the header.  Returns (result, final state, uniforms drawn, normals drawn, zeroings of a non-zero beta)."""
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
    dot, cb, avg = [0.0] * nn, [0.0] * m, [0.0] * m
    sample = np.zeros((m, num_iter))
    h2_per_var, inv_odd_p = h2 / (m * p), (1 - p) / p
    gap0 = 0.0
    for v in bh:
        gap0 = gap0 + v * v
    gap0 = 2 * gap0
    nunif = nnorm = nzeroed = 0
    for k in range(-burn_in, num_iter):
        gap = 0.0
        for j in range(m):
            j2 = int(ind[j])
            res = (bh[j] + cb[j]) - dot[j2] if sampling else bh[j] - (dot[j2] - cb[j])
            C1 = h2_per_var * n[j]
            C2 = 1 / (1 + 1 / C1)
            C3 = C2 * res
            C4 = C2 / n[j]
            postp = 1 / (1 + inv_odd_p * math.sqrt(1 + C1) * float(AR.exp(np.array([-C3 * C3 / C4 / 2]))[0]))
            diff = -cb[j]
            if sparse and postp < p:
                nzeroed += cb[j] != 0
                cb[j] = 0.0
            else:
                u, s = AR.unif(s, 1)
                nunif += 1
                if postp > u[0]:
                    z, s = AR.rnorm(C3, math.sqrt(C4), s)
                    nnorm += 1
                    cb[j] = float(z[0])
                    diff += cb[j]
                    gap += cb[j] * cb[j]
                else:
                    cb[j] = 0.0
                if k >= 0:
                    avg[j] += C3 * postp
                    sample[j, k] = cb[j]
            if diff != 0:
                rows, vals = cols[j2]
                for r, v in zip(rows, vals):
                    dot[r] += v * diff
        if not sampling and gap > gap0:
            return np.full(m, np.nan), s, nunif, nnorm, nzeroed
    out = sample if sampling else np.array([v / num_iter for v in avg])
    return out, s, nunif, nnorm, nzeroed


def small(m=40, seed=3):
    Rm = banded_ld(m, 0.7, 5)
    bh, n, _ = sim_sumstats(Rm, h2=0.5, p=0.2, N=5000, seed=seed)
    return Rm, bh, n


@pytest.mark.parametrize("case", ["plain", "sparse", "p_one", "sparse_p_one", "sampling", "sampling_sparse",
                                  "compact_subset"])
def test_oracle_equals_python_restatement(case):
    Rm, bh, n = small()
    p, h2, sparse, sampling, compact, ind = 0.1, 0.4, False, False, False, np.arange(40)
    if "sparse" in case:
        sparse = True
    if "p_one" in case:
        p = 1.0
    if "sampling" in case:
        sampling = True
    if case == "compact_subset":
        compact, sparse, ind = True, True, np.array([5, 3, 3, 20, 39, 0, 12, 11, 10, 30] * 2)
        bh, n = bh[ind], n[ind]
    st = api.sfbm_storage(Rm, compact=compact)
    state = api.mrg32k3a_seed(9)
    burn_in, num_iter = 4, 6
    got = G.ldpred2_grid(st, bh, n, ind, [p], [h2], [sparse], state[None], burn_in, num_iter, sampling=sampling)
    want, s, nunif, nnorm, _ = py_gibbs(st, bh, n, ind, h2, p, sparse, state, burn_in, num_iter, sampling)
    x = got["sample_beta"] if sampling else got["beta_est"][:, 0]
    assert same(x, want)
    # draws: one uniform per coordinate not zeroed, two more per normal
    assert np.array_equal(got["rng_out"][0], s)
    assert np.array_equal(AR.skip(state, nunif + 2 * nnorm), s)
    if not sparse:
        assert nunif == (burn_in + num_iter) * ind.size


def test_sparse_zeroes_nonzero_coordinates():
    """A sparse point whose postp drops below p after a draw sets beta back to 0 without a uniform."""
    Rm, bh, n = small(60, seed=4)
    st = api.sfbm_storage(Rm)
    state = api.mrg32k3a_seed(2)
    found = False
    for p in (0.3, 0.5, 0.7):
        want, s, nunif, nnorm, nzeroed = py_gibbs(st, bh, n, np.arange(60), 0.5, p, True, state, 3, 5)
        got = G.ldpred2_grid(st, bh, n, np.arange(60), [p], [0.5], [True], state[None], 3, 5)
        assert same(got["beta_est"][:, 0], want) and np.array_equal(got["rng_out"][0], s)
        assert nunif < 8 * 60
        found |= nzeroed > 0
    assert found


def test_divergence_gives_na():
    m = 60
    A = np.eye(m) + np.diag(np.full(m - 1, -0.9), 1) + np.diag(np.full(m - 1, -0.9), -1)
    rng = np.random.default_rng(0)
    bh, n = rng.normal(0, 0.05, m), np.full(m, 1e5)
    st = api.sfbm_storage(sp.csc_matrix(A))
    state = api.mrg32k3a_seed(1)
    got = G.ldpred2_grid(st, bh, n, np.arange(m), [0.9, 0.9], [1.0, 1.0], [False, True], [state, state], 30, 10)
    assert np.all(got["beta_est"].view(np.uint64) == NA_BITS)
    want = py_gibbs(st, bh, n, np.arange(m), 1.0, 0.9, False, state, 30, 10)
    assert np.all(np.isnan(want[0])) and np.array_equal(got["rng_out"][0], want[1])


def test_draw_offset():
    rng = np.random.default_rng(5)
    for _ in range(200):
        d = int(rng.integers(0, 2 ** 32))
        lane = int(rng.integers(0, 32))
        assert G.offset(d, lane) == bin(d & ((1 << lane) - 1)).count("1")


def identity_case(m=300, N=20_000, seed=7):
    rng = np.random.default_rng(seed)
    beta = np.zeros(m)
    c = rng.choice(m, m // 10, replace=False)
    beta[c] = rng.normal(0, 0.03, c.size)
    bh = beta + rng.normal(size=m) / np.sqrt(N)
    n = np.full(m, float(N))
    return api.sfbm_storage(sp.identity(m, format="csc")), bh, n


def closed_form(bh, n, h2, p):
    m = bh.size
    C1 = h2 / (m * p) * n
    C2 = 1 / (1 + 1 / C1)
    C3, C4 = C2 * bh, C2 / n
    postp = 1 / (1 + (1 - p) / p * np.sqrt(1 + C1) * np.exp(-C3 * C3 / C4 / 2))
    return postp, C3, C4


@pytest.mark.parametrize("seed", [1, 2])
def test_identity_ld_is_closed_form(seed):
    """R = I: the residual is beta_hat at every sweep (up to the rounding of dotprods tracking beta), so each average
    is num_iter copies of C3 postp, whatever the draws; a sparse point gives 0 where postp < p."""
    st, bh, n = identity_case()
    m = bh.size
    h2, p = 0.3, 0.05
    postp, C3, _ = closed_form(bh, n, h2, p)
    num_iter = 40
    got = G.ldpred2_grid(st, bh, n, np.arange(m), [p, p], [h2, h2], [False, True],
                         [api.mrg32k3a_seed(seed), api.mrg32k3a_seed(seed + 10)], 10, num_iter)["beta_est"]
    want = C3 * postp
    assert np.allclose(got[:, 0], want, rtol=1e-11, atol=1e-300)
    clear = np.abs(postp - p) > 1e-6
    assert np.all(got[clear & (postp < p), 1] == 0)
    keep = clear & (postp >= p)
    assert np.allclose(got[keep, 1], want[keep], rtol=1e-11, atol=1e-300)


def test_identity_sampling_statistics():
    st, bh, n = identity_case(m=60, seed=3)
    m = bh.size
    h2, p, num_iter = 0.3, 0.1, 3000
    postp, C3, C4 = closed_form(bh, n, h2, p)
    S = G.ldpred2_grid(st, bh, n, np.arange(m), [p], [h2], [False], api.mrg32k3a_seed(4)[None], 10, num_iter,
                       sampling=True)["sample_beta"]
    frac = (S != 0).mean(1)
    assert np.all(np.abs(frac - postp) < 5 * np.sqrt(postp * (1 - postp) / num_iter) + 2 / num_iter)
    mean, var = postp * C3, postp * (C4 + C3 ** 2) - (postp * C3) ** 2
    assert np.all(np.abs(S.mean(1) - mean) < 5 * np.sqrt(var / num_iter) + 1e-12)


def test_sampling_mean_follows_grid_on_ld():
    """test-8-LDpred2.R:63-65 on a synthetic LD matrix: the sampling betas' row means follow the grid's estimate."""
    Rm = banded_ld(400, 0.8, 30)
    bh, n, _ = sim_sumstats(Rm, h2=0.4, p=0.05, N=50_000, seed=6)
    st = api.sfbm_storage(Rm)
    ind = np.arange(400)
    grid = G.ldpred2_grid(st, bh, n, ind, [0.05], [0.4], [False], api.mrg32k3a_seed(1)[None], 50, 300)["beta_est"]
    S = G.ldpred2_grid(st, bh, n, ind, [0.05], [0.4], [False], api.mrg32k3a_seed(2)[None], 50, 300,
                       sampling=True)["sample_beta"]
    assert np.corrcoef(S.mean(1), grid[:, 0])[0, 1] > 0.9


def test_threads_batch_and_ind_corr():
    Rm = banded_ld(500, 0.8, 40)
    bh, n, _ = sim_sumstats(Rm, h2=0.3, p=0.05, N=20_000, seed=5)
    st = api.sfbm_storage(Rm)
    ps, h2s, sps = [0.2, 0.05, 0.01, 0.05, 0.001, 0.1], [0.3, 0.3, 0.2, 0.3, 0.3, 0.5], [0, 1, 1, 0, 1, 0]
    seeds = [api.mrg32k3a_seed(i) for i in range(6)]
    kw = dict(burn_in=10, num_iter=10)
    a = G.ldpred2_grid(st, bh, n, np.arange(500), ps, h2s, sps, seeds, nthreads=1, **kw)
    b = G.ldpred2_grid(st, bh, n, np.arange(500), ps, h2s, sps, seeds, nthreads=4, **kw)
    assert same(a["beta_est"], b["beta_est"]) and np.array_equal(a["rng_out"], b["rng_out"])
    one = G.ldpred2_grid(st, bh, n, np.arange(500), ps[2:3], h2s[2:3], sps[2:3], seeds[2:3], **kw)
    assert same(one["beta_est"][:, 0], a["beta_est"][:, 2])
    assert not np.array_equal(a["beta_est"][:, 1], a["beta_est"][:, 3])  # same p, h2 on another stream, not sparse
    ind = np.sort(np.random.default_rng(1).choice(500, 200, replace=False))
    x = G.ldpred2_grid(st, bh[ind], n[ind], ind, ps, h2s, sps, seeds, **kw)
    y = G.ldpred2_grid(api.sfbm_storage(sp.csc_matrix(Rm[ind][:, ind])), bh[ind], n[ind], np.arange(200), ps, h2s, sps,
                       seeds, **kw)
    assert same(x["beta_est"], y["beta_est"])


def test_oracle_is_uncontracted():
    out = subprocess.run(["objdump", "-d", G.object_file()], capture_output=True, text=True).stdout
    assert "vfmadd" not in out
    assert "-ffp-contract=off" in G.FLAGS


def test_kernel_ptx_has_no_fma(tmp_path):
    ptx = tmp_path / "sparse.ptx"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-ptx", "-arch=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-I",
                           os.path.join(ROOT, "bigsnpr_b200", "csrc"),
                           os.path.join(ROOT, "bigsnpr_b200", "csrc", "bsg_sparse.cu"), "-o", str(ptx)])
    text = ptx.read_text()
    bodies = re.findall(r"\.entry \w*?k_ldpred2_grid\w*\((.*?)\n}\n", text, re.S)
    assert len(bodies) == 2  # the grid and the sampling variant
    for b in bodies:
        assert "fma.rn.f64" not in b and "div.rn.f64" in b and "sqrt.rn.f64" in b


# ---- snp_ldpred2_grid's host logic, the device call replaced by the oracle --------------------------------------------------

class HostSFBM(api.SFBM):
    """An SFBM that keeps its storage on the host (isinstance checks pass; nothing touches a device)."""

    def __init__(self, A, compact=False):
        self.storage = api.sfbm_storage(A, compact=compact)
        self._n = self.storage[0]
        self._h = None

    @property
    def nrow(self):
        return self._n

    @property
    def ncol(self):
        return self._n


@pytest.fixture
def host_grid(monkeypatch):
    def call(corr, beta_hat, n_vec, ind_sub, p, h2, sparse, burn_in, num_iter, rng_state, sampling=False):
        r = G.ldpred2_grid(corr.storage, beta_hat, n_vec, ind_sub, p, h2, sparse, rng_state, burn_in, num_iter,
                           sampling=sampling)
        return {"beta_est": r["beta_est"], "sample_beta": r["sample_beta"], "time": np.zeros(np.size(p))}

    monkeypatch.setattr(api, "_ldpred2_grid_call", call)


def grid_df(m=80, seed=2):
    Rm = banded_ld(m, 0.7, 8)
    rng = np.random.default_rng(seed)
    beta_se = rng.uniform(0.01, 0.02, m)
    N = np.round(rng.uniform(8000, 10000, m))
    bh, _, _ = sim_sumstats(Rm, h2=0.4, p=0.1, N=10_000, seed=seed)
    scale_guess = np.sqrt(N) * beta_se
    return Rm, {"beta": bh * scale_guess, "beta_se": beta_se, "n_eff": N}


def test_order_restores_input_with_ties():
    p = np.array([0.1, 0.3, 0.1, 0.3, 0.1, 0.3, 0.01])
    h2 = np.array([0.2, 0.2, 0.5, 0.2, 0.2, 0.5, 0.2])
    s = np.array([True, False, False, False, True, True, False])
    o = api._ldpred2_grid_order(p, h2, s)
    # R: order(-p, sparse, -h2), ties in input order
    want = sorted(range(7), key=lambda i: (-p[i], s[i], -h2[i], i))
    assert o.tolist() == want


def test_snp_ldpred2_grid_order_seeds_and_scale(host_grid):
    Rm, df = grid_df()
    m = Rm.shape[0]
    corr = HostSFBM(Rm)
    grid = {"p": np.array([0.01, 0.1, 0.1, 0.3, 0.1]), "h2": np.array([0.3, 0.3, 0.5, 0.3, 0.3]),
            "sparse": np.array([False, True, False, False, False])}
    got = api.snp_ldpred2_grid(corr, df, grid, burn_in=5, num_iter=8, seed=11)
    assert got.shape == (m, 5)
    N = df["n_eff"]
    scale = np.sqrt(N * df["beta_se"] ** 2 + df["beta"] ** 2)
    bh = df["beta"] / scale
    order = [3, 2, 4, 1, 0]  # order(-p, sparse, -h2)
    states = [api.mrg32k3a_seed(11)]
    for _ in range(4):
        states.append(api.mrg32k3a_next_stream(states[-1]))
    for i, g in enumerate(order):
        one = G.ldpred2_grid(corr.storage, bh, N, np.arange(m), [grid["p"][g]], [grid["h2"][g]], [grid["sparse"][g]],
                             states[i][None], 5, 8)["beta_est"][:, 0]
        assert same(got[:, g], one * scale)
    again = api.snp_ldpred2_grid(corr, df, grid, burn_in=5, num_iter=8, seed=11)
    assert same(got, again)
    other = api.snp_ldpred2_grid(corr, df, grid, burn_in=5, num_iter=8, seed=12)
    assert not np.array_equal(got, other)
    smp = api.snp_ldpred2_grid(corr, df, {k: v[:1] for k, v in grid.items()}, burn_in=5, num_iter=8,
                               return_sampling_betas=True, seed=11)
    want = G.ldpred2_grid(corr.storage, bh, N, np.arange(m), grid["p"][:1], grid["h2"][:1], grid["sparse"][:1],
                          states[0][None], 5, 8, sampling=True)["sample_beta"]
    assert smp.shape == (m, 8) and same(smp, want * scale[:, None])


def test_snp_ldpred2_grid_argument_errors(host_grid):
    Rm, df = grid_df()
    m = Rm.shape[0]
    corr = HostSFBM(Rm)
    grid = {"p": np.array([0.1, 0.01]), "h2": np.array([0.3, 0.3]), "sparse": np.array([False, True])}
    cases = [
        (dict(df_beta={"beta": df["beta"], "beta_se": df["beta_se"]}), "'df_beta' should have element 'n_eff'."),
        (dict(grid_param={"p": grid["p"], "sparse": grid["sparse"]}), "'grid_param' should have element 'h2'."),
        (dict(ind_corr=np.arange(1, m)), None),
        (dict(ind_corr=np.arange(2, m + 2)), "all(ind.corr %in% cols_along(corr)) is not TRUE"),
        (dict(df_beta=dict(df, beta_se=np.where(np.arange(m) == 3, 0.0, df["beta_se"]))),
         "'df_beta$beta_se' should have only positive values."),
        (dict(grid_param=dict(grid, h2=np.array([0.3, 0.0]))), "'grid_param$h2' should have only positive values."),
        (dict(return_sampling_betas=True), "Only one set of parameters is allowed when using 'return_sampling_betas'."),
    ]
    for kw, msg in cases:
        a = dict(corr=corr, df_beta=df, grid_param=grid)
        a.update(kw)
        with pytest.raises(ValueError) as e:
            api.snp_ldpred2_grid(a.pop("corr"), a.pop("df_beta"), a.pop("grid_param"), burn_in=1, num_iter=1, **a)
        if msg is not None:
            assert str(e.value) == msg
    with pytest.raises(TypeError):
        api.snp_ldpred2_grid(Rm, df, grid)
    with pytest.raises(TypeError):
        api.snp_ldpred2_grid(corr, df, 0.1)
