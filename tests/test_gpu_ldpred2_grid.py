"""snp_ldpred2_grid / bsg_ldpred2_grid and bsg_ldpred2_auto_ex's final states on the device against the CPU oracle
(tests/ldpred2_grid_oracle.c): every output byte-identical (NaN payloads compared), in both SFBM storage forms; launch
independence; the ABI errors."""
import numpy as np
import pytest
import scipy.sparse as sp

import bigsnpr_b200 as B
from bigsnpr_b200 import _lib, api
from tests import ldpred2_grid_ref as G
from tests.test_gpu_lassosum2 import bed_fixture
from tests.test_gpu_ldpred2_auto import inputs
from tests.test_lassosum2_oracle import sumstats

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def example():
    return bed_fixture("example.bed", 1)


@pytest.fixture(scope="module")
def example_missing():
    return bed_fixture("example-missing.bed", 2)


@pytest.fixture(scope="module")
def synth():
    """bsg_open_synth_ld, 2,000 samples x 20,000 SNPs, 100-SNP window (the matrix of test_gpu_ldpred2_auto)."""
    g = B.Bed.synthetic(2000, 20000, seed=11, ld_rho=0.9, ld_block=50)
    G_ = B.read_bed(g, g.rows_along(), g.cols_along(), na_val=3)
    keep = (np.flatnonzero(G_.std(0) > 0) + 1).astype(np.int32)
    corr = B.bed_cor(g, ind_col=keep, size=100)
    g.close()
    return corr, sumstats(G_[:, keep - 1], 5)


def same_bytes(a, b):
    """identical bytes, NaN entries included (payloads compared)"""
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def grid_inputs(df):
    N = np.asarray(df["n_eff"], dtype=np.float64)
    scale = np.sqrt(N * df["beta_se"] ** 2 + df["beta"] ** 2)
    return df["beta"] / scale, N


def check(corr, df, compact, p, h2, sparse, ind=None, seed0=1000, sampling=False, burn_in=20, num_iter=15):
    """The device call == the oracle on the same storage, byte for byte; returns the device result."""
    bh, N = grid_inputs(df)
    st = api.sfbm_storage(corr, compact=compact)
    m = bh.size
    ind = np.arange(m, dtype=np.int32) if ind is None else np.asarray(ind, dtype=np.int32)
    if ind.size != m:
        bh, N = bh[ind], N[ind]
    rng = np.array([api.mrg32k3a_seed(seed0 + i) for i in range(len(p))])
    sf = api.SFBM(st[0], st[0], st[1], st[2], st[3])
    try:
        got = api._ldpred2_grid_call(sf, bh, N, ind, p, h2, sparse, burn_in, num_iter, rng, sampling=sampling)
    finally:
        sf.close()
    want = G.ldpred2_grid(st, bh, N, ind, p, h2, sparse, rng, burn_in, num_iter, sampling=sampling)
    k = "sample_beta" if sampling else "beta_est"
    assert same_bytes(got[k], want[k])
    return got


def full_grid():
    """21 p x 4 h2 x 2 sparse: 168 points"""
    p = api.seq_log(1e-5, 1, 21)
    h2 = np.array([0.7, 1.0, 1.4]) * 0.3
    h2 = np.append(h2, 0.2)
    P, H, S = np.meshgrid(p, h2, [False, True], indexing="ij")
    return P.ravel(), H.ravel(), S.ravel()


@pytest.mark.parametrize("compact", [False, True])
@pytest.mark.parametrize("which", ["example", "example_missing"])
def test_bed_cor_matrices(which, compact, request):
    g, poly, corr, df = request.getfixturevalue(which)
    check(corr, df, compact, [0.3, 0.01, 0.1, 1.0], [0.3, 0.2, 0.5, 0.3], [False, True, True, False])
    check(corr, df, compact, [0.05], [0.3], [True], sampling=True)
    check(corr, df, compact, [0.05], [0.3], [False], sampling=True)


@pytest.mark.parametrize("compact", [False, True])
def test_synth_full_grid(synth, compact):
    corr, df = synth
    p, h2, s = full_grid()
    got = check(corr, df, compact, p, h2, s, burn_in=5, num_iter=5)
    assert got["beta_est"].shape[1] == 168
    # a point's result does not depend on the launch: point 7 alone
    one = check(corr, df, compact, p[7:8], h2[7:8], s[7:8], seed0=1007, burn_in=5, num_iter=5)
    assert one["beta_est"][:, 0].tobytes() == got["beta_est"][:, 7].tobytes()


def test_unsorted_ind_corr_with_repeat(example):
    g, poly, corr, df = example
    rng = np.random.default_rng(3)
    ind = rng.choice(len(corr[0]) - 1, 400, replace=False)
    ind[5] = ind[17]
    check(corr, df, True, [0.05, 0.3], [0.3, 0.3], [True, False], ind=ind)


def test_diverging_point():
    m = 60
    A = np.eye(m) + np.diag(np.full(m - 1, -0.9), 1) + np.diag(np.full(m - 1, -0.9), -1)
    rng = np.random.default_rng(0)
    df = {"beta": rng.normal(0, 0.05, m) * 0.3162, "beta_se": np.full(m, 1e-3), "n_eff": np.full(m, 1e5)}
    got = check(sp.csc_matrix(A), df, False, [0.9, 0.9], [1.0, 1.0], [False, True], burn_in=30, num_iter=10)
    assert np.all(got["beta_est"].view(np.uint64) == 0x7FF00000000007A2)


def test_snp_ldpred2_grid_end_to_end(example):
    g, poly, corr, df = example
    sf = B.as_SFBM(corr)
    grid = {"p": np.array([0.01, 0.1, 0.1, 0.3, 0.1]), "h2": np.array([0.3, 0.3, 0.5, 0.3, 0.3]),
            "sparse": np.array([False, True, False, False, False])}
    try:
        a = B.snp_ldpred2_grid(sf, df, grid, burn_in=10, num_iter=10, seed=5)
        b = B.snp_ldpred2_grid(sf, df, grid, burn_in=10, num_iter=10, seed=5)
        c = B.snp_ldpred2_grid(sf, df, grid, burn_in=10, num_iter=10, seed=6)
        smp = B.snp_ldpred2_grid(sf, df, {k: v[1:2] for k, v in grid.items()}, burn_in=10, num_iter=10,
                                 return_sampling_betas=True, seed=5)
        with pytest.raises(ValueError):
            B.snp_ldpred2_grid(sf, df, grid, return_sampling_betas=True)
    finally:
        sf.close()
    assert same_bytes(a, b) and not np.array_equal(a, c)
    bh, N = grid_inputs(df)
    scale = np.sqrt(N * df["beta_se"] ** 2 + df["beta"] ** 2)
    st = api.sfbm_storage(corr)
    states = [api.mrg32k3a_seed(5)]
    for _ in range(4):
        states.append(api.mrg32k3a_next_stream(states[-1]))
    order = [3, 2, 4, 1, 0]  # order(-p, sparse, -h2)
    want = G.ldpred2_grid(st, bh, N, np.arange(bh.size), grid["p"][order], grid["h2"][order], grid["sparse"][order],
                          np.array(states), 10, 10)["beta_est"]
    for i, k in enumerate(order):
        assert a[:, k].tobytes() == (want[:, i] * scale).tobytes()
    ws = G.ldpred2_grid(st, bh, N, np.arange(bh.size), grid["p"][1:2], grid["h2"][1:2], grid["sparse"][1:2],
                        states[0][None], 10, 10, sampling=True)["sample_beta"]
    assert smp.tobytes() == np.asfortranarray(ws * scale[:, None]).tobytes()


@pytest.mark.parametrize("compact", [False, True])
def test_auto_final_state_continues_into_sparse_gibbs(example, compact):
    """bsg_ldpred2_auto_ex: the chains' outputs equal bsg_ldpred2_auto's and the oracle's, and rng_out is the oracle's
    final state; a sparse grid point run from it with the chain's p_est and h2_est (R/LDpred2.R:266-279) equals the
    oracle's run from the oracle's own state."""
    g, poly, corr, df = example
    st = api.sfbm_storage(corr, compact=compact)
    sf = api.SFBM(st[0], st[0], st[1], st[2], st[3])
    bh, N, lv = inputs(df)
    p_init = np.array([0.2, 0.05, 0.01])
    states = api._mrg_streams(7, 3)
    args = (np.arange(bh.size), p_init, 0.3, 20, 10, 3, False, 1, True, np.array([1e-5, 1.0]), np.array([-0.5, 1.5]))
    try:
        mean_ld = float(np.mean(B.ld_scores_sfbm(sf)))
        plain = api._ldpred2_auto_call(sf, bh, N, lv, *args, mean_ld, states)
        ends = api._ldpred2_auto_call(sf, bh, N, lv, *args, mean_ld, states, rng_out=True)
        p_est, h2_est = ends["path_p_est"][-10:].mean(0), ends["path_h2_est"][-10:].mean(0)
        sparse = api._ldpred2_grid_call(sf, bh, N, np.arange(bh.size), p_est, h2_est, [True] * 3, 50, 100,
                                        ends["rng_out"])
    finally:
        sf.close()
    for k in plain:
        if k not in ("time", "sample_beta"):
            assert plain[k].tobytes() == ends[k].tobytes(), k
    assert plain["sample_beta"].tobytes() == ends["sample_beta"].tobytes()
    want = G.ldpred2_auto_state(st, bh, N, lv, np.arange(bh.size), p_init, 0.3, states, burn_in=20, num_iter=10,
                                report_step=3, mean_ld=mean_ld)
    assert np.array_equal(ends["rng_out"], want["rng_out"])
    for k in ("beta_est", "postp_est", "corr_est", "path_p_est", "path_h2_est", "path_alpha_est"):
        assert ends[k].tobytes() == want[k].tobytes(), k
    assert np.all(np.isfinite(h2_est))
    g1 = G.ldpred2_grid(st, bh, N, np.arange(bh.size), p_est, h2_est, [True] * 3, want["rng_out"], 50, 100)
    assert sparse["beta_est"].tobytes() == g1["beta_est"].tobytes()


def test_auto_final_state_of_a_diverged_chain():
    m = 60
    A = np.eye(m) + np.diag(np.full(m - 1, -0.9), 1) + np.diag(np.full(m - 1, -0.9), -1)
    rng = np.random.default_rng(0)
    bh, N, lv = rng.normal(0, 0.05, m), np.full(m, 1e5), np.full(m, -2.0)
    st = api.sfbm_storage(sp.csc_matrix(A))
    sf = api.SFBM(st[0], st[0], st[1], st[2], st[3])
    states = api._mrg_streams(1, 1)
    args = (np.arange(m), np.array([0.9]), 0.3, 30, 10, 11, False, 1, False, np.array([0.9, 0.9]), np.array([0.0, 0.0]),
            3.0, states)
    try:
        ends = api._ldpred2_auto_call(sf, bh, N, lv, *args, rng_out=True)
    finally:
        sf.close()
    want = G.ldpred2_auto_state(st, bh, N, lv, *args[:3], states, burn_in=30, num_iter=10, report_step=11,
                                use_mle=False, p_bounds=(0.9, 0.9), alpha_bounds=(0.0, 0.0), mean_ld=3.0)
    assert np.all(np.isnan(ends["beta_est"])) and np.array_equal(ends["rng_out"], want["rng_out"])


def test_abi_errors(example):
    g, poly, corr, df = example
    bh, N = grid_inputs(df)
    m = bh.size
    st = api.sfbm_storage(corr)
    sf = api.SFBM(st[0], st[0], st[1], st[2], st[3])
    ind = np.arange(m, dtype=np.int32)
    good = dict(rng=np.array([api.mrg32k3a_seed(1)]), burn_in=2, num_iter=2, ind=ind, p=[0.1], sampling=False)

    def call(**kw):
        a = dict(good, **kw)
        n = len(a["p"])
        api._ldpred2_grid_call(sf, bh, N, a["ind"], a["p"], [0.3] * n, [False] * n, a["burn_in"], a["num_iter"],
                               a["rng"], sampling=a["sampling"])

    try:
        call()
        call(sampling=True)
        bad_state = np.array([[0, 0, 0, 1, 2, 3]], dtype=np.uint32)
        big_state = np.array([[4294967087, 1, 2, 1, 2, 3]], dtype=np.uint32)
        two = np.array([api.mrg32k3a_seed(1), api.mrg32k3a_seed(2)])
        cases = [dict(rng=bad_state), dict(rng=big_state), dict(num_iter=0), dict(burn_in=-1),
                 dict(sampling=True, p=[0.1, 0.2], rng=two)]
        for kw in cases:
            with pytest.raises(_lib.BsgError) as e:
                call(**kw)
            assert e.value.code == 9, kw
        with pytest.raises(_lib.BsgError) as e:
            call(ind=np.full(m, st[0], dtype=np.int32))
        assert e.value.code == 2
    finally:
        sf.close()
    rect = api.SFBM(st[0] + 1, st[0], st[1], st[2], st[3])
    try:
        with pytest.raises(_lib.BsgError) as e:
            api._ldpred2_grid_call(rect, bh, N, ind, [0.1], [0.3], [False], 2, 2, good["rng"])
        assert e.value.code == 1
    finally:
        rect.close()
