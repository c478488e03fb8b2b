"""snp_ldpred2_auto / bsg_ldpred2_auto on the device against the CPU oracle (tests/ldpred2_auto_oracle.c): every output
byte-identical (NaN as NaN), in both SFBM storage forms; launch independence; the ABI errors."""
import numpy as np
import pytest

import bigsnpr_b200 as B
from bigsnpr_b200 import _lib, api
from tests import ldpred2_auto_ref as R
from tests.test_gpu_lassosum2 import bed_fixture
from tests.test_ldpred2_auto_oracle import same
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
    """bsg_open_synth_ld, 2,000 samples x 20,000 SNPs, 100-SNP window (the matrix of test_gpu_ldpred2_inf)."""
    g = B.Bed.synthetic(2000, 20000, seed=11, ld_rho=0.9, ld_block=50)
    G = B.read_bed(g, g.rows_along(), g.cols_along(), na_val=3)
    keep = (np.flatnonzero(G.std(0) > 0) + 1).astype(np.int32)
    corr = B.bed_cor(g, ind_col=keep, size=100)
    g.close()
    return corr, sumstats(G[:, keep - 1], 5)


def inputs(df):
    N = np.asarray(df["n_eff"], dtype=np.float64)
    sd = 1 / np.sqrt(N * df["beta_se"] ** 2 + df["beta"] ** 2)
    return df["beta"] * sd, N, 2 * np.log(sd)


def check(corr, df, compact, p_init=(0.1,), ind=None, mean_ld=None, **kw):
    """The device call == the oracle on the same storage, byte for byte; returns the device result."""
    bh, N, lv = inputs(df)
    st = api.sfbm_storage(corr, compact=compact)
    m = bh.size
    ind = np.arange(m, dtype=np.int32) if ind is None else np.asarray(ind, dtype=np.int32)
    if ind.size != m:
        bh, N, lv = bh[ind], N[ind], lv[ind]
    p_init = np.asarray(p_init, dtype=np.float64)
    rng = np.array([api.mrg32k3a_seed(1000 + i) for i in range(p_init.size)])
    args = dict(burn_in=30, num_iter=20, report_step=5, no_jump_sign=False, shrink_corr=1.0, use_mle=True,
                p_bounds=(1e-5, 1.0), alpha_bounds=(-0.5, 1.5), h2_init=0.3)
    args.update(kw)
    sf = api.SFBM(st[0], st[0], st[1], st[2], st[3])
    try:
        if mean_ld is None:
            mean_ld = float(np.mean(B.ld_scores_sfbm(sf, ind + 1)))
        got = api._ldpred2_auto_call(sf, bh, N, lv, ind, p_init, args["h2_init"], args["burn_in"], args["num_iter"],
                                     args["report_step"], args["no_jump_sign"], args["shrink_corr"], args["use_mle"],
                                     np.array(args["p_bounds"]), np.array(args["alpha_bounds"]), mean_ld, rng)
    finally:
        sf.close()
    want = R.ldpred2_auto(st, bh, N, lv, ind, p_init, rng=rng, mean_ld=mean_ld, **args)
    same(got, want)
    return got


@pytest.mark.parametrize("compact", [False, True])
@pytest.mark.parametrize("which", ["example", "example_missing"])
def test_bed_cor_matrices(which, compact, request):
    g, poly, corr, df = request.getfixturevalue(which)
    check(corr, df, compact, p_init=(0.2, 0.01, 0.1))
    check(corr, df, compact, use_mle=False, no_jump_sign=True)
    check(corr, df, compact, shrink_corr=0.95, p_bounds=(0.05, 0.05), alpha_bounds=(0.0, 0.0), report_step=1)


@pytest.mark.parametrize("compact", [False, True])
def test_synth_30_chains(synth, compact):
    corr, df = synth
    got = check(corr, df, compact, p_init=api.seq_log(1e-4, 0.2, 30), burn_in=20, num_iter=10)
    assert np.all(np.isfinite(got["beta_est"]))


def test_more_chains_than_sms(example):
    g, poly, corr, df = example
    p = np.tile(api.seq_log(1e-3, 0.5, 10), 20)  # 200 chains
    got = check(corr, df, False, p_init=p, burn_in=5, num_iter=5)
    # a chain's result does not depend on the launch: chain 7 alone
    one = check(corr, df, False, p_init=p[:8], burn_in=5, num_iter=5)
    assert got["beta_est"][:, 7].tobytes() == one["beta_est"][:, 7].tobytes()


def test_unsorted_ind_corr_with_repeat(example):
    g, poly, corr, df = example
    rng = np.random.default_rng(3)
    ind = rng.choice(len(corr[0]) - 1, 400, replace=False)
    ind[5] = ind[17]
    check(corr, df, True, ind=ind, p_init=(0.05, 0.3))


def test_diverging_case():
    m = 60
    A = np.eye(m) + np.diag(np.full(m - 1, -0.9), 1) + np.diag(np.full(m - 1, -0.9), -1)
    import scipy.sparse as sp

    rng = np.random.default_rng(0)
    df = {"beta": rng.normal(0, 0.05, m) * 0.3162, "beta_se": np.full(m, 1e-3), "n_eff": np.full(m, 1e5)}
    got = check(sp.csc_matrix(A), df, False, p_init=(0.9,), burn_in=30, num_iter=10, p_bounds=(0.9, 0.9),
                use_mle=False, mean_ld=3.0)
    assert np.all(np.isnan(got["beta_est"]))


def test_snp_ldpred2_auto_end_to_end(example):
    g, poly, corr, df = example
    sf = B.as_SFBM(corr)
    try:
        kw = dict(vec_p_init=[0.01, 0.2, 0.05], burn_in=20, num_iter=10, report_step=3, seed=5)
        a = B.snp_ldpred2_auto(sf, df, 0.3, **kw)
        b = B.snp_ldpred2_auto(sf, df, 0.3, **kw)
        mean_ld = float(np.mean(B.ld_scores_sfbm(sf)))
    finally:
        sf.close()
    assert len(a) == 3 and [r["p_init"] for r in a] == [0.01, 0.2, 0.05]
    for x, y in zip(a, b):  # two calls are identical
        assert x["beta_est"].tobytes() == y["beta_est"].tobytes()
        assert (x["sample_beta"] != y["sample_beta"]).nnz == 0
    # the chains ran in order(-vec_p_init): 0.2 on the first stream, 0.05 on the second, 0.01 on the third
    bh, N, lv = inputs(df)
    sd = 1 / np.sqrt(N * df["beta_se"] ** 2 + df["beta"] ** 2)  # as snp_ldpred2_auto forms it
    s0 = api.mrg32k3a_seed(5)
    s1 = api.mrg32k3a_next_stream(s0)
    s2 = api.mrg32k3a_next_stream(s1)
    st = api.sfbm_storage(corr)
    want = R.ldpred2_auto(st, bh, N, lv, np.arange(bh.size), np.array([0.2, 0.05, 0.01]), h2_init=0.3,
                          rng=np.array([s0, s1, s2]), burn_in=20, num_iter=10, report_step=3, mean_ld=mean_ld)
    for i, c in enumerate([1, 2, 0]):
        r = a[c]
        assert r["beta_est"].tobytes() == (want["beta_est"][:, i] / sd).tobytes()
        assert r["sample_beta"].shape == (bh.size, 3)
        assert np.array_equal(r["sample_beta"].toarray(), want["sample_beta"][:, :, i])
        assert r["h2_est"] == np.mean(want["path_h2_est"][-10:, i])
        assert r["alpha_est"] == np.mean(want["path_alpha_est"][-10:, i])
    with pytest.raises(NotImplementedError):
        B.snp_ldpred2_auto(None, df, 0.3, sparse=True)


def test_abi_errors(example):
    g, poly, corr, df = example
    bh, N, lv = inputs(df)
    m = bh.size
    st = api.sfbm_storage(corr)
    sf = api.SFBM(st[0], st[0], st[1], st[2], st[3])
    ind = np.arange(m, dtype=np.int32)
    good = dict(rng=np.array([api.mrg32k3a_seed(1)]), p_bounds=np.array([1e-5, 1.0]), alpha_bounds=np.array([-0.5, 1.5]),
                burn_in=2, num_iter=2, report_step=1, mean_ld=2.0, ind=ind)

    def call(**kw):
        a = dict(good, **kw)
        api._ldpred2_auto_call(sf, bh, N, lv, a["ind"], np.array([0.1]), 0.3, a["burn_in"], a["num_iter"],
                               a["report_step"], False, 1.0, True, a["p_bounds"], a["alpha_bounds"], a["mean_ld"], a["rng"])

    try:
        call()
        bad_state = np.array([[0, 0, 0, 1, 2, 3]], dtype=np.uint32)
        big_state = np.array([[4294967087, 1, 2, 1, 2, 3]], dtype=np.uint32)
        cases = [dict(rng=bad_state), dict(rng=big_state), dict(num_iter=0), dict(burn_in=-1), dict(report_step=0),
                 dict(p_bounds=np.array([0.5, 0.1])), dict(alpha_bounds=np.array([1.0, 0.0])), dict(mean_ld=0.0)]
        for kw in cases:
            with pytest.raises(_lib.BsgError) as e:
                call(**kw)
            assert e.value.code == 9, kw
        with pytest.raises(_lib.BsgError) as e:
            call(ind=np.full(m, st[0], dtype=np.int32))
        assert e.value.code == 2
    finally:
        sf.close()
