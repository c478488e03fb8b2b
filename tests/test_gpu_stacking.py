"""big_spLinReg / big_spLogReg over dense float32 / float64 matrices (bsg_splreg_dense) and snp_grid_stacking on the device.

- Dense fits equal tests/splreg_ref.py on X.astype(float64) byte for byte (paths, losses, messages, coefficients, chosen
  alpha): 0 / 10 covariates, base, zero pf_X, repeated rows, an all-zero column (dropped), an np.memmap.
- The dense path is the genotype path's solver: a float32 matrix of example.bed's codes gives the Bed fit's bytes;
  permuted columns and other alphas in the call change nothing.
- The reference's test-6-SCT.R scenario on example.bed, and an LD-structured case against the C oracle.
- Refusals: non-finite cells, dtypes, non-0/1 binary y, dimensions, a device-memory shortfall."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import gwas_ref as GR
from tests import splreg_ref as S
from tests.test_gpu_splreg import _bytes, _cols, _pheno, _same
from tests.test_stacking_ref import r_fold

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
N, M = 517, 4542
PATH = dict(nlambda=30, lambda_min_ratio=1e-2, nlam_min=10, n_abort=5)


@pytest.fixture(scope="module")
def B():
    import bigsnpr_b200 as B

    return B


@pytest.fixture(scope="module")
def codes():
    return GR.read_bed_codes(os.path.join(GOLDEN, "example.bed"), N, M)


def _run(B, X, rows, cols, y, family, covar=None, base=None, pf_X=None, pf_covar=None, alphas=(1.0,), K=4, seed=3,
         path=True, engine="c", **kw):
    fn = B.big_spLogReg if family else B.big_spLinReg
    mod = fn(X, y, ind_train=rows, ind_col=cols, covar_train=covar, base_train=base, pf_X=pf_X, pf_covar=pf_covar,
             alphas=alphas, K=K, seed=seed, return_path=path, **kw)
    Xd = np.asarray(X)[np.ix_(np.asarray(rows) - 1, np.asarray(cols) - 1)].astype(np.float64)
    sets = S.folds_from_seed(len(rows), K, seed)
    assert np.array_equal(mod.ind_sets, sets)
    ref = S.splreg(Xd, y, family, sets, K, covar=covar, base=base, pf_X=pf_X, pf_covar=pf_covar, alphas=alphas,
                   keep_path=path, col_key=np.asarray(cols), engine=engine, **kw)
    assert np.array_equal(mod.ind_col, np.asarray(cols)[ref["kept"]])
    _bytes(mod.center, ref["center"][_cols(ref)])
    _bytes(mod.scale, ref["scale"][_cols(ref)])
    _same(B, mod, ref, len(alphas), K)
    return mod, ref, Xd


def _dense(rng, n, m, dtype):
    """correlated continuous columns (a random walk across columns, like C+T scores over thresholds)"""
    X = np.cumsum(rng.normal(size=(n, m)), axis=1) / np.sqrt(np.arange(1, m + 1))
    return np.asfortranarray(X.astype(dtype))


CASES = [
    (0, 0, False, False, (1.0,), False),
    (0, 10, True, True, (1.0, 0.5, 1e-4), True),
    (1, 0, False, False, (1.0, 0.5), True),
    (1, 10, True, True, (1.0, 1e-4), False),
]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("family,Kc,use_base,pf0,alphas,repeats", CASES)
def test_dense_fits(B, dtype, family, Kc, use_base, pf0, alphas, repeats):
    rng = np.random.default_rng(family * 10 + Kc + len(alphas))
    n, m = 700, 160
    X = _dense(rng, n, m, dtype)
    X[:, 7] = 0.0                                               # an all-zero column: dropped
    cols = rng.permutation(np.setdiff1d(np.arange(1, m + 1), [8]))[:120]
    cols = np.concatenate([cols, [8]])
    rows = rng.choice(n, 600, replace=False) + 1
    if repeats:
        rows = np.concatenate([rows, rng.choice(n, 60) + 1])
    nr = rows.size
    y = _pheno(rng, np.asarray(X, dtype=np.float64)[np.ix_(rows - 1, cols - 1)], family)
    covar = rng.normal(size=(nr, Kc)) if Kc else None
    base = 0.2 * rng.normal(size=nr) if use_base else None
    pf_X = None
    if pf0:
        pf_X = np.ones(cols.size)
        pf_X[:2] = 0.0
    pf_covar = np.zeros(Kc) if (pf0 and Kc) else None
    mod, ref, Xd = _run(B, X, rows, cols, y, family, covar=covar, base=base, pf_X=pf_X, pf_covar=pf_covar,
                        alphas=alphas, **PATH)
    assert 8 not in mod.ind_col and mod.ind_col.size == cols.size - 1
    # predict on the dense matrix: the host product of the returned beta
    i = mod.best_alpha
    pred = mod.predict(X, rows, covar, base_row=base)
    G = mod.ind_col.size
    host = Xd[:, ref["kept"]] @ mod.beta[i][:G] + mod.intercept[i] + (0 if base is None else base)
    if Kc:
        host = host + covar @ mod.beta[i][G:]
    np.testing.assert_allclose(pred, host, rtol=1e-12, atol=1e-12 * np.abs(host).max())


def test_memmap_and_c_order(B, tmp_path):
    rng = np.random.default_rng(4)
    n, m = 500, 90
    X = _dense(rng, n, m, np.float32)
    mm = np.memmap(str(tmp_path / "multi.bk"), dtype=np.float32, mode="w+", shape=(n, m), order="F")
    mm[:] = X
    mm.flush()
    ro = np.memmap(str(tmp_path / "multi.bk"), dtype=np.float32, mode="r", shape=(n, m), order="F")
    rows, cols = np.arange(1, n + 1), np.arange(1, m + 1)
    y = _pheno(rng, X.astype(np.float64), 0)
    a = _run(B, ro, rows, cols, y, 0, **PATH)[0]
    b = B.big_spLinReg(np.ascontiguousarray(X), y, K=4, seed=3, **PATH)   # copied into Fortran order first
    _bytes(a.raw["beta"], b.raw["beta"])
    _bytes(a.raw["b0"], b.raw["b0"])
    big = np.asfortranarray(np.vstack([X, X[:37]]))                       # a row slice: leading dimension n + 37
    c = B.big_spLinReg(big[:n], y, K=4, seed=3, **PATH)
    _bytes(a.raw["beta"], c.raw["beta"])


def test_same_solver_as_genotypes(B, codes):
    """A float32 matrix of example.bed's decoded codes: the Bed fit's bytes, paths included; then permuted columns and
    other alphas in the call."""
    rng = np.random.default_rng(17)
    Xb = B.Bed(os.path.join(GOLDEN, "example.bed"))
    cols = np.sort(rng.choice(M, 250, replace=False)) + 1
    y = _pheno(rng, codes[:, cols - 1].astype(float), 1)
    cov = rng.normal(size=(N, 3))
    kw = dict(K=4, seed=2, covar_train=cov, return_path=True, **PATH)
    for fn in (B.big_spLinReg, B.big_spLogReg):
        yy = y if fn is B.big_spLogReg else y + rng.normal(size=N)
        g = fn(Xb, yy, ind_col=cols, alphas=(1.0, 0.5), **kw)
        D = np.asfortranarray(codes[:, cols - 1].astype(np.float32))
        d = fn(D, yy, alphas=(1.0, 0.5), **kw)
        for key in ("beta", "b0", "best", "length", "message"):
            _bytes(g.raw[key], d.raw[key])
        for a in range(2):
            for k in range(4):
                for key in ("lambda_", "loss", "nnz", "passes", "beta", "intercept"):
                    _bytes(g.path[a][k][key], d.path[a][k][key])
        _bytes(g.center, d.center)
        _bytes(g.scale, d.scale)
        # permuted columns, one alpha: the same bytes once the permutation is undone
        perm = rng.permutation(cols.size)
        p = fn(D, yy, ind_col=perm + 1, alphas=(0.5,), **kw)
        at = {c: i for i, c in enumerate(p.ind_col)}
        idx = np.array([at[c] for c in d.ind_col] + list(p.ind_col.size + np.arange(3)))
        _bytes(p.raw["beta"][0][:, idx], d.raw["beta"][1])
        _bytes(p.raw["b0"][0], d.raw["b0"][1])


def _sct_setup(B, codes, typ):
    """test-6-SCT.R on example.bed: two chromosomes, a 3 x 2 grid, thresholds 0:5, seeded lpval, betas and 0/1 y."""
    G = B.Bed(os.path.join(GOLDEN, "example.bed"))
    CHR = np.repeat([1, 2], [2542, 2000])
    POS = np.array([float(ln.split()[3]) for ln in open(os.path.join(GOLDEN, "example.bim"))])
    rng = np.random.default_rng(2024)
    lpval = -np.log10(rng.uniform(size=M))
    betas = rng.normal(scale=0.1, size=M)
    y = rng.integers(0, 2, size=N).astype(np.float64)
    all_keep = B.snp_grid_clumping(G, CHR, POS, lpval, grid_thr_r2=(0.05, 0.2, 0.8), grid_base_size=(100, 200))
    multi = B.snp_grid_PRS(G, all_keep, betas, lpval, grid_lpS_thr=np.arange(6.0), type=typ)
    assert multi.shape == (N, 6 * sum(len(c) for c in all_keep))
    return G, multi, y


def _all_equal(target, current):
    """R's all.equal for numeric vectors: the mean relative difference"""
    return np.mean(np.abs(target - current)) / np.mean(np.abs(target))


@pytest.mark.parametrize("typ,tol", [("float", 1e-6), ("double", 1e-10)])
def test_sct_reference_scenario(B, codes, typ, tol):
    G, multi, y = _sct_setup(B, codes, typ)
    res = B.snp_grid_stacking(multi, y, alphas=1e-3)
    assert res["beta.covar"].size == 0
    pred = res["mod"].predict(multi)
    want = res["intercept"] + B.bed_prodVec(G, res["beta.G"])
    assert _all_equal(pred, want) < tol
    # the whole output: splreg_ref on multi.astype(float64), then the literal fold of R/SCT.R
    mod = res["mod"]
    nc = multi.shape[1]
    sets = S.folds_from_seed(N, 10, 1)
    ref = S.splreg(np.asarray(multi, dtype=np.float64), y, 1, sets, 10, alphas=(1e-3,), engine="c")
    _same(B, mod, ref, 1, 10)
    ob, oi = B.api.splreg_unscale(np.array([[r["beta"] for r in ref["fits"]]]), np.array([[r["b0"] for r in ref["fits"]]]),
                                  ref["center"][_cols(ref)], ref["scale"][_cols(ref)])
    w = np.zeros(nc)
    w[np.flatnonzero(ref["kept"])] = ob[0]
    _bytes(res["beta.G"], r_fold(w, multi.lpS, multi.grid_lpS_thr, multi.betas, multi.all_keep))
    _bytes(res["intercept"], oi[0])


@pytest.mark.parametrize("family", [0, 1])
def test_ld_pipeline_against_c_oracle(B, family):
    """20,000 rows, 4 pseudo-chromosomes, ~1,000 C+T columns, K = 3, a short path: the C oracle's bytes."""
    n, m = 20_000, 4_000
    g = B.Bed.synthetic(n, m, seed=9, ld_rho=0.9, ld_block=50)
    rng = np.random.default_rng(8)
    causal = np.sort(rng.choice(m, 40, replace=False)) + 1
    Xc = B.read_bed(g, g.rows_along(), causal).astype(np.float64)
    lin = (Xc - Xc.mean(0)) @ rng.normal(size=causal.size)
    lin = lin / np.std(lin)
    y = lin + rng.normal(size=n) * 1.5 if family == 0 else (rng.random(n) < 1 / (1 + np.exp(-lin))).astype(float)
    train = np.sort(rng.choice(n, 15_000, replace=False)) + 1
    gw = B.big_univLinReg(g, y[train - 1], ind_train=train)
    lp = -gw.predict()
    chr_ = np.repeat(np.arange(1, 5), m // 4)
    pos = np.tile(np.arange(1, m // 4 + 1) * 1000.0, 4)
    keep = B.snp_grid_clumping(g, chr_, pos, lp, ind_row=train, grid_thr_r2=(0.1, 0.2, 0.8),
                             grid_base_size=(50, 200))
    multi = B.snp_grid_PRS(g, keep, gw.estim, lp, n_thr_lpS=40, ind_row=train)
    assert 800 <= multi.shape[1] <= 1400
    # the logistic descent over near-collinear score columns is slow far down the path: its path is shorter
    path = dict(nlambda=8, lambda_min_ratio=0.3) if family == 0 else dict(nlambda=4, lambda_min_ratio=0.6)
    path.update(nlam_min=path["nlambda"], n_abort=path["nlambda"])
    res = B.snp_grid_stacking(multi, y[train - 1], alphas=(1.0,), K=3, **path)
    sets = S.folds_from_seed(train.size, 3, 1)
    ref = S.splreg(np.asarray(multi, dtype=np.float64), y[train - 1], family, sets, 3, alphas=(1.0,), engine="c",
                   **path)
    assert res["mod"].family == ("binomial" if family else "gaussian")
    _same(B, res["mod"], ref, 1, 3)


def test_refusals(B):
    rng = np.random.default_rng(3)
    n, m = 300, 40
    X = _dense(rng, n, m, np.float32)
    y = rng.normal(size=n)
    for bad, col in ((np.nan, 5), (np.inf, 17), (-np.inf, 33)):
        Xb = X.copy(order="F")
        Xb[11, col - 1] = bad
        with pytest.raises(B.BsgError, match="Column %d " % col):
            B.big_spLinReg(Xb, y, K=3)
        rows = np.setdiff1d(np.arange(1, n + 1), [12])      # the cell's row is not a training row: accepted
        B.big_spLinReg(Xb, y[rows - 1], ind_train=rows, K=3, nlambda=5)
        B.big_spLinReg(Xb, y, ind_col=np.setdiff1d(np.arange(1, m + 1), [col]), K=3, nlambda=5)
    for dt in (np.int32, np.float16, np.uint8):
        with pytest.raises(TypeError):
            B.big_spLinReg(X.astype(dt), y, K=3)
    yb = np.where(y > 0, 2.0, 1.0)                           # two values, not 0 / 1: the logistic choice refuses it
    multi = X.view(B.GridPRS)
    multi.lpS, multi.grid_lpS_thr, multi.betas = np.ones(4), np.array([0.5]), np.ones(4)
    multi.all_keep = [[np.array([1])] * 40, [np.zeros(0, dtype=int)] * 0]
    with pytest.raises(B.BsgError, match="0 or 1"):
        B.snp_grid_stacking(multi, yb, K=3)
    with pytest.raises(ValueError):
        B.big_spLinReg(X, y[:-1], K=3)
    with pytest.raises(ValueError):
        B.big_spLinReg(X, y, K=3, covar_train=rng.normal(size=(n - 1, 2)))
    with pytest.raises(ValueError):
        B.big_spLinReg(X[:, 0].copy(), y, K=3)
    with pytest.raises(B.BsgError):
        B.big_spLinReg(X, y, ind_col=[1, m + 1], K=3)
    with pytest.raises(ValueError):                           # predict: a non-finite value on a kept column
        mod = B.big_spLinReg(X, y, K=3, nlambda=5)
        Xn = X.copy(order="F")
        Xn[0, mod.ind_col[0] - 1] = np.nan
        mod.predict(Xn)


def test_device_memory_shortfall_is_refused_before_allocation(B):
    """A declared 1,000,000 x 20,000 double matrix (160 GB staged) over a buffer that is never read: BSG_ERR_ALLOC with
    the bytes needed, before anything is allocated or read."""
    from bigsnpr_b200 import _lib

    nr, nc, F, nl = 1_000_000, 20_000, 2, 5
    tiny = np.zeros(1)
    y = np.zeros(nr)
    sets = (np.arange(nr) % 2 + 1).astype(np.int32)
    al = np.array([1.0])
    D = lambda a: a.ctypes.data_as(_lib.c_dbl_p)  # noqa: E731
    I = lambda a: a.ctypes.data_as(_lib.c_int_p)  # noqa: E731
    center, scale, kept = np.zeros(nc), np.zeros(nc), np.zeros(nc, dtype=np.uint8)
    beta, b0 = np.zeros(F * nc), np.zeros(F)
    best, length, msg = (np.zeros(F, dtype=np.int32) for _ in range(3))
    lam, loss = np.zeros(F * nl), np.zeros(F * nl)
    nnz, npass = np.zeros(F * nl, dtype=np.int32), np.zeros(F * nl, dtype=np.int32)
    rc = _lib.lib().bsg_splreg_dense(C.c_void_p(tiny.ctypes.data), 1, nr, nr, nc, None, nr, None, nc, 0, 0, D(y), None,
                                     0, None, None, None, D(al), 1, I(sets), 2, nl, 0.01, 1, 1, 100, 1e-5, 10, 1.0, 0.0,
                                     D(center), D(scale), kept.ctypes.data_as(_lib.c_u8_p), D(beta), D(b0), I(best),
                                     I(length), I(msg), D(lam), D(loss), I(nnz), I(npass), None, None)
    assert rc == 7  # BSG_ERR_ALLOC
    err = _lib.lib().bsg_last_error().decode()
    assert "bytes of device memory" in err and "160000080000 bytes staged" in err, err
