"""big_spLinReg / big_spLogReg on the device (bsg_splreg) against the restatement of tests/splreg_ref.py, byte for byte:
column statistics, kept columns, every fit's path (lambda, validation loss, nonzero count, passes, coefficients), stop
messages, best lambdas, the averaged model and the chosen alpha -- on example.bed (linear and logistic, 0 / 10
covariates, base, zero penalty factors, three alphas, repeated rows, every stop reason), example-missing.bed (refused,
then its imputed FBM twin), a dosage FBM and an LD-structured 100,000-row matrix with 10 PCs.  Also the KKT
certificates of the device's own paths, determinism under column permutation and other alphas in the call, predict,
and the refusals."""
import os

import numpy as np
import pytest

from tests import gwas_ref as G
from tests import splreg_ref as S
from tests.test_splreg_oracle import _kkt_violation

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
N, M = 517, 4542
NM, MM = 200, 500


@pytest.fixture(scope="module")
def B():
    import bigsnpr_b200 as B

    return B


@pytest.fixture(scope="module")
def codes():
    return G.read_bed_codes(os.path.join(GOLDEN, "example.bed"), N, M)


def _bytes(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.array_equal(a.view(np.int64), b.view(np.int64))


def _same(B, mod, ref, A, K):
    J = ref["J"]
    assert np.array_equal(mod.raw["beta"].shape, (A, K, J))
    for a in range(A):
        for k in range(K):
            r = ref["fits"][a * K + k]
            p = mod.path[a][k]
            assert mod.raw["length"][a, k] == r["length"] and mod.raw["message"][a, k] == r["message"]
            assert mod.raw["best"][a, k] == r["best"]
            _bytes(p["lambda_"], r["lam"])
            _bytes(p["loss"], r["loss"])
            assert np.array_equal(p["nnz"], r["nnz"]) and np.array_equal(p["passes"], r["npass"])
            _bytes(mod.raw["beta"][a, k], r["beta"])
            _bytes(mod.raw["b0"][a, k], r["b0"])
            if "beta" in p:
                _bytes(p["beta"], np.array(r["pbeta"]).reshape(-1, J))
                _bytes(p["intercept"], r["pb0"])
    ob, oi = B.api.splreg_unscale(
        np.array([[r["beta"] for r in ref["fits"][a * K:(a + 1) * K]] for a in range(A)]),
        np.array([[r["b0"] for r in ref["fits"][a * K:(a + 1) * K]] for a in range(A)]),
        ref["center"][_cols(ref)], ref["scale"][_cols(ref)])
    _bytes(mod.beta, ob)
    _bytes(mod.intercept, oi)
    vl = np.array([np.mean([r["loss"][r["best"]] for r in ref["fits"][a * K:(a + 1) * K]]) for a in range(A)])
    _bytes(mod.validation_loss, vl)
    assert mod.best_alpha == int(np.argmin(vl))


def _cols(ref):
    nc = ref["kept"].size
    Kc = ref["J"] - int(ref["kept"].sum())
    return np.concatenate([np.flatnonzero(ref["kept"]), nc + np.arange(Kc)])


def _run(B, X, vals, rows, cols, y, family, D=1, covar=None, base=None, pf_X=None, pf_covar=None, alphas=(1.0,), K=4,
         seed=3, path=True, **kw):
    fn = B.big_spLogReg if family else B.big_spLinReg
    mod = fn(X, y, ind_train=rows, ind_col=cols, covar_train=covar, base_train=base, pf_X=pf_X, pf_covar=pf_covar,
             alphas=alphas, K=K, seed=seed, return_path=path, **kw)
    Xd = vals[np.ix_(np.asarray(rows) - 1, np.asarray(cols) - 1)].astype(np.float64) / D
    sets = S.folds_from_seed(len(rows), K, seed)
    assert np.array_equal(mod.ind_sets, sets)
    ref = S.splreg(Xd, y, family, sets, K, covar=covar, base=base, pf_X=pf_X, pf_covar=pf_covar, alphas=alphas,
                   keep_path=path, col_key=np.asarray(cols), **kw)
    assert np.array_equal(mod.ind_col, np.asarray(cols)[ref["kept"]])
    _bytes(mod.center, ref["center"][_cols(ref)])
    _bytes(mod.scale, ref["scale"][_cols(ref)])
    _same(B, mod, ref, len(alphas), K)
    return mod, ref, Xd, sets


def _pheno(rng, Xd, family, nca=8):
    eff = np.zeros(Xd.shape[1])
    eff[rng.choice(Xd.shape[1], nca, replace=False)] = rng.normal(size=nca)
    lin = (Xd - Xd.mean(0)) @ eff
    lin = lin / max(np.std(lin), 1e-12)
    if family == 0:
        return lin + rng.normal(size=lin.size)
    return (rng.random(lin.size) < 1 / (1 + np.exp(-lin))).astype(np.float64)


PATH = dict(nlambda=30, lambda_min_ratio=1e-2, nlam_min=10, n_abort=5)
CASES = [
    (0, 0, False, False, (1.0,), False, {}),
    (0, 10, True, True, (1.0, 0.5, 1e-4), True, {}),
    (1, 0, False, False, (1.0, 0.5), False, {}),
    (1, 10, True, True, (1.0, 1e-4), True, {}),
    (0, 0, False, False, (0.5,), False, dict(dfmax=4)),
    (1, 0, False, False, (1.0,), False, dict(nlambda=6, nlam_min=6, n_abort=10)),
    (0, 0, False, False, (1.0,), False, dict(nlambda=80, lambda_min_ratio=1e-4, nlam_min=5, n_abort=3)),
]


@pytest.mark.parametrize("family,Kc,use_base,pf0,alphas,repeats,extra", CASES)
def test_example_bed(B, codes, family, Kc, use_base, pf0, alphas, repeats, extra):
    rng = np.random.default_rng(family * 10 + Kc + len(alphas))
    X = B.Bed(os.path.join(GOLDEN, "example.bed"))
    cols = np.sort(rng.choice(M, 300, replace=False)) + 1
    ok = (codes[:, cols - 1] != 3).all(axis=0)
    cols = cols[ok]
    rows = np.arange(1, N + 1)
    if repeats:
        rows = np.concatenate([rows, rng.choice(N, 50) + 1])
    nr = rows.size
    y = _pheno(rng, codes[np.ix_(rows - 1, cols - 1)].astype(float), family)
    covar = rng.normal(size=(nr, Kc)) if Kc else None
    base = 0.2 * rng.normal(size=nr) if use_base else None
    pf_X = None
    if pf0:
        pf_X = np.ones(cols.size)
        pf_X[:2] = 0.0
    pf_covar = np.zeros(Kc) if (pf0 and Kc) else None
    kw = dict(PATH, **extra)
    mod, ref, Xd, sets = _run(B, X, codes, rows, cols, y, family, covar=covar, base=base, pf_X=pf_X, pf_covar=pf_covar,
                              alphas=alphas, **kw)
    if "dfmax" in extra:
        assert (mod.raw["message"] == 2).all()
    elif extra.get("nlambda") == 6:
        assert (mod.raw["message"] == 0).all()
    elif "n_abort" in extra:
        assert (mod.raw["message"] == 1).all()
    # KKT certificates on the device's own paths, plain fp64 from the dense matrix
    Xall = Xd if covar is None else np.column_stack([Xd, covar])
    Xt = (Xall[:, _cols(ref)] - mod.center) / mod.scale
    pf = np.concatenate([np.ones(mod.ind_col.size) if pf_X is None else pf_X[ref["kept"]],
                         np.ones(Kc) if pf_covar is None else pf_covar])
    b = np.zeros(nr) if base is None else base
    for a, al in enumerate(alphas):
        for k in range(4):
            p = mod.path[a][k]
            train = np.flatnonzero(sets != k + 1)
            for i in range(p["lambda_"].size):
                beta = p["beta"][i]
                tol = 20 * 1e-5 * max(1.0, np.abs(beta).max(), abs(p["intercept"][i]))
                assert _kkt_violation(Xt, y, b, pf, al, p["lambda_"][i], p["intercept"][i], beta, train, family) <= tol
    # predict: the host product of the returned beta
    pred = mod.predict(X, rows, covar, base_row=base)
    i = mod.best_alpha
    host = Xd @ mod.beta[i][:mod.ind_col.size] + mod.intercept[i] + (0 if base is None else base)
    if Kc:
        host = host + covar @ mod.beta[i][mod.ind_col.size:]
    np.testing.assert_allclose(pred, host, rtol=1e-10, atol=1e-10 * np.abs(host).max())


def test_missing_refused_then_imputed_twin(B):
    X = B.Bed(os.path.join(GOLDEN, "example-missing.bed"))
    cm = G.read_bed_codes(os.path.join(GOLDEN, "example-missing.bed"), NM, MM)
    rng = np.random.default_rng(21)
    y = rng.normal(size=NM)
    with pytest.raises(B.BsgError):
        B.big_spLinReg(X, y, K=4)
    imp = cm.copy()
    imp[imp == 3] = 4  # CODE_IMPUTE_PRED: bytes 4..6 read as 0..2; each missing call imputed as 0
    code256 = np.full(256, np.nan)
    code256[:3] = [0, 1, 2]
    code256[4:7] = [0, 1, 2]
    F = B.Bed.from_fbm(imp.astype(np.uint8), code256)
    vals = np.where(imp == 4, 0, imp)
    cols = np.arange(1, MM + 1)
    mod = _run(B, F, vals, np.arange(1, NM + 1), cols, y, 0, **PATH)[0]
    with pytest.raises(ValueError):  # the .bed itself holds the missing calls: predict refuses them too
        mod.predict(X)


def test_dosage_fbm(B):
    rng = np.random.default_rng(12)
    code256 = np.full(256, np.nan)
    code256[:201] = np.arange(201) / 100
    byt = rng.integers(0, 201, size=(600, 200)).astype(np.uint8)
    F = B.Bed.from_fbm(byt, code256)
    assert F.dosage_scale == 100
    rows = np.arange(1, 601)
    cols = rng.permutation(200) + 1
    y = _pheno(rng, byt[:, cols - 1] / 100.0, 1)
    mod, _, Xd, _ = _run(B, F, byt, rows, cols, y, 1, D=100, alphas=(1.0, 0.5), **PATH)
    i = mod.best_alpha
    np.testing.assert_allclose(mod.predict(F, rows), Xd @ mod.beta[i] + mod.intercept[i], rtol=1e-10, atol=1e-10)
    byt2 = byt.copy()
    byt2[5, mod.ind_col[0] - 1] = 255  # an NA code on a kept column
    F2 = B.Bed.from_fbm(byt2, code256)
    with pytest.raises(ValueError):
        mod.predict(F2, rows)


def test_ld_synthetic_with_pcs(B):
    from tests.synth_ref import synth_matrix_ld

    n, m = 100_000, 2000
    X = B.Bed.synthetic(n, m, seed=77, ld_rho=0.9, ld_block=50)
    vals = synth_matrix_ld(n, m, seed=77, rho=0.9, ld_block=50)
    svd = B.bed_randomSVD(X, k=10)
    pcs = svd["u"] * svd["d"]
    rng = np.random.default_rng(14)
    y = _pheno(rng, vals[:, :400].astype(float), 0, nca=20)
    cols = np.arange(1, m + 1)
    _run(B, X, vals, np.arange(1, n + 1), cols, y, 0, covar=pcs, K=3, path=False, nlambda=20, lambda_min_ratio=0.05,
         nlam_min=20, n_abort=20)


def test_determinism(B, codes):
    rng = np.random.default_rng(31)
    X = B.Bed(os.path.join(GOLDEN, "example.bed"))
    cols = np.sort(rng.choice(M, 200, replace=False)) + 1
    cols = cols[(codes[:, cols - 1] != 3).all(axis=0)]
    y = _pheno(rng, codes[:, cols - 1].astype(float), 1)
    kw = dict(K=4, seed=2, nlambda=25, lambda_min_ratio=1e-2, nlam_min=10, n_abort=5)
    a = B.big_spLogReg(X, y, ind_col=cols, alphas=(1.0, 0.5, 1e-4), **kw)
    b = B.big_spLogReg(X, y, ind_col=cols, alphas=(1.0, 0.5, 1e-4), **kw)
    _bytes(a.raw["beta"], b.raw["beta"])
    one = B.big_spLogReg(X, y, ind_col=cols, alphas=(0.5,), **kw)
    _bytes(one.raw["beta"][0], a.raw["beta"][1])
    _bytes(one.raw["b0"][0], a.raw["b0"][1])
    perm = rng.permutation(cols.size)
    c = B.big_spLogReg(X, y, ind_col=cols[perm], alphas=(0.5,), **kw)
    _bytes(c.raw["b0"][0], one.raw["b0"][0])
    # a column's coefficient does not depend on where it sits: same bytes after undoing the permutation
    _bytes(c.raw["beta"][0][:, np.argsort(perm)], one.raw["beta"][0])


def test_refusals(B, codes):
    X = B.Bed(os.path.join(GOLDEN, "example.bed"))
    y = np.random.default_rng(1).normal(size=N)
    cols = np.arange(1, 30)
    for kw in (dict(power_scale=0.5), dict(power_adaptive=1), dict(alphas=0), dict(alphas=1.5), dict(K=1)):
        with pytest.raises(B.BsgError):
            B.big_spLinReg(X, y, ind_col=cols, **kw)
    with pytest.raises(B.BsgError):
        B.big_spLogReg(X, y, ind_col=cols)
    yb = y.copy()
    yb[3] = np.nan
    with pytest.raises(B.BsgError):
        B.big_spLinReg(X, yb, ind_col=cols)
    with pytest.raises(B.BsgError) as e:
        B.big_spLinReg(X, y, ind_col=[1, M + 1])
    assert e.value.code == 2
    code256 = np.full(256, np.nan)
    code256[:3] = [0, 0.1234567, 2]  # not a dosage table: no scale D makes every code an integer byte
    with pytest.raises(B.BsgError) as e:
        B.big_spLinReg(B.Bed.from_fbm(codes, code256), y, ind_col=cols)
    assert e.value.code == 10
