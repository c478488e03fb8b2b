"""CPU checks of the big_spLinReg / big_spLogReg restatement (tests/splreg_ref.py), independent of its summation order:
the 256-slot sum against its explicit loop; the KKT conditions of the stated objective at every lambda of every fit,
from a plain fp64 gradient of the dense decoded matrix; the objective against a long FISTA run; the lasso and ridge
closed forms on an orthogonal design; and every stop reason."""
import os

import numpy as np
import pytest

from tests import gwas_ref as G
from tests import splreg_ref as S

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
N, M = 517, 4542


@pytest.fixture(scope="module")
def codes():
    return G.read_bed_codes(os.path.join(GOLDEN, "example.bed"), N, M)


def _problem(codes, seed, nc=120, family=0):
    rng = np.random.default_rng(seed)
    cols = rng.choice(M, nc, replace=False)
    X = codes[:, cols].astype(np.float64)
    X[codes[:, cols] == 3] = 0.0
    eff = np.zeros(nc)
    eff[:6] = rng.normal(size=6)
    lin = (X - X.mean(0)) @ eff
    y = lin + rng.normal(size=N) if family == 0 else (rng.random(N) < 1 / (1 + np.exp(-lin))).astype(np.float64)
    return X, y, rng


def _std(X, cov, res):
    Xall = X if cov is None else np.column_stack([X, cov])
    cols = np.concatenate([np.flatnonzero(res["kept"]), X.shape[1] + np.arange(0 if cov is None else cov.shape[1])])
    return (Xall[:, cols] - res["center"][cols]) / res["scale"][cols]


def _kkt_violation(Xt, y, base, pf, alpha, lam, b0, beta, train, family):
    """max over columns of the KKT residual of (1/n) loss + lam sum pf (alpha |b| + (1 - alpha) / 2 b^2), plain fp64."""
    Xn, yn, bn = Xt[train], y[train], base[train]
    eta = bn + b0 + Xn @ beta
    res = yn - eta if family == 0 else yn - 1 / (1 + np.exp(-eta))
    g = Xn.T @ res / train.size
    g_int = res.mean()
    ridge = lam * (1 - alpha) * pf * beta
    l1 = lam * alpha * pf
    nz = beta != 0
    v = np.where(nz, np.abs(g - ridge - l1 * np.sign(beta)), np.maximum(np.abs(g) - l1, 0.0))
    return max(v.max(initial=0.0), abs(g_int))


def test_s256_is_the_loop():
    rng = np.random.default_rng(0)
    for n in (1, 255, 256, 257, 3000):
        v = rng.standard_normal((n, 3)) * np.exp(8 * rng.standard_normal((n, 3)))
        assert np.array_equal(S.seg256(v), S.s256_loop(v))
        assert np.array_equal(S.seg256(v[:, 0]), S.s256_loop(v[:, 0]))
    v = rng.standard_normal(3 * S.SEG + 5)
    want = S.s256_loop(v[:S.SEG]) + S.s256_loop(v[S.SEG:2 * S.SEG]) + S.s256_loop(v[2 * S.SEG:3 * S.SEG])
    assert S.s256(v) == want + S.s256_loop(v[3 * S.SEG:])


CASES = [
    # family, Kc, base, pf zeros, alphas, repeats
    (0, 0, False, False, (1.0,), False),
    (0, 10, True, True, (1.0, 0.5, 1e-4), True),
    (1, 0, False, False, (1.0, 0.5), False),
    (1, 10, True, True, (1.0, 1e-4), True),
]


@pytest.mark.parametrize("family,Kc,use_base,pf0,alphas,repeats", CASES)
def test_kkt_certificates(codes, family, Kc, use_base, pf0, alphas, repeats):
    """At every lambda of every fit the KKT conditions hold on the fold's training rows.  The solver stops when the
    largest coordinate change of a pass is at most eps * max |coef|, so the gradient is off by a few such steps times
    the column norms: tolerance 20 eps max(1, max |coef|)."""
    X, y, rng = _problem(codes, 1 + family + Kc, family=family)
    if repeats:
        idx = np.concatenate([np.arange(N), rng.choice(N, 60)])
        X, y = X[idx], y[idx]
    nr = X.shape[0]
    cov = rng.normal(size=(nr, Kc)) if Kc else None
    base = 0.3 * rng.normal(size=nr) if use_base else None
    pfx = np.ones(X.shape[1])
    if pf0:
        pfx[:3] = 0.0
    pfc = np.zeros(Kc) if (pf0 and Kc) else None
    K = 4
    sets = S.folds_from_seed(nr, K, 5)
    eps = 1e-7
    res = S.splreg(X, y, family, sets, K, covar=cov, base=base, pf_X=pfx, pf_covar=pfc, alphas=alphas, nlambda=25,
                   lambda_min_ratio=1e-2, nlam_min=5, n_abort=4, eps=eps, keep_path=True)
    Xt = _std(X, cov, res)
    pf = np.concatenate([pfx[res["kept"]], np.ones(Kc) if pfc is None else pfc])
    b = np.zeros(nr) if base is None else base
    f = 0
    for a in alphas:
        for k in range(1, K + 1):
            fit = res["fits"][f]
            train = np.flatnonzero(sets != k)
            for i in range(fit["length"]):
                beta, b0 = fit["pbeta"][i], fit["pb0"][i]
                tol = 20 * eps * max(1.0, np.abs(beta).max(), abs(b0))
                v = _kkt_violation(Xt, y, b, pf, a, fit["lam"][i], b0, beta, train, family)
                assert v <= tol, (a, k, i, v, tol)
            assert fit["message"] in (0, 1, 2)
            f += 1


def _objective(Xn, yn, b0, beta, lam, alpha, pf, family):
    eta = b0 + Xn @ beta
    if family == 0:
        loss = 0.5 * np.mean((yn - eta) ** 2)
    else:
        loss = np.mean(np.logaddexp(0, eta) - yn * eta)
    return loss + lam * np.sum(pf * (alpha * np.abs(beta) + (1 - alpha) / 2 * beta ** 2))


def _fista(Xn, yn, lam, alpha, pf, family, iters=20000):
    n, p = Xn.shape
    A = np.column_stack([np.ones(n), Xn])
    L = np.linalg.norm(A, 2) ** 2 / n * (1.0 if family == 0 else 0.25)
    w = np.zeros(p + 1)
    z, t = w.copy(), 1.0
    pfe = np.concatenate([[0.0], pf])
    for _ in range(iters):
        eta = A @ z
        r = (eta - yn) if family == 0 else (1 / (1 + np.exp(-eta)) - yn)
        g = A.T @ r / n
        u = z - g / L
        wn = np.sign(u) * np.maximum(np.abs(u) - lam * alpha * pfe / L, 0) / (1 + lam * (1 - alpha) * pfe / L)
        tn = (1 + np.sqrt(1 + 4 * t * t)) / 2
        z = wn + (t - 1) / tn * (wn - w)
        w, t = wn, tn
    return w


@pytest.mark.parametrize("family", [0, 1])
def test_objective_matches_fista(codes, family):
    X, y, rng = _problem(codes, 40 + family, nc=200, family=family)
    X, y = X[:500], y[:500]
    sets = S.folds_from_seed(500, 2, 3)
    alpha = 0.5
    res = S.splreg(X, y, family, sets, 2, alphas=(alpha,), nlambda=12, lambda_min_ratio=0.05, nlam_min=12, n_abort=12,
                   eps=1e-12, keep_path=True)
    Xt = _std(X, None, res)
    fit = res["fits"][0]
    train = np.flatnonzero(sets != 1)
    pf = np.ones(Xt.shape[1])
    for i in (2, 6, fit["length"] - 1):
        lam = fit["lam"][i]
        ours = _objective(Xt[train], y[train], fit["pb0"][i], fit["pbeta"][i], lam, alpha, pf, family)
        w = _fista(Xt[train], y[train], lam, alpha, pf, family)
        theirs = _objective(Xt[train], y[train], w[0], w[1:], lam, alpha, pf, family)
        assert ours <= theirs * (1 + 1e-8), (i, ours, theirs)
        assert abs(ours - theirs) <= 1e-8 * abs(theirs), (i, ours, theirs)


@pytest.mark.parametrize("alpha", [1.0, 1e-4])
def test_orthogonal_closed_forms(alpha):
    """Columns orthonormal (x'x / n = 1, mean 0) on the training rows: beta_j = soft(z_j, lam alpha) / (1 + lam (1 -
    alpha)) with z_j = x_j'y / n, the lasso (alpha = 1) and nearly ridge (alpha = 1e-4) closed forms."""
    n, p = 256, 16
    H = np.array([[1.0]])
    while H.shape[0] < n:
        H = np.block([[H, H], [H, -H]])
    Xt = H[:, 1:p + 1]  # orthogonal, mean 0, x'x / n = 1
    rng = np.random.default_rng(9)
    y = Xt @ np.linspace(-2, 2, p) + rng.normal(size=n) + 3.0
    Xv = rng.normal(size=(20, p))  # held-out rows
    yv = rng.normal(size=20)
    Xall, yall = np.vstack([Xt, Xv]), np.concatenate([y, yv])
    train, val = np.arange(n), n + np.arange(20)
    out = S.fit_path(Xall, yall, np.zeros(n + 20), np.ones(p), alpha, train, val, 0, 15, 0.8, 15, 15, 10 ** 6, 1e-13,
                     1000, keep_path=True)
    z = Xt.T @ y / n
    for i in range(out["length"]):
        lam = out["lam"][i]
        want = np.sign(z) * np.maximum(np.abs(z) - lam * alpha, 0) / (1 + lam * (1 - alpha))
        np.testing.assert_allclose(out["pbeta"][i], want, rtol=0, atol=1e-11)
        assert abs(out["pb0"][i] - y.mean()) < 1e-11
    assert abs(out["lam"][0] - np.abs(z).max() / alpha) <= 1e-12 * out["lam"][0]


def test_stop_reasons(codes):
    X, y, _ = _problem(codes, 7, nc=150)
    sets = S.folds_from_seed(N, 3, 1)
    full = S.splreg(X, y, 0, sets, 3, nlambda=8, lambda_min_ratio=0.3, nlam_min=8, n_abort=20)
    assert all(f["message"] == 0 and f["length"] == 8 for f in full["fits"])
    many = S.splreg(X, y, 0, sets, 3, nlambda=60, lambda_min_ratio=1e-3, nlam_min=2, n_abort=60, dfmax=5)
    assert all(f["message"] == 2 and f["length"] < 60 for f in many["fits"])
    assert all(f["nnz"][-1] > 5 >= max(f["nnz"][:-1], default=0) for f in many["fits"])
    noimp = S.splreg(X, y, 0, sets, 3, nlambda=80, lambda_min_ratio=1e-4, nlam_min=5, n_abort=3)
    for f in noimp["fits"]:
        assert f["message"] == 1 and f["length"] - 1 - f["best"] == 3
        assert f["loss"][f["best"]] == min(f["loss"])


ORACLE_CASES = CASES + [
    (0, 0, False, False, (0.5,), False, dict(dfmax=4)),
    (0, 0, False, False, (1.0,), False, dict(nlambda=80, lambda_min_ratio=1e-4, nlam_min=5, n_abort=3)),
    (1, 0, False, False, (1.0,), False, dict(nlambda=6, nlam_min=6, n_abort=10)),
]


def _same_fits(a, b):
    assert np.array_equal(a["kept"], b["kept"]) and a["J"] == b["J"]
    for fa, fb in zip(a["fits"], b["fits"]):
        for key in ("best", "length", "message", "nnz", "npass"):
            assert fa[key] == fb[key], key
        for key in ("lam", "loss", "pb0"):
            assert np.array_equal(np.asarray(fa[key]).view(np.int64), np.asarray(fb[key]).view(np.int64)), key
        assert np.array_equal(fa["beta"].view(np.int64), fb["beta"].view(np.int64))
        assert np.float64(fa["b0"]).view(np.int64) == np.float64(fb["b0"]).view(np.int64)
        assert np.array_equal(np.asarray(fa["pbeta"]).view(np.int64), np.asarray(fb["pbeta"]).view(np.int64))


@pytest.mark.parametrize("case", ORACLE_CASES)
def test_c_oracle_is_the_restatement(codes, case):
    """tests/splreg_oracle.c against the NumPy restatement, byte for byte, on example.bed: linear and logistic, 0 / 10
    covariates, base, zero penalty factors, alpha in {1, 0.5, 1e-4}, repeated rows and every stop reason."""
    family, Kc, use_base, pf0, alphas, repeats = case[:6]
    extra = case[6] if len(case) > 6 else {}
    X, y, rng = _problem(codes, 60 + family + Kc, family=family)
    if repeats:
        idx = np.concatenate([np.arange(N), rng.choice(N, 60)])
        X, y = X[idx], y[idx]
    nr = X.shape[0]
    cov = rng.normal(size=(nr, Kc)) if Kc else None
    base = 0.3 * rng.normal(size=nr) if use_base else None
    pfx = np.ones(X.shape[1])
    if pf0:
        pfx[:3] = 0.0
    pfc = np.zeros(Kc) if (pf0 and Kc) else None
    kw = dict(dict(nlambda=25, lambda_min_ratio=1e-2, nlam_min=5, n_abort=4), **extra)
    sets = S.folds_from_seed(nr, 4, 8)
    args = (X, y, family, sets, 4)
    opts = dict(covar=cov, base=base, pf_X=pfx, pf_covar=pfc, alphas=alphas, keep_path=True,
                col_key=rng.permutation(X.shape[1]), **kw)
    a, b = S.splreg(*args, **opts), S.splreg(*args, engine="c", **opts)
    _same_fits(a, b)
    if "dfmax" in extra:
        assert all(f["message"] == 2 for f in a["fits"])
    elif extra.get("nlambda") == 6:
        assert all(f["message"] == 0 for f in a["fits"])
    elif "n_abort" in extra:
        assert all(f["message"] == 1 for f in a["fits"])


def test_c_oracle_segments():
    """More than one 8,192-row segment: the segmented sums of the C oracle and of NumPy agree."""
    rng = np.random.default_rng(4)
    nr, p = 2 * S.SEG + 300, 12
    X = rng.integers(0, 3, size=(nr, p)).astype(np.float64)
    y = X[:, :3] @ np.array([0.5, -0.3, 0.2]) + rng.normal(size=nr)
    sets = S.folds_from_seed(nr, 2, 1)
    opts = dict(alphas=(1.0, 0.5), nlambda=10, lambda_min_ratio=1e-2, nlam_min=10, n_abort=10, keep_path=True)
    _same_fits(S.splreg(X, y, 0, sets, 2, **opts), S.splreg(X, y, 0, sets, 2, engine="c", **opts))
    yb = (y > 0).astype(np.float64)
    _same_fits(S.splreg(X, yb, 1, sets, 2, **opts), S.splreg(X, yb, 1, sets, 2, engine="c", **opts))
