"""CPU restatement of big_univLogReg (bigstatsr's IRLS + R glue, not vendored in the reference): the definition the device
path (bsg_univlogreg, bigsnpr_b200/csrc/bsg_logreg.cu) is held to.

- `glm_fit`: R's glm.fit for family = binomial() (logit link): the null model of step 1 and the refit of step 3.
- `irls`: step 2 on a dense matrix, vectorised over SNPs: from beta = (gamma0, 0), H = A'WA and r = A'W z with
  A = [U, x], beta_new = H^-1 r, until max |beta_new - beta| < tol or maxiter steps; std.err from the last H solved.
- `univlogreg`: the whole statistic (basis, null model, IRLS, refit of the SNPs that did not meet tol).
- `newton_mle`: the fully converged maximum-likelihood fit of one SNP (Newton to 1e-14), for the accuracy checks.
NaN estim / std.err (niter 0, never refitted) for a column with an NA value or constant over the rows, or an H that is
not positive definite.
"""
from __future__ import annotations

import numpy as np

THRESH, MTHRESH = 30.0, -30.0
EPS = np.finfo(np.float64).eps


def covar_basis(covar, n, thr_eigval=1e-4):
    """The R glue's U (as bigsnpr_b200.api.univlinreg_covar_basis, restated without the package)."""
    cols = [np.ones(n)]
    if covar is not None:
        cv = np.asarray(covar, dtype=np.float64)
        cols.append(cv.reshape(n, -1) if cv.ndim == 1 else cv)
    C = np.column_stack(cols)
    u, d, _ = np.linalg.svd(C, full_matrices=False)
    return u[:, d / (np.sqrt(n) + np.sqrt(C.shape[1]) - 1) > thr_eigval]


def glm_fit(A, y, eps=1e-8, maxit=25):
    """glm.fit(A, y, family = binomial()): mustart = (y + 0.5) / 2; per iteration z = eta + (y - mu) / mu.eta,
    w = sqrt(mu.eta^2 / var(mu)), least squares of z w on A w; stop when |dev - devold| / (|dev| + 0.1) < eps.  The logit
    link's clamps (eta beyond +-30) as in R's C code.  Returns (coef, se, iterations, converged); se from the last fit."""
    A = np.asarray(A, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    mu = (y + 0.5) / 2
    eta = np.log(mu / (1 - mu))

    def dev_of(mu):
        return 2 * np.sum(np.where(y == 1, -np.log(mu), -np.log1p(-mu)))

    devold = dev_of(mu)
    conv, it, coef, Aw = False, 0, None, A
    for it in range(1, maxit + 1):
        with np.errstate(over="ignore"):
            e = np.exp(eta)
        me = np.where((eta > THRESH) | (eta < MTHRESH), EPS, e / ((1 + e) * (1 + e)))
        z = eta + (y - mu) / me
        w = np.sqrt(me ** 2 / (mu * (1 - mu)))
        Aw = A * w[:, None]
        coef = np.linalg.lstsq(Aw, z * w, rcond=None)[0]
        eta = A @ coef
        t = np.where(eta < MTHRESH, EPS, np.where(eta > THRESH, 1 / EPS, np.exp(np.clip(eta, MTHRESH, THRESH))))
        mu = t / (1 + t)
        dev = dev_of(mu)
        if abs(dev - devold) / (abs(dev) + 0.1) < eps:
            conv = True
            break
        devold = dev
    with np.errstate(invalid="ignore"):
        se = np.sqrt(np.diag(np.linalg.pinv(Aw.T @ Aw)))
    return coef, se, it, conv


def irls(Xd, y, U, gamma0, tol=1e-8, maxiter=20, block=512):
    """Step 2 on the dense nr x m matrix Xd of the training observations (NaN = NA).  Returns a dict: estim, std_err,
    niter (steps taken), converged (tol met), steps (m x maxiter step sizes max |beta_new - beta_old|, NaN past the end)."""
    Xd = np.asarray(Xd, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    nr, m = Xd.shape
    K = U.shape[1]
    P = K + 1
    UU = (U[:, :, None] * U[:, None, :]).reshape(nr, K * K)
    out = dict(estim=np.full(m, np.nan), std_err=np.full(m, np.nan), niter=np.zeros(m, dtype=np.int64),
               converged=np.zeros(m, dtype=bool), steps=np.full((m, maxiter), np.nan))
    bad = np.isnan(Xd).any(axis=0) | np.all(Xd == Xd[:1], axis=0)
    for b0 in range(0, m, block):
        idx = np.arange(b0, min(m, b0 + block))
        idx = idx[~bad[idx]]
        if not idx.size:
            continue
        X = Xd[:, idx]
        beta = np.zeros((idx.size, P))
        beta[:, :K] = gamma0
        active = np.ones(idx.size, dtype=bool)
        for it in range(1, maxiter + 1):
            a = np.flatnonzero(active)
            if not a.size:
                break
            x = X[:, a]
            eta = U @ beta[a, :K].T + x * beta[a, K]
            p = 1 / (1 + np.exp(-eta))
            w = p * (1 - p)
            wz = w * eta + (y[:, None] - p)  # W z with z = eta + (y - p) / w
            H = np.empty((a.size, P, P))
            H[:, :K, :K] = (UU.T @ w).T.reshape(a.size, K, K)
            H[:, :K, K] = H[:, K, :K] = (U.T @ (w * x)).T
            H[:, K, K] = np.einsum("ij,ij->j", w * x, x)
            r = np.empty((a.size, P))
            r[:, :K] = (U.T @ wz).T
            r[:, K] = np.einsum("ij,ij->j", wz, x)
            for t, j in enumerate(a):
                try:
                    L = np.linalg.cholesky(H[t])
                except np.linalg.LinAlgError:
                    L = None
                if L is None or not np.all(np.isfinite(L)):
                    active[j] = False
                    out["niter"][idx[j]] = 0
                    continue
                bn = np.linalg.solve(L.T, np.linalg.solve(L, r[t]))
                if not np.all(np.isfinite(bn)):
                    active[j] = False
                    continue
                diff = np.max(np.abs(bn - beta[j]))
                beta[j] = bn
                k = idx[j]
                out["steps"][k, it - 1] = diff
                if diff < tol or it == maxiter:
                    active[j] = False
                    out["estim"][k] = bn[K]
                    out["std_err"][k] = 1 / L[K, K]
                    out["niter"][k] = it
                    out["converged"][k] = diff < tol
    return out


def univlogreg(Xd, y01, covar=None, tol=1e-8, maxiter=20, U=None):
    """big_univLogReg on the dense matrix Xd of the training observations: basis, null model, IRLS, refit.  Returns the
    irls dict plus score, refitted and U / gamma0."""
    nr = Xd.shape[0]
    if U is None:
        U = covar_basis(covar, nr)
    gamma0 = glm_fit(U, y01)[0]
    res = irls(Xd, y01, U, gamma0, tol, maxiter)
    ok = ~np.isnan(res["estim"])
    refit = ok & ~res["converged"]
    for j in np.flatnonzero(refit):
        coef, se, it, _ = glm_fit(np.column_stack([U, Xd[:, j]]), y01)
        res["estim"][j], res["std_err"][j], res["niter"][j] = coef[-1], se[-1], it
    res["refitted"] = refit
    res["score"] = res["estim"] / res["std_err"]
    res["U"], res["gamma0"] = U, gamma0
    return res


def newton_mle(A, y, tol=1e-14, maxiter=100):
    """The maximum-likelihood fit of the logistic regression of y on A by Newton steps until max |step| < tol.  Returns
    (coef, se) with se from the Hessian at the optimum."""
    beta = np.zeros(A.shape[1])
    for _ in range(maxiter):
        p = 1 / (1 + np.exp(-(A @ beta)))
        H = (A * (p * (1 - p))[:, None]).T @ A
        step = np.linalg.solve(H, A.T @ (y - p))
        beta = beta + step
        if np.max(np.abs(step)) < tol:
            break
    p = 1 / (1 + np.exp(-(A @ beta)))
    H = (A * (p * (1 - p))[:, None]).T @ A
    return beta, np.sqrt(np.diag(np.linalg.inv(H)))


def read_fam_affection(path):
    """The .fam file's phenotype column (1 = control, 2 = case)."""
    return np.loadtxt(path, dtype=str)[:, 5].astype(int)
