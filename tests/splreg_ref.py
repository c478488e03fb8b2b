"""Restatement of big_spLinReg / big_spLogReg (bigstatsr's elastic net with cross-model selection and averaging,
power_scale = 1, power_adaptive = 0) -- the definition the device (bsg_splreg, DESIGN.md section 4.19) reproduces byte
for byte.

bigstatsr is not vendored in the reference; this follows its documentation and Prive, Aschard & Blum (2019, Genetics
212:65-74).  The points where the restatement had to choose are marked (unconfirmed) in DESIGN.md section 4.19.

Arithmetic: NumPy fp64, one rounding per operation (no fused multiply-add), exp / log from the fdlibm restatement shared
with LDpred2 (tests/ldpred2_auto_ref.py), and every sum over observations the 256-slot sum ``s256``.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tests import ldpred2_auto_ref as LA

ST = 256
SEG = 8192
W_MIN = 1e-5
SD_MIN = 1e-8
MESSAGES = ("Complete path", "No more improvement", "Too many variables")


def s256(v):
    """Sum over axis 0 in the fixed order of the device: the positions are cut into segments of SEG = 8192, and the
    segment sums are added in segment order (left to right).  Within a segment, slot t (0..255) adds positions t,
    t + 256, t + 512, ... in order from +0, then slots are halved pairwise, t += t + h for h = 128, 64, ..., 1 (the
    256-slot sum, ``seg256``)."""
    v = np.asarray(v, dtype=np.float64)
    tot = None
    for b in range(0, max(v.shape[0], 1), SEG):
        part = seg256(v[b:b + SEG])
        tot = part if tot is None else tot + part
    return tot


def seg256(v):
    """The 256-slot sum over axis 0.  (NumPy's reduction over the leading axis of a C-contiguous array adds rows in
    order; test_splreg_oracle checks it against an explicit loop.)"""
    v = np.asarray(v, dtype=np.float64)
    n = v.shape[0]
    m = max(1, -(-n // ST))
    p = np.zeros((m * ST,) + v.shape[1:])
    p[:n] = v
    acc = p.reshape((m, ST) + v.shape[1:]).sum(axis=0)
    h = ST // 2
    while h >= 1:
        acc = acc[:h] + acc[h:2 * h]
        h //= 2
    return acc[0]


def s256_loop(v):
    """seg256 by an explicit loop over the 256-row chunks (the definition, slow)."""
    v = np.asarray(v, dtype=np.float64)
    n = v.shape[0]
    acc = np.zeros((ST,) + v.shape[1:])
    for c in range(0, n, ST):
        blk = np.zeros((ST,) + v.shape[1:])
        blk[:min(ST, n - c)] = v[c:c + ST]
        acc = acc + blk
    h = ST // 2
    while h >= 1:
        acc = acc[:h] + acc[h:2 * h]
        h //= 2
    return acc[0]


def _soft(u, t):
    return u - t if u > t else (u + t if u < -t else 0.0)


def prob(eta):
    return 1.0 / (1.0 + LA.exp(-np.asarray(eta, dtype=np.float64)))


def binom_loss(eta, y):
    """log(1 + e^eta) - y eta per observation, as the device evaluates it."""
    eta = np.asarray(eta, dtype=np.float64)
    pos = eta > 0
    l = np.where(pos, eta + LA.log(1.0 + LA.exp(-np.abs(eta))), LA.log(1.0 + LA.exp(np.minimum(eta, 0.0))))
    # the two branches evaluate exactly the device's expressions: exp(-eta) for eta > 0, exp(eta) otherwise
    return l - y * eta


def column_stats(Xall):
    """centre and sd (divisor nr) of every column over all observations, by 256-slot sums."""
    nr = Xall.shape[0]
    c = s256(Xall) / float(nr)
    d = Xall - c
    return c, np.sqrt(s256(d * d) / float(nr))


def folds_from_seed(n, K, seed):
    """The folds when ind_sets is not given: (a seeded permutation of 0..n-1) mod K, plus 1 (R's sample is not
    reproduced)."""
    return (np.random.default_rng(seed).permutation(n) % K + 1).astype(np.int32)


class _Fit:
    def __init__(self, Xt, y, base, pf, alpha, train, val, family, eps, max_iter):
        self.pos = np.concatenate([train, val])
        self.n, self.nr = train.size, self.pos.size
        self.X = Xt[self.pos]          # standardised values at each position
        self.y = y[self.pos]
        self.pf = pf
        self.alpha, self.oma = alpha, 1.0 - alpha
        self.logit = family == 1
        self.eps, self.max_iter = eps, max_iter
        J = Xt.shape[1]
        self.beta = np.zeros(J)
        self.v = np.full(J, -1.0)
        self.b0 = 0.0
        b = base[self.pos]
        self.R = b.copy() if self.logit else self.y - b
        self.dn = float(self.n)

    def irls_weights(self):
        n = self.n
        p = prob(self.R[:n])
        self.W = np.maximum(p * (1.0 - p), W_MIN)
        self.S = self.y[:n] - p

    def cd_pass(self, lam, ws):
        n = self.n
        la1, la2 = lam * self.alpha, lam * self.oma
        if not self.logit:
            d0 = s256(self.R[:n]) / self.dn
            self.R = self.R - d0
        else:
            self.irls_weights()
            d0 = s256(self.S) / s256(self.W)
            self.R = self.R + d0
            self.S = self.S - self.W * d0
        self.b0 = self.b0 + d0
        maxd = abs(d0)
        maxb = abs(self.b0)
        for j in ws:
            x = self.X[:, j]
            bj = self.beta[j]
            if not self.logit:
                if self.v[j] < 0:
                    self.v[j] = s256(x[:n] * x[:n]) / self.dn
                h = self.v[j]
                g = s256(x[:n] * self.R[:n]) / self.dn
            else:
                g = s256(x[:n] * self.S) / self.dn
                h = s256((self.W * x[:n]) * x[:n]) / self.dn
            pf = self.pf[j]
            u = g + h * bj
            bn = _soft(u, la1 * pf) / (h + la2 * pf)
            d = bn - bj
            if d != 0.0:
                if not self.logit:
                    self.R = self.R - x * d
                else:
                    self.R = self.R + x * d
                    self.S = self.S - (self.W * x[:n]) * d
                self.beta[j] = bn
            maxd = max(maxd, abs(d))
            maxb = max(maxb, abs(bn))
        return maxd <= self.eps * maxb

    def full_pass(self):
        n = self.n
        res = self.y[:n] - prob(self.R[:n]) if self.logit else self.R[:n]
        return s256(self.X[:n] * res[:, None]) / self.dn

    def val_loss(self):
        n, nv = self.n, self.nr - self.n
        if self.logit:
            return 2.0 * (s256(binom_loss(self.R[n:], self.y[n:])) / float(nv))
        r = self.R[n:]
        return s256(r * r) / float(nv)


def fit_path(Xt, y, base, pf, alpha, train, val, family, nlambda, step, nlam_min, n_abort, dfmax, eps, max_iter,
             keep_path=False):
    """One fit (one alpha, one fold) over the lambda path; the device's k_splreg, sequentially."""
    F = _Fit(Xt, y, base, pf, alpha, train, val, family, eps, max_iter)
    J = Xt.shape[1]
    ws_mask = pf == 0.0
    ever = np.zeros(J, dtype=bool)
    ws = np.flatnonzero(ws_mask)
    for _ in range(max_iter):
        if F.cd_pass(0.0, ws):
            break
    z = F.full_pass()
    pen = pf > 0
    lmax = float(np.max(np.abs(z[pen]) / (alpha * pf[pen]))) if pen.any() else 0.0
    lam = lprev = lmax
    out = dict(lam=[], loss=[], nnz=[], npass=[], pbeta=[], pb0=[])
    best_loss, best, stop = np.inf, 0, -1
    bbest, b0best = np.zeros(J), 0.0
    for kk in range(nlambda):
        if kk > 0:
            lam = lam * step
        thr = alpha * (2.0 * lam - lprev)
        ws_mask = ever | (np.abs(z) >= thr * pf)
        la1 = lam * alpha
        passes = 0
        while True:
            ws = np.flatnonzero(ws_mask)
            while True:
                conv = F.cd_pass(lam, ws)
                passes += 1
                if conv or passes >= max_iter:
                    break
            z = F.full_pass()
            viol = ~ws_mask & (np.abs(z) > la1 * pf)
            if not viol.any():
                break
            ws_mask = ws_mask | viol
        nz = F.beta != 0.0
        ever |= nz
        loss = F.val_loss()
        out["lam"].append(lam)
        out["loss"].append(loss)
        out["nnz"].append(int(nz.sum()))
        out["npass"].append(passes)
        if keep_path:
            out["pbeta"].append(F.beta.copy())
            out["pb0"].append(F.b0)
        if loss < best_loss:
            best_loss, best = loss, kk
            bbest, b0best = F.beta.copy(), F.b0
        lprev = lam
        if nz.sum() > dfmax:
            stop = 2
        elif kk - best >= n_abort and kk + 1 >= nlam_min:
            stop = 1
        elif kk == nlambda - 1:
            stop = 0
        if stop >= 0:
            break
    out.update(beta=bbest, b0=b0best, best=best, length=kk + 1, message=stop)
    return out


def splreg(Xd, y, family, ind_sets, K, covar=None, base=None, pf_X=None, pf_covar=None, alphas=(1.0,), nlambda=200,
           lambda_min_ratio=1e-4, nlam_min=50, n_abort=10, dfmax=50000, eps=1e-5, max_iter=1000, keep_path=False,
           col_key=None, engine="numpy"):
    """Xd: nr x nc decoded genotype values at the observations (codes, or byte / D), y[nr], ind_sets[nr] in 1..K.
    col_key[nc] (default 0..nc-1; the device uses the genotype line): coordinate descent visits the kept columns by
    increasing key, ties in column order, then the covariates.  Returns the raw per-fit results of bsg_splreg (fit
    f = ia * K + k, coefficients of the kept columns in column order, then the covariates) plus the column
    statistics.  engine="c" runs the fits through the C oracle (tests/splreg_oracle.c, same arithmetic, fits in
    parallel over OpenMP threads)."""
    Xd = np.asarray(Xd, dtype=np.float64)
    nr, nc = Xd.shape
    Kc = 0 if covar is None else covar.shape[1]
    Xall = Xd if Kc == 0 else np.column_stack([Xd, covar])
    center, scale = column_stats(Xall)
    kept = scale[:nc] > SD_MIN
    kc = np.flatnonzero(kept)
    key = np.arange(nc) if col_key is None else np.asarray(col_key)
    order = np.argsort(key[kc], kind="stable")
    cols = np.concatenate([kc[order], nc + np.arange(Kc)])
    c, isd = center[cols], 1.0 / scale[cols]
    Xt = (Xall[:, cols] - c) * isd
    pf = np.concatenate([np.ones(nc) if pf_X is None else np.asarray(pf_X, float),
                         np.ones(Kc) if pf_covar is None else np.asarray(pf_covar, float)])[cols]
    base = np.zeros(nr) if base is None else np.asarray(base, float)
    y = np.asarray(y, float)
    step = lambda_min_ratio ** (1.0 / (nlambda - 1)) if nlambda > 1 else 1.0
    ind_sets = np.asarray(ind_sets)
    if engine == "c":
        fits = _fits_c(Xt, y, base, pf, family, alphas, ind_sets, K, nlambda, step, nlam_min, n_abort, dfmax, eps,
                       max_iter, keep_path)
    else:
        fits = _fits_numpy(Xt, y, base, pf, family, alphas, ind_sets, K, nlambda, step, nlam_min, n_abort, dfmax, eps,
                           max_iter, keep_path)
    back = np.concatenate([np.argsort(order, kind="stable"), kc.size + np.arange(Kc)])  # descent order -> column order
    for fit in fits:
        fit["beta"] = fit["beta"][back]
        fit["pbeta"] = [b[back] for b in fit["pbeta"]]
    return dict(center=center, scale=scale, kept=kept, fits=fits, J=cols.size)


def _fits_numpy(Xt, y, base, pf, family, alphas, ind_sets, K, nlambda, step, nlam_min, n_abort, dfmax, eps, max_iter,
                keep_path):
    fits = []
    for a in alphas:
        for k in range(1, K + 1):
            train, val = np.flatnonzero(ind_sets != k), np.flatnonzero(ind_sets == k)
            fits.append(fit_path(Xt, y, base, pf, float(a), train, val, family, nlambda, step, nlam_min, n_abort,
                                 dfmax, eps, max_iter, keep_path))
    return fits


_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, "splreg_oracle.c")
HEADER = os.path.join(os.path.dirname(_HERE), "bigsnpr_b200", "csrc", "bsg_ldpred2_auto.cuh")
_lib = None


def lib():
    """The C oracle, compiled on first use (-O2 -ffp-contract=off -fopenmp) into a per-user temporary directory."""
    global _lib
    if _lib is None:
        d = os.path.join(tempfile.gettempdir(), "bsg_splreg_oracle_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        h = hashlib.sha1(open(SRC, "rb").read() + open(HEADER, "rb").read()).hexdigest()[:12]
        so = os.path.join(d, "splreg_oracle_%s.so" % h)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared", SRC, "-o", tmp,
                                   "-lm"])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
    return _lib


def _fits_c(Xt, y, base, pf, family, alphas, ind_sets, K, nlambda, step, nlam_min, n_abort, dfmax, eps, max_iter,
            keep_path):
    nr, J = Xt.shape
    A = len(alphas)
    F = A * K
    D = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    I = lambda a: a.ctypes.data_as(C.POINTER(C.c_int))  # noqa: E731
    X = np.ascontiguousarray(Xt.T)
    al = np.ascontiguousarray(alphas, dtype=np.float64)
    sets = np.ascontiguousarray(ind_sets, dtype=np.int32)
    beta, b0 = np.zeros(max(F * J, 1)), np.zeros(F)
    best, length, msg = (np.zeros(F, dtype=np.int32) for _ in range(3))
    lam, loss = np.zeros(F * nlambda), np.zeros(F * nlambda)
    nnz, npass = np.zeros(F * nlambda, dtype=np.int32), np.zeros(F * nlambda, dtype=np.int32)
    pbeta = np.zeros(max(F * nlambda * J, 1)) if keep_path else None
    pb0 = np.zeros(F * nlambda) if keep_path else None
    rc = lib().splreg_fits(D(X), C.c_int(nr), C.c_int(J), D(np.ascontiguousarray(y, dtype=np.float64)),
                           D(np.ascontiguousarray(base, dtype=np.float64)), D(np.ascontiguousarray(pf, dtype=np.float64)),
                           C.c_int(family), D(al), C.c_int(A), I(sets), C.c_int(K), C.c_int(nlambda), C.c_double(step),
                           C.c_int(nlam_min), C.c_int(n_abort), C.c_int(dfmax), C.c_double(eps), C.c_int(max_iter),
                           D(beta), D(b0), I(best), I(length), I(msg), D(lam), D(loss), I(nnz), I(npass),
                           D(pbeta) if keep_path else None, D(pb0) if keep_path else None)
    if rc != 0:
        raise MemoryError("splreg oracle: allocation failure")
    fits = []
    for f in range(F):
        L = int(length[f])
        sl = slice(f * nlambda, f * nlambda + L)
        fits.append(dict(lam=list(lam[sl]), loss=list(loss[sl]), nnz=[int(v) for v in nnz[sl]],
                         npass=[int(v) for v in npass[sl]],
                         pbeta=[pbeta[(f * nlambda + i) * J:(f * nlambda + i + 1) * J].copy() for i in range(L)]
                         if keep_path else [],
                         pb0=list(pb0[sl]) if keep_path else [], beta=beta[f * J:(f + 1) * J].copy(), b0=float(b0[f]),
                         best=int(best[f]), length=L, message=int(msg[f])))
    return fits
