"""CPU oracle of lassosum2 and ld_scores_sfbm -- test infrastructure only.

ctypes wrapper over ``tests/lassosum2_oracle.c`` (literal restatements of src/lassosum2.cpp:20-70 and
src/ld-scores-sfbm.cpp:9-69 over bigsparser's storage), compiled on first use with -O2 -ffp-contract=off -fopenmp into a
temporary directory.  Storage arrays are those of ``bigsnpr_b200.api.sfbm_storage``; indices are 0-based like the .Call
targets'.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lassosum2_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), "bsg_lassosum2_oracle_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "lassosum2_oracle_%s.so" % hashlib.sha1(src).hexdigest()[:12])
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", _SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
    return _lib


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def lassosum2(storage, beta_hat, ind_sub, lam, dp1, dfmax, maxiter, tol, nthreads=None, counts=False):
    """Grid of src/lassosum2.cpp:20-70 calls: lam / dp1 are m x ngrid (column g = one call's lambda / delta_plus_one).
    Returns (beta m x ngrid, num_iter); with counts, also (moves, entries, seconds) per point: coordinates that moved,
    stored values their column updates read, and each point's wall time."""
    n, p, data, first_i = storage
    beta_hat = np.ascontiguousarray(beta_hat, dtype=np.float64)
    ind_sub = np.ascontiguousarray(ind_sub, dtype=np.int32)
    lam, dp1 = np.asfortranarray(lam, dtype=np.float64), np.asfortranarray(dp1, dtype=np.float64)
    m, ngrid = lam.shape
    assert beta_hat.size == m and ind_sub.size == m and dp1.shape == lam.shape
    assert np.all((ind_sub >= 0) & (ind_sub < n))
    fi = None if first_i is None else np.ascontiguousarray(first_i, dtype=np.int32)
    beta = np.empty((m, ngrid), order="F")
    it = np.empty(ngrid, dtype=np.int32)
    mv, ent, secs = np.zeros(ngrid, dtype=np.int64), np.zeros(ngrid, dtype=np.int64), np.zeros(ngrid)
    rc = lib().lso_lassosum2(_p(p, C.c_double), _p(data, C.c_double), _p(fi, C.c_int), n, _p(beta_hat, C.c_double), m,
                             _p(ind_sub, C.c_int), ngrid, _p(lam, C.c_double), _p(dp1, C.c_double), C.c_double(dfmax),
                             int(maxiter), C.c_double(tol), _p(beta, C.c_double), _p(it, C.c_int), _p(mv, C.c_longlong),
                             _p(ent, C.c_longlong), _p(secs, C.c_double), int(nthreads or os.cpu_count() or 1))
    if rc:
        raise MemoryError("lassosum2 oracle: allocation failure")
    return (beta, it, mv, ent, secs) if counts else (beta, it)


def ld_scores(storage, ind_sub):
    n, p, data, first_i = storage
    ind_sub = np.ascontiguousarray(ind_sub, dtype=np.int32)
    fi = None if first_i is None else np.ascontiguousarray(first_i, dtype=np.int32)
    out = np.empty(ind_sub.size)
    if lib().lso_ld_scores(_p(p, C.c_double), _p(data, C.c_double), _p(fi, C.c_int), n, n, _p(ind_sub, C.c_int), ind_sub.size,
                           _p(out, C.c_double)):
        raise MemoryError("ld_scores oracle: allocation failure")
    return out


def grid_inputs(df_beta, delta=(0.001, 0.01, 0.1, 1), nlambda=30, lambda_min_ratio=0.01):
    """R/lassosum2.R:40-51 restated independently of the package: (beta_hat, scale, lam m x ngrid, dp1, lambda, delta)."""
    import math

    beta, se, N = (np.asarray(df_beta[k], dtype=np.float64) for k in ("beta", "beta_se", "n_eff"))
    scale = np.sqrt(N * se ** 2 + beta ** 2)
    beta_hat = beta / scale
    pf = np.sqrt(np.max(N) / N)
    lambda0 = np.max(np.abs(beta_hat / pf))
    n = nlambda + 1
    a, b = math.log(lambda0), math.log(lambda_min_ratio * lambda0)
    by = (b - a) / (n - 1)
    s = [a] + [a + i * by for i in range(1, n - 1)] + [b]
    seq_lam = np.array([math.exp(v) for v in s])[1:]
    delta = np.asarray(delta, dtype=np.float64)
    g_lam = np.array([lv for _ in delta for lv in seq_lam])
    g_del = np.array([d for d in delta for _ in seq_lam])
    lam = np.asfortranarray(np.outer(pf, g_lam))
    dp1 = np.asfortranarray(pf[:, None] * g_del[None, :] + 1)
    return beta_hat, scale, lam, dp1, g_lam, g_del
