"""CPU oracle of LDpred2-auto -- test infrastructure only.

ctypes wrapper over ``tests/ldpred2_auto_oracle.c`` (a literal restatement of src/ldpred2-auto.cpp:56-202 on the draws and
math of ``bigsnpr_b200/csrc/bsg_ldpred2_auto.cuh``), compiled on first use with -O2 -ffp-contract=off -fopenmp into a
temporary directory; the build is keyed on both the .c file and the header.  Storage arrays are those of
``bigsnpr_b200.api.sfbm_storage``; indices are 0-based like the .Call target's.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, "ldpred2_auto_oracle.c")
HEADER = os.path.join(os.path.dirname(_HERE), "bigsnpr_b200", "csrc", "bsg_ldpred2_auto.cuh")
FLAGS = ["-O2", "-ffp-contract=off", "-fopenmp", "-fPIC"]
_lib = None

_D, _I, _U = C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_uint32)


def _build_dir():
    d = os.path.join(tempfile.gettempdir(), "bsg_ldpred2_auto_oracle_%d" % os.getuid())
    os.makedirs(d, exist_ok=True)
    h = hashlib.sha1(open(SRC, "rb").read() + open(HEADER, "rb").read()).hexdigest()[:12]
    return d, h


def object_file():
    """The oracle compiled to an object file (for inspecting its instructions)."""
    d, h = _build_dir()
    o = os.path.join(d, "ldpred2_auto_oracle_%s.o" % h)
    if not os.path.exists(o):
        tmp = o + ".%d.tmp" % os.getpid()
        subprocess.check_call(["gcc"] + FLAGS + ["-c", SRC, "-o", tmp])
        os.replace(tmp, o)
    return o


def lib():
    global _lib
    if _lib is None:
        d, h = _build_dir()
        so = os.path.join(d, "ldpred2_auto_oracle_%s.so" % h)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc"] + FLAGS + ["-shared", SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.lda_draw_p_1.restype = C.c_double
        L.lda_draw_p_1.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, _U]
        L.lda_mle_objective.restype = C.c_double
        L.lda_mle_objective.argtypes = [_D, _D, C.c_int, C.c_double, C.c_double, C.c_double, _D]
        L.lda_mle_fit.argtypes = [_D, _D, C.c_int, C.c_double, C.c_double, _D]
        L.lda_skip_k.argtypes = [_U, C.c_uint64]
        L.lda_rnorm_n.argtypes = [C.c_double, C.c_double, _U, C.c_int, _D]
        L.lda_rbeta_n.argtypes = [C.c_double, C.c_double, _U, C.c_int, _D]
        L.lda_coord_1.argtypes = [C.c_double] * 6 + [C.c_int] + [C.c_double] * 3 + [_D]
        _lib = L
    return _lib


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def _state(s):
    return np.ascontiguousarray(np.asarray(s, dtype=np.uint32).reshape(6)).copy()


def unif(state, n):
    """(n uniforms, the state after them)"""
    s, out = _state(state), np.empty(n)
    lib().lda_unif_n(_p(s, C.c_uint32), int(n), _p(out, C.c_double))
    return out, s


def skip(state, k):
    s = _state(state)
    lib().lda_skip_k(_p(s, C.c_uint32), int(k))
    return s


def jump127(state):
    s = _state(state)
    lib().lda_jump(_p(s, C.c_uint32))
    return s


def _vec(fn, x):
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.empty_like(x)
    getattr(lib(), fn)(_p(x, C.c_double), int(x.size), _p(out, C.c_double))
    return out


def exp(x):
    return _vec("lda_exp_n", x)


def log(x):
    return _vec("lda_log_n", x)


def qnorm(x):
    return _vec("lda_qnorm_n", x)


def rnorm(mu, sigma, state, n=1):
    s, out = _state(state), np.empty(n)
    lib().lda_rnorm_n(float(mu), float(sigma), _p(s, C.c_uint32), int(n), _p(out, C.c_double))
    return out, s


def rbeta(a, b, state, n=1):
    s, out = _state(state), np.empty(n)
    lib().lda_rbeta_n(float(a), float(b), _p(s, C.c_uint32), int(n), _p(out, C.c_double))
    return out, s


def draw_p(nb, m, mean_ld, p_lo, p_hi, state):
    s = _state(state)
    v = lib().lda_draw_p_1(int(nb), int(m), float(mean_ld), float(p_lo), float(p_hi), _p(s, C.c_uint32))
    return v, s


def coord(beta_hat, dotprod, cur, n, log_var, shrink, use_mle, alpha_plus_one, sigma2, inv_odd_p):
    """(postp, C3, C4, dotprod_shrunk) of one coordinate"""
    out = np.empty(4)
    lib().lda_coord_1(beta_hat, dotprod, cur, n, log_var, shrink, int(use_mle), alpha_plus_one, sigma2, inv_odd_p,
                      _p(out, C.c_double))
    return tuple(out)


def mle_fit(a, b, t_lo, t_hi, par):
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    par = np.array(par, dtype=np.float64)
    lib().lda_mle_fit(_p(a, C.c_double), _p(b, C.c_double), int(a.size), float(t_lo), float(t_hi), _p(par, C.c_double))
    return par


def mle_objective(a, b, t, s2_lo, s2_hi):
    """(profiled objective at t, its sigma2)"""
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    s2 = C.c_double()
    f = lib().lda_mle_objective(_p(a, C.c_double), _p(b, C.c_double), int(a.size), float(t), float(s2_lo), float(s2_hi),
                                C.byref(s2))
    return f, s2.value


def ldpred2_auto(storage, beta_hat, n_vec, log_var, ind_sub, p_init, h2_init, rng, burn_in=500, num_iter=200,
                 report_step=None, no_jump_sign=False, shrink_corr=1.0, use_mle=True, p_bounds=(1e-5, 1.0),
                 alpha_bounds=(-0.5, 1.5), mean_ld=1.0, sample=True, nthreads=None, counts=False):
    """Every chain of ldpred2_gibbs_auto (chain c: p_init[c], MRG32k3a state rng[c]); alpha_bounds are alpha + 1, as the
    .Call receives them.  A dict like bigsnpr_b200.api._ldpred2_auto_call's; with counts, also moves / entries per chain
    (column updates and the stored values they read) and each chain's wall seconds."""
    n, p, data, first_i = storage
    p_init = np.ascontiguousarray(np.atleast_1d(p_init), dtype=np.float64)
    nchain = p_init.size
    m = int(np.size(beta_hat))
    report_step = num_iter + 1 if report_step is None else int(report_step)
    T, nrep = burn_in + num_iter, num_iter // report_step
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    beta_hat, n_vec, log_var = f64(beta_hat), f64(n_vec), f64(log_var)
    ind_sub = np.ascontiguousarray(ind_sub, dtype=np.int32)
    assert n_vec.size == m and log_var.size == m and ind_sub.size == m and np.all((ind_sub >= 0) & (ind_sub < n))
    rng = np.ascontiguousarray(np.asarray(rng, dtype=np.uint32).reshape(nchain * 6))
    fi = None if first_i is None else np.ascontiguousarray(first_i, dtype=np.int32)
    est = [np.empty((m, nchain), order="F") for _ in range(3)]
    paths = [np.empty((T, nchain), order="F") for _ in range(3)]
    smp = np.empty((m, nrep, nchain), order="F") if sample else None
    mv, ent, secs = np.zeros(nchain, dtype=np.int64), np.zeros(nchain, dtype=np.int64), np.zeros(nchain)
    pb, ab = f64(p_bounds), f64(alpha_bounds)
    rc = lib().lda_ldpred2_auto(
        _p(p, C.c_double), _p(data, C.c_double), _p(fi, C.c_int), int(n), _p(beta_hat, C.c_double), _p(n_vec, C.c_double),
        _p(log_var, C.c_double), m, _p(ind_sub, C.c_int), nchain, _p(p_init, C.c_double), C.c_double(h2_init),
        int(burn_in), int(num_iter), int(report_step), int(bool(no_jump_sign)), C.c_double(shrink_corr), int(bool(use_mle)),
        _p(pb, C.c_double), _p(ab, C.c_double), C.c_double(mean_ld), _p(rng, C.c_uint32), *(_p(a, C.c_double) for a in est),
        *(_p(a, C.c_double) for a in paths), _p(smp, C.c_double), _p(mv, C.c_longlong), _p(ent, C.c_longlong),
        _p(secs, C.c_double), int(nthreads or os.cpu_count() or 1))
    if rc:
        raise MemoryError("ldpred2_auto oracle: allocation failure")
    out = dict(zip(("beta_est", "postp_est", "corr_est"), est))
    out.update(zip(("path_p_est", "path_h2_est", "path_alpha_est"), paths))
    out["sample_beta"] = smp
    if counts:
        out["moves"], out["entries"], out["seconds"] = mv, ent, secs
    return out
