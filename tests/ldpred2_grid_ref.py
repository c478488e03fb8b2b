"""CPU oracle of LDpred2-grid -- test infrastructure only.

ctypes wrapper over ``tests/ldpred2_grid_oracle.c`` (literal restatements of src/ldpred2.cpp:9-69 and
src/ldpred2-sampling.cpp:9-59 on the draws and math of ``bigsnpr_b200/csrc/bsg_ldpred2_auto.cuh``, plus LDpred2-auto's
chain with its final state), compiled on first use with -O2 -ffp-contract=off -fopenmp into a temporary directory; the
build is keyed on the .c files and the header.  Storage arrays are those of ``bigsnpr_b200.api.sfbm_storage``; indices
are 0-based like the .Call target's.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tests import ldpred2_auto_ref as AR

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, "ldpred2_grid_oracle.c")
FLAGS = AR.FLAGS
_lib = None

_D, _I, _U = C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_uint32)


def _build_dir():
    d = os.path.join(tempfile.gettempdir(), "bsg_ldpred2_grid_oracle_%d" % os.getuid())
    os.makedirs(d, exist_ok=True)
    h = hashlib.sha1(b"".join(open(f, "rb").read() for f in (SRC, AR.SRC, AR.HEADER))).hexdigest()[:12]
    return d, h


def object_file():
    """The oracle compiled to an object file (for inspecting its instructions)."""
    d, h = _build_dir()
    o = os.path.join(d, "ldpred2_grid_oracle_%s.o" % h)
    if not os.path.exists(o):
        tmp = o + ".%d.tmp" % os.getpid()
        subprocess.check_call(["gcc"] + FLAGS + ["-c", SRC, "-o", tmp])
        os.replace(tmp, o)
    return o


def lib():
    global _lib
    if _lib is None:
        d, h = _build_dir()
        so = os.path.join(d, "ldpred2_grid_oracle_%s.so" % h)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc"] + FLAGS + ["-shared", SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.ldg_coord_1.argtypes = [C.c_double, C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_double, _D]
        L.ldg_offset.argtypes = [C.c_uint32, C.c_int]
        _lib = L
    return _lib


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def coord(beta_hat, dotprod, cur, sampling, h2_per_var, n, inv_odd_p):
    """(postp, C3, C4) of one coordinate, the residual formed as the variant forms it"""
    out = np.empty(3)
    lib().ldg_coord_1(beta_hat, dotprod, cur, int(bool(sampling)), h2_per_var, n, inv_odd_p, _p(out, C.c_double))
    return tuple(out)


def offset(draws, lane):
    return lib().ldg_offset(int(draws), int(lane))


def ldpred2_grid(storage, beta_hat, n_vec, ind_sub, p, h2, sparse, rng, burn_in=50, num_iter=100, sampling=False,
                 nthreads=None, counts=False):
    """Every point of ldpred2_gibbs_one (point g: p[g], h2[g], sparse[g], MRG32k3a state rng[g]), or with `sampling` the
    one point of ldpred2_gibbs_one_sampling.  A dict: beta_est (m x npoint) or sample_beta (m x num_iter), rng_out
    (npoint x 6, each point's final state); with counts, also moves / entries per point (column updates and the stored
    values they read), sweeps per point (the diverging one included; 0 with sampling) and each point's wall seconds."""
    n, pp, data, first_i = storage
    f64 = lambda a: np.ascontiguousarray(np.atleast_1d(a), dtype=np.float64)
    p, h2 = f64(p), f64(h2)
    npoint = p.size
    sparse = np.ascontiguousarray(np.atleast_1d(sparse).astype(bool), dtype=np.int32)
    assert h2.size == npoint and sparse.size == npoint and (not sampling or npoint == 1)
    m = int(np.size(beta_hat))
    beta_hat, n_vec = f64(beta_hat), f64(n_vec)
    ind_sub = np.ascontiguousarray(ind_sub, dtype=np.int32)
    assert n_vec.size == m and ind_sub.size == m and np.all((ind_sub >= 0) & (ind_sub < n))
    rng = np.ascontiguousarray(np.asarray(rng, dtype=np.uint32).reshape(npoint * 6))
    fi = None if first_i is None else np.ascontiguousarray(first_i, dtype=np.int32)
    est = None if sampling else np.empty((m, npoint), order="F")
    smp = np.empty((m, num_iter), order="F") if sampling else None
    rout = np.empty((npoint, 6), dtype=np.uint32)
    mv, ent, secs = np.zeros(npoint, dtype=np.int64), np.zeros(npoint, dtype=np.int64), np.zeros(npoint)
    sweeps = np.zeros(npoint, dtype=np.int32)
    rc = lib().ldg_ldpred2_grid(
        _p(pp, C.c_double), _p(data, C.c_double), _p(fi, C.c_int), int(n), _p(beta_hat, C.c_double),
        _p(n_vec, C.c_double), m, _p(ind_sub, C.c_int), npoint, _p(p, C.c_double), _p(h2, C.c_double),
        _p(sparse, C.c_int), int(burn_in), int(num_iter), int(bool(sampling)), _p(rng, C.c_uint32), _p(est, C.c_double),
        _p(smp, C.c_double), _p(rout, C.c_uint32), _p(mv, C.c_longlong), _p(ent, C.c_longlong), _p(sweeps, C.c_int),
        _p(secs, C.c_double), int(nthreads or os.cpu_count() or 1))
    if rc:
        raise MemoryError("ldpred2_grid oracle: allocation failure")
    out = {"beta_est": est, "sample_beta": smp, "rng_out": rout}
    if counts:
        out["moves"], out["entries"], out["sweeps"], out["seconds"] = mv, ent, sweeps, secs
    return out


def ldpred2_auto_state(storage, beta_hat, n_vec, log_var, ind_sub, p_init, h2_init, rng, burn_in=500, num_iter=200,
                       report_step=None, no_jump_sign=False, shrink_corr=1.0, use_mle=True, p_bounds=(1e-5, 1.0),
                       alpha_bounds=(-0.5, 1.5), mean_ld=1.0, nthreads=None):
    """ldpred2_auto_ref.ldpred2_auto's estimates and paths (no sample_beta), and each chain's final MRG32k3a state
    (rng_out, nchain x 6)."""
    n, p, data, first_i = storage
    p_init = np.ascontiguousarray(np.atleast_1d(p_init), dtype=np.float64)
    nchain = p_init.size
    m = int(np.size(beta_hat))
    report_step = num_iter + 1 if report_step is None else int(report_step)
    T = burn_in + num_iter
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    beta_hat, n_vec, log_var = f64(beta_hat), f64(n_vec), f64(log_var)
    ind_sub = np.ascontiguousarray(ind_sub, dtype=np.int32)
    rng = np.ascontiguousarray(np.asarray(rng, dtype=np.uint32).reshape(nchain * 6))
    fi = None if first_i is None else np.ascontiguousarray(first_i, dtype=np.int32)
    est = [np.empty((m, nchain), order="F") for _ in range(3)]
    paths = [np.empty((T, nchain), order="F") for _ in range(3)]
    rout = np.empty((nchain, 6), dtype=np.uint32)
    pb, ab = f64(p_bounds), f64(alpha_bounds)
    rc = lib().lda_ldpred2_auto_state(
        _p(p, C.c_double), _p(data, C.c_double), _p(fi, C.c_int), int(n), _p(beta_hat, C.c_double), _p(n_vec, C.c_double),
        _p(log_var, C.c_double), m, _p(ind_sub, C.c_int), nchain, _p(p_init, C.c_double), C.c_double(h2_init),
        int(burn_in), int(num_iter), int(report_step), int(bool(no_jump_sign)), C.c_double(shrink_corr), int(bool(use_mle)),
        _p(pb, C.c_double), _p(ab, C.c_double), C.c_double(mean_ld), _p(rng, C.c_uint32), *(_p(a, C.c_double) for a in est),
        *(_p(a, C.c_double) for a in paths), _p(rout, C.c_uint32), int(nthreads or os.cpu_count() or 1))
    if rc:
        raise MemoryError("ldpred2_auto oracle: allocation failure")
    out = dict(zip(("beta_est", "postp_est", "corr_est"), est))
    out.update(zip(("path_p_est", "path_h2_est", "path_alpha_est"), paths))
    out["rng_out"] = rout
    return out
