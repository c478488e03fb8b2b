"""CPU oracle of sp_solve_sym -- test infrastructure only.

ctypes wrapper over ``tests/spsolve_oracle.c`` (Eigen's ConjugateGradient with the identity preconditioner from x = 0, in
this project's declared reduction order), compiled on first use with -O2 -ffp-contract=off -fopenmp into a temporary
directory.  Storage arrays are those of ``bigsnpr_b200.api.sfbm_storage``.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile
import time

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "spsolve_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), "bsg_spsolve_oracle_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "spsolve_oracle_%s.so" % hashlib.sha1(src).hexdigest()[:12])
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", _SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
    return _lib


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def solve(storage, b, add_to_diag, tol=1e-10, maxiter=None, nthreads=None, timed=False):
    """(x, iters, error) of the CG solve of (A + diag(add_to_diag)) x = b; add_to_diag has length 1 or n; maxiter None is
    10 n.  With timed, also the wall seconds of the call."""
    n, p, data, first_i = storage
    b = np.ascontiguousarray(b, dtype=np.float64)
    d = np.ascontiguousarray(np.atleast_1d(add_to_diag), dtype=np.float64).reshape(-1)
    assert b.size == n and d.size in (1, n)
    fi = None if first_i is None else np.ascontiguousarray(first_i, dtype=np.int32)
    x = np.empty(n)
    it, err = C.c_int(), C.c_double()
    t0 = time.time()
    rc = lib().spo_solve(_p(p, C.c_double), _p(data, C.c_double), _p(fi, C.c_int), n, _p(b, C.c_double),
                         _p(d, C.c_double), d.size, C.c_double(tol), int(10 * n if maxiter is None else maxiter),
                         _p(x, C.c_double), C.byref(it), C.byref(err), int(nthreads or os.cpu_count() or 1))
    secs = time.time() - t0
    if rc:
        raise MemoryError("sp_solve_sym oracle: allocation failure")
    return (x, it.value, err.value, secs) if timed else (x, it.value, err.value)
