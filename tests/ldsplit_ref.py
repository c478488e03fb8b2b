"""CPU oracle of snp_ldsplit -- test infrastructure only.

ctypes wrapper over ``tests/ldsplit_oracle.c`` (literal restatements of get_L, get_C and get_perc, src/split-LD.cpp),
compiled on first use with -O2 -ffp-contract=off into a temporary directory, and a restatement of the R driver
(R/split-LD.R:99-138 and reconstruct_paths, R/split-LD.R:3-40) over them.  corr is the lower triangle in CSC as
``bigsnpr_b200.api.ldsplit_lower`` returns it.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ldsplit_oracle.c")
_lib = None
NA_INTEGER = -2147483648


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), "bsg_ldsplit_oracle_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "ldsplit_oracle_%s.so" % hashlib.sha1(src).hexdigest()[:12])
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", _SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.ldo_get_L.restype = C.c_longlong
        L.ldo_get_C.restype = C.c_longlong
        L.ldo_get_perc.restype = C.c_double
        _lib = L
    return _lib


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def get_L(lower, thr_r2, max_r2):
    """src/split-LD.cpp:15-61: (i, j, x) triplets, 0-based, by column of corr and row descending."""
    p, i, x = (np.ascontiguousarray(lower[0], dtype=np.int64), np.ascontiguousarray(lower[1], dtype=np.int32),
               np.ascontiguousarray(lower[2], dtype=np.float64))
    m = p.size - 1
    args = (_p(p, C.c_longlong), _p(i, C.c_int), _p(x, C.c_double), m, C.c_double(thr_r2), C.c_double(max_r2))
    n = lib().ldo_get_L(*args, None, None, None)
    li, lj, lx = np.empty(n, dtype=np.int32), np.empty(n, dtype=np.int32), np.empty(n)
    lib().ldo_get_L(*args, _p(li, C.c_int), _p(lj, C.c_int), _p(lx, C.c_double))
    return li, lj, lx


def L_csc(triplets, m):
    """Matrix::sparseMatrix(i, j, x, dims = c(m, m + 1), index1 = FALSE) as CSC (lp, li, lx)."""
    li, lj, lx = triplets
    o = np.lexsort((li, lj))
    lp = np.zeros(m + 2, dtype=np.int64)
    np.cumsum(np.bincount(lj, minlength=m + 1), out=lp[1:])
    return lp, li[o].astype(np.int32), lx[o].astype(np.float64)


def get_C(L, m, min_size, max_size, max_K, max_cost, pos_scaled, layers=False):
    """src/split-LD.cpp:65-145 on L in CSC (m x (m + 1)): (C m x max_K, best_ind 1-based with NA), and the layers run."""
    lp, li, lx = (np.ascontiguousarray(L[0], dtype=np.int64), np.ascontiguousarray(L[1], dtype=np.int32),
                  np.ascontiguousarray(L[2], dtype=np.float64))
    pos = np.ascontiguousarray(pos_scaled, dtype=np.float64)
    C1 = np.empty((m, max_K), order="F")
    best = np.empty((m, max_K), dtype=np.int32, order="F")
    nl = C.c_int(0)
    rc = lib().ldo_get_C(_p(lp, C.c_longlong), _p(li, C.c_int), _p(lx, C.c_double), m, int(min_size), int(max_size),
                         int(max_K), C.c_double(max_cost), _p(pos, C.c_double), _p(C1, C.c_double), _p(best, C.c_int),
                         C.byref(nl))
    if rc < 0:
        raise MemoryError("get_C oracle: allocation failure")
    return (C1, best, nl.value) if layers else (C1, best)


def get_perc(lower, all_last0):
    p, i = np.ascontiguousarray(lower[0], dtype=np.float64), np.ascontiguousarray(lower[1], dtype=np.int32)
    al = np.ascontiguousarray(all_last0, dtype=np.int32)
    return lib().ldo_get_perc(_p(p, C.c_double), _p(i, C.c_int), p.size - 1, C.c_longlong(i.size), _p(al, C.c_int))


def snp_ldsplit(lower, thr_r2, min_size, max_size, max_K=500, max_r2=0.3, max_cost=None, pos_scaled=None, layers=None):
    """R/split-LD.R:99-138 over the oracle.  Returns None or the dict of columns of bigsnpr_b200.api.snp_ldsplit.
    layers: a list that receives the layers get_C ran for each sorted max_size."""
    p, i, x = lower
    m = len(p) - 1
    max_cost = m / 200 if max_cost is None else float(max_cost)
    pos = np.zeros(m) if pos_scaled is None else np.asarray(pos_scaled, dtype=np.float64)
    ss = 0.0
    for v in np.asarray(x, dtype=np.float64):  # crossprod(corr@x), folded in order
        ss = ss + v * v
    max_cost = min(max_cost, ss * 2)
    L = L_csc(get_L(lower, thr_r2, max_r2), m)
    prev = np.full(max_K, np.inf)
    rows = []
    for S in sorted(int(s) for s in np.atleast_1d(max_size)):
        assert 1 <= min_size <= S <= m  # get_C is undefined otherwise
        C1, best, nl = get_C(L, m, min_size, S, max_K, max_cost, pos, layers=True)
        if layers is not None:
            layers.append(nl)
        for K in range(1, max_K + 1):
            cost = C1[0, K - 1]
            if cost > max_cost:
                continue
            if not cost < prev[K - 1]:
                continue
            prev[K - 1] = cost
            all_last, j, k = [], 0, K
            while True:
                j = int(best[j, k - 1])
                all_last.append(j)
                if k == 1:
                    break
                k -= 1
            all_last = np.array(all_last, dtype=np.int32)
            assert all_last.size == K
            size = np.diff(np.concatenate([[0], all_last])).astype(np.int32)
            assert np.all((size >= min_size) & (size <= S))
            rows.append((S, K, cost, float(np.sum(size.astype(np.float64) ** 2)), get_perc(lower, all_last - 1),
                         all_last, size))
    if not rows:
        return None
    return {"max_size": np.array([r[0] for r in rows], dtype=np.int32), "n_block": np.array([r[1] for r in rows], dtype=np.int32),
            "cost": np.array([r[2] for r in rows]), "cost2": np.array([r[3] for r in rows]),
            "perc_kept": np.array([r[4] for r in rows]), "all_last": [r[5] for r in rows], "all_size": [r[6] for r in rows]}
