"""Exact host model of the GRM's arithmetic (bsg_tcrossprod: bsg_la.cu tcrossprod_impl, bsg_gramt.cu gramt_grm,
bsg_gram5.cu k_wgram5, bsg_la.cu k_wgram), so a K computed on the device can be compared with it byte for byte.

K = X~ X~^T with X~ = (X - c) / s over the non-missing entries is computed as

    K_ij = sum_k W1 a_ik a_jk + W2' (a_ik n_jk + n_ik a_jk) + W3 n_ik n_jk      (weighted integer Grams)
         + r_i + r_j + sum W3 - q_i - q_j                                        (vector terms)

with a the genotype (missing -> 0), n the missing indicator, and (k_grm_weights) u = 1/s, t = -c/s, W1 = u u,
W2' = -(u t), W3 = t t, w2 = u t, r = A w2, q = N W3.  The steps the model restates:

* weight classes (tcrossprod_impl): class(k) = floor(log2(max W1 / W1_k) / 4) (W1_k = 0: class 0), so every W1 of a
  class lies within a factor 16 of the class maximum.  One class: the columns keep their order.
  Several: the columns are stably sorted by class, and each class is quantised and folded on its own, in class order;
* quantisation per class and weight: e = dbits nslices - 1 - ex(class max), digit s = bits [dbits s, dbits s + dbits) of
  rint(W 2^e) (ties to even, __double2ll_rn), slice scale 2^(dbits s - e); dbits = 7, or 6 on the non-TMA kernels above
  4,000,000 columns;
* integer Grams per slice and product: aa (W1), an and na (W2'), nn (W3).  Every partial sum is an integer below 2^53, so
  an fp64 GEMM is exact in any order; an, na and nn vanish on tiles without a missing value, so tile lists do not matter;
* fold order into K (products of powers of two and integers, so FMA contraction cannot change a byte):
  - k_gramt (default, <= 4 slices): per class, per k-block of at most 262,144 codes starting at the class's first
    128-code block, per product aa, an, na, nn: K += s2 S2 + s3 S3, then K += s0 S0 + s1 S1 (each pair sum exact);
  - k_wgram5 / k_wgram: per class, slices from the most significant down, per slice aa, an, na, nn: K += scale S;
* vector terms through the matvec engine (tests/fixedpoint_ref.py): r = X.w2 on the unscaled view (k_pmv on the
  sample-major copy, or the SNP-major kernels when the file holds a missing value); only when a selected row holds a
  missing value, q = (X~_{c=1,s=1}.W3 - A.W3) + sumW3 on the host; sumW3 a left-to-right fp64 sum in column order;
* k_grm_finish: K_ij = (((K_ij + r_i) + r_j) + sumW3) - (q_i + q_j) for i >= j, mirrored to the upper triangle.

`old_classes=True` models the single-class quantisation that preceded the weight classes (one exponent per weight
vector), for the accuracy comparison.
"""
from __future__ import annotations

import math

import numpy as np

from tests import fixedpoint_ref as fx

KBLK = 262144   # codes per k-block of gramt_grm (int32 head-room of the accumulators)
BK = 128        # codes per TMA k-block: a class's k-range is rounded out to it
CLASS_BITS = 4  # a weight class spans at most a factor 2^4 below its maximum


def grm_weights(center, scale):
    """k_grm_weights: (W1, W2', W3, w2), plain IEEE operations."""
    c, s = np.asarray(center, dtype=np.float64), np.asarray(scale, dtype=np.float64)
    with np.errstate(all="ignore"):
        u = 1.0 / s
        t = -c / s
        return u * u, -(u * t), t * t, u * t


def degenerate(W1, W2p, W3) -> bool:
    """Weights the integer Gram cannot take (non-finite, or W2' < 0): the library computes K with cuBLAS DSYRK."""
    return not (np.all(np.isfinite(W1)) and np.all(np.isfinite(W2p)) and np.all(np.isfinite(W3))) or bool(np.any(W2p < 0))


def _ex(x: float) -> int:
    return math.frexp(x)[1] if x > 0 else 0


def weight_classes(W1, old_classes=False) -> np.ndarray:
    """class(k) = floor(log2(max W1 / W1_k) / 4) exactly: max / 16^(c+1) < W1_k <= max / 16^c; W1_k = 0 -> class 0."""
    W1 = np.asarray(W1, dtype=np.float64)
    if old_classes or W1.size == 0:
        return np.zeros(W1.size, dtype=np.int64)
    m = float(np.max(W1))
    c = (_ex(m) - np.frexp(W1)[1].astype(np.int64)) // CLASS_BITS
    up = np.ldexp(W1, CLASS_BITS * (c + 1)) <= m
    down = ~up & (c > 0) & (np.ldexp(W1, CLASS_BITS * np.maximum(c, 0)) > m)
    c = np.where(up, c + 1, np.where(down, c - 1, c))
    return np.where(W1 > 0, c, 0)


def quant_digits(W, wmax: float, nslices: int, dbits: int):
    """(digits (len, nslices) int64, scales) of rint(W 2^e) with e from the class maximum."""
    e = dbits * nslices - 1 - _ex(wmax)
    v = np.rint(np.ldexp(np.asarray(W, dtype=np.float64), e)).astype(np.int64)
    D = np.stack([(v >> (dbits * s)) & ((1 << dbits) - 1) for s in range(nslices)], axis=1)
    return D, [math.ldexp(1.0, dbits * s - e) for s in range(nslices)]


def _gram(X, D, Y) -> np.ndarray:
    """sum_k X_ik D_k Y_jk, exact (integers below 2^53)."""
    return X @ (Y * D[None, :]).T


def _products(A, N, any_na):
    # (A operand, B operand, weight index) of aa, an, na, nn
    return [(A, A, 0)] + ([(A, N, 1), (N, A, 1), (N, N, 2)] if any_na else [])


def gram_fold(Gs, W1, W2p, W3, nslices=4, path="gramt", old_classes=False):
    """Lower triangle (i >= j) of the weighted integer Grams folded into K, before the vector terms.  Gs: selected
    codes (lines x columns, 3 = missing).  path: 'gramt' (k_gramt) or 'wgram' (k_wgram5 / k_wgram)."""
    Gs = np.asarray(Gs)
    nr, nc = Gs.shape
    A = np.where(Gs == 3, 0, Gs).astype(np.float64)
    N = (Gs == 3).astype(np.float64)
    any_na = bool(N.any())
    cls = weight_classes(W1, old_classes)
    order = np.argsort(cls, kind="stable")
    A, N, cls = A[:, order], N[:, order], cls[order]
    Ws = [np.asarray(W, dtype=np.float64)[order] for W in (W1, W2p, W3)]
    dbits = 7 if (path == "gramt" or nc <= 4000000) else 6
    K = np.zeros((nr, nr))
    for c in np.unique(cls):
        lo, hi = np.searchsorted(cls, c, "left"), np.searchsorted(cls, c, "right")
        inside = (np.arange(nc) >= lo) & (np.arange(nc) < hi)
        dig = [quant_digits(np.where(inside, W, 0.0), float(np.max(W[lo:hi])), nslices, dbits) for W in Ws]
        prods = _products(A, N, any_na)
        if path == "gramt":
            kb0, kb1 = lo // BK * BK, min(nc, -(-hi // BK) * BK)
            kblk = min(KBLK, -(-(kb1 - kb0) // BK) * BK)
            for k0 in range(kb0, kb1, kblk):
                ks = slice(k0, min(k0 + kblk, kb1))
                for X, Y, w in prods:
                    D, sc = dig[w]
                    for pair in ((2, 3), (0, 1)):
                        v = np.zeros((nr, nr))
                        for s in pair:
                            if s < nslices:
                                v = v + sc[s] * _gram(X[:, ks], D[ks, s], Y[:, ks])
                        K = K + v
        else:
            for s in range(nslices - 1, -1, -1):
                for X, Y, w in prods:
                    D, sc = dig[w]
                    K = K + sc[s] * _gram(X, D[:, s], Y)
    return K


def _sel(G, ir, ic):
    n, m = G.shape
    r0 = np.arange(n) if ir is None else np.asarray(ir, dtype=np.int64) - 1
    c0 = np.arange(m) if ic is None else np.asarray(ic, dtype=np.int64) - 1
    return r0, c0


def xy(G, ir, ic, y, center=None, scale=None, lists=False):
    """X.y as the GRM's views compute it: k_pmv on the sample-major copy, or the SNP-major kernels when the file holds
    a missing value (lists: the handle's missing-value lists are in use)."""
    if np.any(G == 3):
        return fx.prod_T(G, ir, ic, y, center, scale, lists=lists)
    return fx.prod_pmv(G, ir, ic, y, center, scale)


def tcrossprod(G, center, scale, ir=None, ic=None, nslices=4, path="gramt", lists=False, old_classes=False):
    """The bytes of bsg_tcrossprod on the full code matrix G (n x m, 3 = missing) with 1-based selections ir / ic
    (None = all).  Returns None where the library takes the DSYRK path (not modelled)."""
    G = np.asarray(G)
    r0, c0 = _sel(G, ir, ic)
    W1, W2p, W3, w2 = grm_weights(center, scale)
    if r0.size == 0 or c0.size == 0 or degenerate(W1, W2p, W3):
        return None
    Gs = G[np.ix_(r0, c0)]
    K = gram_fold(Gs, W1, W2p, W3, nslices, path, old_classes)
    sumW3 = float(np.cumsum(W3)[-1])
    r = xy(G, ir, ic, w2, lists=lists)
    K = ((K + r[:, None]) + r[None, :]) + sumW3
    if np.any(Gs == 3):
        ones = np.ones(c0.size)
        q = (xy(G, ir, ic, W3, ones, ones, lists=lists) - xy(G, ir, ic, W3, lists=lists)) + sumW3
        K = K - (q[:, None] + q[None, :])
    low = np.tril(np.ones(K.shape, dtype=bool))
    return np.where(low, K, K.T)


def n_classes(center, scale) -> int:
    W1 = grm_weights(center, scale)[0]
    return int(np.unique(weight_classes(W1)).size) if W1.size else 0


def exact_K(G, center, scale, ir=None, ic=None) -> np.ndarray:
    """X~ X~^T in fp64 from the scaled matrix (missing -> 0 after scaling): the reference's definition."""
    G = np.asarray(G)
    r0, c0 = _sel(G, ir, ic)
    Gs = G[np.ix_(r0, c0)].astype(np.float64)
    with np.errstate(all="ignore"):
        X = (Gs - np.asarray(center)[None, :]) / np.asarray(scale)[None, :]
    X[G[np.ix_(r0, c0)] == 3] = 0.0
    return X @ X.T
