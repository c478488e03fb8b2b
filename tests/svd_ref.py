"""Plain NumPy references for the Lanczos driver behind bed_randomSVD (bsg_la.cu, lanczos_svd): test matrices with a known
kind of spectrum, the dense truth, a posteriori certificates for a computed (d, U, V), and an independent top-k solver.

Generators return uint8 code matrices (n x m, 0 / 1 / 2 and 3 for a missing value), seeded:
  * balding_nichols: P subpopulations drawn from one ancestral frequency per SNP with drift F_ST (well separated top values);
  * symmetric_tree: four leaves of the same size and the same drift from one root (two clades with no drift between
    them): the three contrasts between leaves carry the same variance, a near tie sigma_1 ~ sigma_2 ~ sigma_3;
  * block_copies: G copies of one random block on the diagonal, zero elsewhere; with identity scaling (center 0, scale 1)
    every singular value of the block appears exactly G times;
  * few_distinct: r distinct rows (or columns); a multiset ind_row / ind_col over them gives a rank-deficient X~.

Certificates work on the Gram operator the driver iterates on: A = X~ X~^T (row side, n <= m) or X~^T X~ (column side).
For a unit vector x with Rayleigh quotient theta and residual r = |A x - theta x|, a symmetric A has an eigenvalue within r
of theta, and within r^2 / gap when no other eigenvalue is closer than gap (Kato-Temple); the angle to that eigenvector
is at most r / gap (Davis-Kahan).  Ritz values of any subspace interlace with the spectrum (theta_i <= lambda_i) and their
top-k sum is at most the top-k eigenvalue sum (Ky Fan).

block_topk is randomized block Krylov with a seeded Gaussian start of k + 10 columns, fp64 QR and Rayleigh-Ritz over the
whole basis, restarted from its top Ritz vectors when the basis reaches a size cap.  It is written over an abstract matvec
on vectors stored as rows and over the array module `xp` (numpy here, torch on the device), so the same code certifies the
driver where no dense SVD fits.
"""
from __future__ import annotations

import numpy as np

EPS23 = np.finfo(np.float64).eps ** (2.0 / 3.0)  # ARPACK / Spectra: |Ritz residual| <= tol * max(eps^(2/3), |theta|)


# ---- generators --------------------------------------------------------------------------------------------------------
def _genotypes(rng, p_rows, na_rate):
    """Binomial(2, p) calls for a (n, m) matrix of allele frequencies, then a fraction na_rate set missing (code 3)."""
    G = rng.binomial(2, p_rows).astype(np.uint8)
    if na_rate > 0:
        G[rng.random(G.shape) < na_rate] = 3
    return G


def _drift(rng, p, f):
    """Balding-Nichols draw around frequencies p with drift f: Beta(p (1 - f) / f, (1 - p) (1 - f) / f)."""
    if f <= 0:
        return p.copy()
    a = p * (1 - f) / f
    return rng.beta(a, a * (1 - p) / p)


def balding_nichols(sizes, m, fst, seed, na_rate=0.0):
    rng = np.random.default_rng(seed)
    p0 = rng.uniform(0.05, 0.95, size=m)
    rows = np.concatenate([np.broadcast_to(_drift(rng, p0, fst), (s, m)) for s in sizes])
    return _genotypes(rng, rows, na_rate)


def symmetric_tree(n_leaf, m, f_leaf, seed, na_rate=0.0):
    rng = np.random.default_rng(seed)
    p0 = rng.uniform(0.1, 0.9, size=m)
    rows = [np.broadcast_to(_drift(rng, p0, f_leaf), (n_leaf, m)) for _ in range(4)]
    return _genotypes(rng, np.concatenate(rows), na_rate)


def block_copies(nb, mb, copies, seed):
    rng = np.random.default_rng(seed)
    blk = rng.integers(0, 3, size=(nb, mb)).astype(np.uint8)
    G = np.zeros((nb * copies, mb * copies), dtype=np.uint8)
    for c in range(copies):
        G[c * nb:(c + 1) * nb, c * mb:(c + 1) * mb] = blk
    return G


def random_genotypes(n, m, seed, na_rate=0.0):
    rng = np.random.default_rng(seed)
    return _genotypes(rng, np.broadcast_to(rng.uniform(0.05, 0.5, size=m), (n, m)), na_rate)


def few_distinct(r, count, seed):
    """A 1-based multiset of `count` draws from 1..r, each of the r values at least once."""
    rng = np.random.default_rng(seed)
    idx = np.concatenate([np.arange(1, r + 1), rng.integers(1, r + 1, size=count - r)])
    return rng.permutation(idx).astype(np.int32)


# ---- dense truth ---------------------------------------------------------------------------------------------------------
def dense_scaled(oracle, codes, ind_row, ind_col, center, scale):
    """X~ as the reference reads it (missing values become 0 after scaling): oracle.read_bed_scaled on the packed codes."""
    n, m = codes.shape
    o = oracle.OracleBed.from_packed(oracle.write_bed_bytes(codes), n, m)
    return oracle.read_bed_scaled(o, ind_row, ind_col, center, scale)


def dense_svd(X):
    U, s, Vt = np.linalg.svd(X, full_matrices=False)
    return s, U, Vt.T


def numerical_rank(s, rel=1e-10):
    return int(np.sum(s > rel * s[0])) if s.size and s[0] > 0 else 0


# ---- certificates ------------------------------------------------------------------------------------------------------
def side_vectors(n, m, U, V, row_side=None):
    """The vectors of the side the driver iterates on (rows when n <= m) and whether it is the row side."""
    row = (n <= m) if row_side is None else row_side
    return (U if row else V), row


def gram_apply(X, x, row):
    return X @ (X.T @ x) if row else X.T @ (X @ x)


def ritz_certificates(X, d, U, V, row_side=None):
    """Per computed triplet: Rayleigh quotient theta_i and residual r_i = |A x_i - theta_i x_i| of the unit side vector."""
    n, m = X.shape
    S, row = side_vectors(n, m, U, V, row_side)
    S = S / np.linalg.norm(S, axis=0)
    AS = gram_apply(X, S, row)
    theta = np.sum(S * AS, axis=0)
    r = np.linalg.norm(AS - S * theta, axis=0)
    return theta, r


def gaps(theta, lam, i):
    """Distance from theta to the nearest eigenvalue of the full spectrum `lam` other than lam[i]."""
    others = np.delete(np.asarray(lam, dtype=np.float64), i)
    return float(np.min(np.abs(others - theta))) if others.size else np.inf


def eig_bound(theta, r, gap):
    """|theta - lambda| <= min(r, r^2 / gap): the residual bound, sharpened by Kato-Temple when the gap is known."""
    return min(r, r * r / gap) if gap > 0 else r


def sv_bound(d, sigma, theta_bound):
    """The same bound moved to singular values: |d - sigma| = |d^2 - sigma^2| / (d + sigma)."""
    return theta_bound / max(d + sigma, np.finfo(np.float64).tiny)


def orth_error(Q):
    """|Q^T Q - I|_2"""
    Q = np.asarray(Q, dtype=np.float64)
    return float(np.linalg.norm(Q.T @ Q - np.eye(Q.shape[1]), 2))


def sin_angle(x, y):
    """sin of the angle between two vectors (|x - (x.y) y| for unit vectors, accurate near 0)."""
    x, y = x / np.linalg.norm(x), y / np.linalg.norm(y)
    return float(np.linalg.norm(x - (x @ y) * y))


def interlaces(theta, lam, rel=0.0):
    """Ritz values of a subspace lie below the eigenvalues of the same rank: theta_i <= lambda_i (1 + rel)."""
    theta, lam = np.sort(theta)[::-1], np.sort(lam)[::-1][:len(theta)]
    return bool(np.all(theta <= lam * (1 + rel) + np.finfo(np.float64).tiny))


def ky_fan_ok(theta, lam, rel=0.0):
    """sum of the top-k Ritz values <= sum of the top-k eigenvalues (1 + rel)."""
    k = len(theta)
    return float(np.sum(theta)) <= float(np.sum(np.sort(lam)[::-1][:k])) * (1 + rel)


# ---- independent top-k: restarted randomized block Krylov ----------------------------------------------------------------
def gaussian_start(N, b, seed):
    return np.random.default_rng(seed).standard_normal((b, N))


def _orth_rows(xp, W, Q=None):
    """Rows of W orthonormalised (fp64 QR), first against the rows of Q (block Gram-Schmidt, twice)."""
    if Q is not None:
        for _ in range(2):
            W = W - (W @ Q.T) @ Q
    q, _ = xp.linalg.qr(W.T)
    return q.T


def _zeros_like_rows(like, rows):
    return like.new_zeros((rows, like.shape[1])) if hasattr(like, "new_zeros") else np.zeros((rows, like.shape[1]))


def _top(xp, w, S, k):
    """the k largest eigenpairs of eigh's ascending output, largest first"""
    if hasattr(S, "flip"):
        return w[-k:].flip(0), S[:, -k:].flip(1)
    return w[::-1][:k], S[:, ::-1][:, :k]


def block_topk(matvec, start, k, tol=1e-8, max_rows=600, maxit=400, xp=np, progress=None):
    """Top-k eigenpairs of the symmetric PSD operator `matvec` (rows in, rows out): returns (theta, Y, r, iters) with Y
    the k Ritz vectors as rows and r their residuals |A y - theta y| relative to theta_1.  Stops when max r <= tol.
    The basis and its products live in two preallocated buffers of max_rows rows."""
    Q = _orth_rows(xp, start)
    b = Q.shape[0]
    Qbuf, Pbuf = _zeros_like_rows(Q, max_rows), _zeros_like_rows(Q, max_rows)
    Qbuf[:b] = Q
    nq = b  # rows of the basis; the products of all of them are known after each matvec below
    theta = Y = r = None
    for it in range(1, maxit + 1):
        Pbuf[nq - b:nq] = matvec(Qbuf[nq - b:nq])
        Qa, AQa = Qbuf[:nq], Pbuf[:nq]
        H = Qa @ AQa.T
        H = 0.5 * (H + H.T)
        w, S = xp.linalg.eigh(H)
        theta, top = _top(xp, w, S, k)
        Y, AY = top.T @ Qa, top.T @ AQa
        r = ((AY - theta[:, None] * Y) ** 2).sum(1) ** 0.5 / theta[0]
        if progress is not None:
            progress(it, r)
        if float(r.max()) <= tol:
            return theta, Y, r, it
        if nq + b > max_rows:  # restart from the top b Ritz vectors; their products are known
            _, keep = _top(xp, w, S, b)
            Qk, Pk = keep.T @ Qa, keep.T @ AQa
            Qbuf[:b], Pbuf[:b] = Qk, Pk
            nq = b
        Qbuf[nq:nq + b] = _orth_rows(xp, Pbuf[nq - b:nq], Qbuf[:nq])
        nq += b
    return theta, Y, r, maxit
