"""The helpers of tests/svd_ref.py against matrices whose spectrum is fixed by construction (X = Q1 diag(sigma) Q2^T): the
certificates accept the exact triplets and reject a swapped value or a vector rotated by 1e-6, the block solver reaches
its stated residual, and the generators give the spectra their names promise.  No GPU."""
import numpy as np
import pytest

from tests import svd_ref as sr


def _built(n, m, sigma, seed):
    rng = np.random.default_rng(seed)
    Q1, _ = np.linalg.qr(rng.standard_normal((n, len(sigma))))
    Q2, _ = np.linalg.qr(rng.standard_normal((m, len(sigma))))
    return Q1 * sigma @ Q2.T, Q1, Q2


SIGMA = np.array([40.0, 31.0, 30.5, 12.0, 11.0, 7.0, 3.0, 2.5, 1.0, 0.5])


@pytest.mark.parametrize("n,m", [(60, 90), (90, 60)])
def test_certificates_accept_exact_and_reject_perturbed(n, m):
    X, Q1, Q2 = _built(n, m, SIGMA, 1)
    k = 5
    d, U, V = SIGMA[:k].copy(), Q1[:, :k].copy(), Q2[:, :k].copy()
    theta, r = sr.ritz_certificates(X, d, U, V)
    lam = SIGMA ** 2
    assert np.max(np.abs(theta - lam[:k]) / lam[0]) < 1e-14 and np.max(r) < 1e-12 * lam[0]
    for i in range(k):
        b = sr.eig_bound(theta[i], r[i], sr.gaps(theta[i], lam, i))
        assert abs(d[i] - SIGMA[i]) <= sr.sv_bound(d[i], SIGMA[i], b) + 1e-14 * SIGMA[0]
    assert sr.orth_error(U) < 1e-14 and sr.orth_error(V) < 1e-14
    assert sr.interlaces(theta, lam, 1e-14) and sr.ky_fan_ok(theta, lam, 1e-14)

    # a swapped value: the residual of the pair (d_1, u_2) no longer vanishes and exceeds what the bound allows
    d2 = d.copy()
    d2[[1, 2]] = d2[[2, 1]]
    row = n <= m
    S = U if row else V
    res = np.linalg.norm(sr.gram_apply(X, S[:, 1], row) - d2[1] ** 2 * S[:, 1])
    assert res > 1e3 * r[1] and abs(d2[1] - SIGMA[1]) > sr.sv_bound(d2[1], SIGMA[1], sr.eig_bound(theta[1], r[1], 1.0))

    # a side vector rotated by 1e-6 towards another singular vector: residual ~ 1e-6 (lambda_1 - lambda_4), seen
    Q = Q1 if row else Q2
    rot = np.cos(1e-6) * S[:, 0] + np.sin(1e-6) * Q[:, 3]
    S2 = S.copy()
    S2[:, 0] = rot
    U2, V2 = (S2, V) if row else (U, S2)
    _, r2 = sr.ritz_certificates(X, d, U2, V2)
    assert r2[0] > 0.5e-6 * (lam[0] - lam[3]) and r2[0] < 2e-6 * lam[0]
    assert sr.sin_angle(rot, S[:, 0]) == pytest.approx(1e-6, rel=1e-6)
    # a vector rotated inside the span of the others breaks orthonormality at the same size
    S3 = S.copy()
    S3[:, 1] = np.cos(1e-6) * S[:, 1] + np.sin(1e-6) * S[:, 0]
    assert 0.5e-6 < sr.orth_error(S3) < 2e-6


def test_interlacing_and_ky_fan_reject_values_above_the_spectrum():
    lam = SIGMA ** 2
    assert sr.interlaces(lam[:4] * (1 - 1e-9), lam) and sr.ky_fan_ok(lam[:4], lam)
    bad = lam[:4].copy()
    bad[2] = lam[1]  # a copy of the second value in third place: above lambda_3
    assert not sr.interlaces(bad, lam) and not sr.ky_fan_ok(bad, lam)
    assert not sr.interlaces(lam[:4] * (1 + 1e-9), lam)


def test_kato_temple_is_sharp_and_sound():
    # A = diag(lam); x = cos(t) e_0 + sin(t) e_1: theta - lam_0 = -sin^2 (lam_0 - lam_1), r = sin cos (lam_0 - lam_1)
    lam = np.array([10.0, 4.0, 1.0])
    for t in (1e-2, 1e-4, 1e-6):
        x = np.array([np.cos(t), np.sin(t), 0.0])
        theta = x @ (lam * x)
        r = np.linalg.norm(lam * x - theta * x)
        err = abs(theta - lam[0])
        b = sr.eig_bound(theta, r, sr.gaps(theta, lam, 0))
        slack = 4 * np.finfo(float).eps * lam[0]  # rounding of theta itself
        assert err <= b + slack and b < 1.01 * err + slack
    assert sr.eig_bound(1.0, 1e-3, 0.0) == 1e-3  # exact tie: the residual bound alone


@pytest.mark.parametrize("n,m,k", [(300, 200, 5), (150, 400, 10)])
def test_block_solver_reaches_its_residual(n, m, k):
    sigma = np.geomspace(50.0, 0.1, 60) * (1 + 0.003 * np.arange(60)[::-1] / 60)  # clustered, no tie
    X, Q1, Q2 = _built(n, m, sigma, 3)
    row = n <= m
    A = X @ X.T if row else X.T @ X
    start = sr.gaussian_start(A.shape[0], k + 10, 7)
    theta, Y, r, iters = sr.block_topk(lambda R: R @ A, start, k, tol=1e-10, max_rows=60)
    assert iters > 1 and np.max(r) <= 1e-10
    lam = sigma ** 2
    assert sr.interlaces(theta, lam, 1e-13)
    np.testing.assert_allclose(theta, lam[:k], rtol=1e-12)
    assert sr.orth_error(Y.T) < 1e-12
    Q = Q1 if row else Q2
    for i in range(k):
        assert sr.sin_angle(Y[i], Q[:, i]) < 1e-8
    # the same start with an iteration cap: residuals still reported, values still below the spectrum
    theta1, _, r1, it1 = sr.block_topk(lambda R: R @ A, start, k, tol=1e-30, maxit=2)
    assert it1 == 2 and np.max(r1) > 1e-10 and sr.interlaces(theta1, lam, 1e-13)


def test_generators_have_the_promised_spectra():
    from numpy.linalg import svd

    def scaled(G):
        X = G.astype(np.float64)
        c = X.mean(0)
        s = np.sqrt(c / 2 * (1 - c / 2))
        return (X - c) / np.where(s > 0, s, 1)

    G = sr.balding_nichols([60, 80, 100], 600, 0.1, 5)
    assert G.shape == (240, 600) and G.dtype == np.uint8 and G.max() <= 2
    s = svd(scaled(G), compute_uv=False)
    assert s[1] / s[2] > 1.5  # two structured directions above the bulk
    G = sr.symmetric_tree(60, 2000, 0.2, 5)
    s = svd(scaled(G), compute_uv=False)
    assert s[0] / s[1] < 1.05 and s[1] / s[2] < 1.05 and s[2] / s[3] > 1.5  # star-like: three near-tied values on top
    G = sr.block_copies(7, 11, 3, 5)
    s = svd(G.astype(np.float64), compute_uv=False)
    assert np.allclose(s[0:3], s[0], rtol=1e-13) and np.allclose(s[3:6], s[3], rtol=1e-13)
    assert np.sum(s > 1e-10 * s[0]) == 21
    G = sr.random_genotypes(50, 70, 5, na_rate=0.02)
    assert 0 < np.mean(G == 3) < 0.05
    idx = sr.few_distinct(6, 40, 5)
    assert idx.size == 40 and set(idx.tolist()) == set(range(1, 7))
