"""snp_grid_stacking's host side (R/SCT.R:266-304) without a GPU: the fold from stacking weights to per-SNP effects
(api.stacking_fold) against a literal restatement of R/SCT.R:287-296, the SCT identity multi_PRS @ w == X @ beta.G on
scores from tests/prs_ref.py, and how snp_grid_stacking assembles R's list from a fitted model."""
import numpy as np
import pytest

from bigsnpr_b200 import api
from tests import prs_ref as P


def r_fold(beta_stacking, lpS, lpS_thr, beta_gwas, all_keep):
    """R/SCT.R:287-296 statement by statement, 1-based like R; NA is None.  R's cumsum adds in long double."""
    ind_last_thr = [None if np.isnan(lp) else 1 + sum(1 for t in lpS_thr if lp > t) for lp in lpS]
    coef = [0.0] * len(beta_gwas)
    n_thr_pval = len(lpS_thr)
    ind = list(range(1, n_thr_pval + 1))
    for ind_keep in [k for chrom in all_keep for k in chrom]:
        b = [beta_stacking[i - 1] for i in ind]
        acc, b2 = np.longdouble(0), [0.0]
        for v in b:
            acc = acc + np.longdouble(v)
            b2.append(float(acc))
        new = list(coef)  # coef[ind.keep] <- coef[ind.keep] + ...: the right side reads coef before the assignment
        for i in ind_keep:
            li = ind_last_thr[i - 1]
            new[i - 1] = coef[i - 1] + (np.nan if li is None else b2[li - 1])
        coef = new
        ind = [i + n_thr_pval for i in ind]
    return np.array([c * b for c, b in zip(coef, beta_gwas)])


def _same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape
    assert np.array_equal(a.view(np.int64), b.view(np.int64))


def _keep_sets(rng, m, chroms, nsets, frac=0.3):
    """chromosome-major keep sets: per chromosome, nsets sorted subsets of its SNPs (1-based)"""
    bounds = np.linspace(0, m, len(chroms) + 1).astype(int)
    out = []
    for c, (b, e) in enumerate(zip(bounds[:-1], bounds[1:])):
        if chroms[c] == "empty":
            out.append([np.zeros(0, dtype=np.int64) for _ in range(nsets)])
        else:
            out.append([np.sort(rng.choice(np.arange(b, e), int(frac * (e - b)), replace=False)) + 1
                        for _ in range(nsets)])
    return out


@pytest.mark.parametrize("seed", range(6))
def test_fold_matches_r_loop(seed):
    rng = np.random.default_rng(seed)
    m, nsets = 400, 5
    thr = np.round(np.linspace(0.1, 4, 9), 1)                   # lp in 0.1 steps: some equal a threshold exactly
    lpS = np.round(rng.uniform(0, 5, m), 1)
    betas = rng.normal(size=m)
    all_keep = _keep_sets(rng, m, ["full", "empty", "full", "full"], nsets)
    inside = np.unique(np.concatenate([s for c in all_keep for s in c]))
    outside = np.setdiff1d(np.arange(1, m + 1), inside)
    lpS[outside[:10] - 1] = np.nan                              # NaN lpS outside every keep set
    betas[inside[:3] - 1] = np.nan                              # NaN betas inside and outside the sets
    betas[outside[10:13] - 1] = np.nan
    assert np.any(lpS[inside - 1][:, None] == thr[None, :])
    w = rng.normal(size=4 * nsets * thr.size)
    w[rng.choice(w.size, w.size // 5, replace=False)] = 0.0     # dropped (constant) columns have weight 0
    got = api.stacking_fold(w, lpS, thr, betas, all_keep)
    _same(got, r_fold(w, lpS, thr, betas, all_keep))
    assert np.isnan(got[inside[:3] - 1]).all()
    assert np.isnan(got[outside[10:13] - 1]).all()              # 0 * NaN
    assert (got[outside[:10] - 1] == 0).all()


def test_fold_nan_lpS_inside_a_set_is_nan():
    lpS = np.array([1.0, np.nan, 3.0])
    got = api.stacking_fold(np.array([1.0, 2.0]), lpS, np.array([0.5, 2.0]), np.ones(3), [[np.array([1, 2, 3])]])
    _same(got, r_fold([1.0, 2.0], lpS, [0.5, 2.0], np.ones(3), [[[1, 2, 3]]]))
    assert np.isnan(got[1]) and got[0] == 1.0 and got[2] == 3.0


def test_fold_refuses_wrong_width():
    with pytest.raises(ValueError):
        api.stacking_fold(np.zeros(5), np.zeros(3), np.array([0.5, 2.0]), np.ones(3), [[np.array([1, 2])]])


def test_sct_identity():
    """multi_PRS @ w == X @ beta.G: the fold turns a weighting of the C+T scores into one of the SNPs."""
    rng = np.random.default_rng(11)
    n, m = 300, 500
    G = rng.integers(0, 3, size=(n, m)).astype(np.uint8)
    lpS = rng.exponential(1.5, size=m)
    betas = rng.normal(scale=0.1, size=m)
    thr = 0.9999 * api.seq_log(0.1, float(lpS.max()), 12)
    all_keep = _keep_sets(rng, m, ["full", "empty", "full"], 4)
    ind_row = np.arange(1, n + 1)
    multi = P.grid(G, ind_row, all_keep, betas, lpS, thr, fn=P.literal)
    w = rng.normal(size=multi.shape[1])
    lhs = multi @ w
    rhs = G.astype(np.float64) @ api.stacking_fold(w, lpS, thr, betas, all_keep)
    np.testing.assert_allclose(lhs, rhs, rtol=0, atol=1e-12 * np.abs(multi).sum(axis=1).max() * np.abs(w).max())


class _Fake:
    def __init__(self, family):
        self.family, self.calls = family, []

    def __call__(self, X, y, **kw):
        self.calls.append((self.family, X, y, kw))
        nc = X.shape[1]
        kept = np.flatnonzero(np.arange(nc) % 3 != 1) + 1          # every third column dropped
        Kc = 0 if kw.get("covar_train") is None else np.asarray(kw["covar_train"]).shape[1]
        A = np.atleast_1d(kw["alphas"]).size
        beta = np.arange(1.0, 1.0 + A * (kept.size + Kc)).reshape(A, -1)
        return api.SpModel(alphas=np.atleast_1d(kw["alphas"]), intercept=0.5 - np.arange(A), beta=beta,
                           validation_loss=A - np.arange(A, dtype=float), nb_var=np.ones(A), message=[[]] * A,
                           ind_col=kept.astype(np.int32))


def test_stacking_assembly(monkeypatch):
    rng = np.random.default_rng(5)
    m, n = 60, 40
    lpS = rng.uniform(0, 3, m)
    all_keep = _keep_sets(rng, m, ["full", "full"], 2, frac=0.5)
    thr = np.array([0.5, 1.0, 2.0])
    multi = rng.normal(size=(n, 12)).astype(np.float32).view(api.GridPRS)
    multi.lpS, multi.grid_lpS_thr, multi.betas, multi.all_keep = lpS, thr, rng.normal(size=m), all_keep
    lin, log = _Fake(0), _Fake(1)
    monkeypatch.setattr(api, "big_spLinReg", lin)
    monkeypatch.setattr(api, "big_spLogReg", log)
    y01 = (rng.random(n) < 0.5).astype(float)
    cov = rng.normal(size=(n, 2))
    res = api.snp_grid_stacking(multi, y01, covar_train=cov, K=4)
    assert len(log.calls) == 1 and not lin.calls
    assert log.calls[0][3]["alphas"] == (1, 0.01, 0.0001) and log.calls[0][3]["K"] == 4
    mod = res["mod"]
    w = np.zeros(12)
    w[mod.ind_col - 1] = mod.beta[2][:mod.ind_col.size]       # the best alpha: the lowest validation loss
    _same(res["beta.G"], r_fold(w, lpS, thr, multi.betas, all_keep))
    _same(res["beta.covar"], mod.beta[2][mod.ind_col.size:])
    assert res["beta.covar"].size == 2 and res["intercept"] == -1.5
    api.snp_grid_stacking(multi, rng.normal(size=n), alphas=0.5)
    assert len(lin.calls) == 1 and lin.calls[0][3]["alphas"] == 0.5
    api.snp_grid_stacking(multi, np.repeat([0.0, 1.0, 2.0], [10, 10, 20]))  # three values: linear
    assert len(lin.calls) == 2
    with pytest.raises(ValueError):
        api.snp_grid_stacking(np.zeros((n, 12), dtype=np.float32), y01)


def test_dense_operand_layouts():
    F = np.asfortranarray(np.arange(24, dtype=np.float32).reshape(6, 4))
    X, dt, ld = api._dense_operand(F)
    assert X is F and dt == 0 and ld == 6
    big = np.asfortranarray(np.zeros((10, 5)))
    X, dt, ld = api._dense_operand(big[2:8, 1:4])                   # a row slice keeps the parent's leading dimension
    assert dt == 1 and ld == 10 and X.base is not None
    C_ = np.ascontiguousarray(F)
    X, dt, ld = api._dense_operand(C_)
    assert X.flags.f_contiguous and ld == 6 and np.array_equal(X, C_)
    for bad in (np.zeros((3, 3), dtype=np.int32), np.zeros((3, 3), dtype=np.float16), [[1, 2], [3, 4]]):
        with pytest.raises(TypeError):
            api._dense_operand(bad)
    with pytest.raises(ValueError):
        api._dense_operand(np.zeros(4))
