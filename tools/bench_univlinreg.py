"""big_univLinReg on one GPU (bsg_univlinreg): a linear GWAS with covariates over every SNP of the UK Biobank-shaped
synthetic matrix of BASELINE.json configs[4] (487,000 x 500,000, SNP-major copy only), and over a CODE_DOSAGE FBM at
n = 50,000.

    python tools/bench_univlinreg.py [--n 487000] [--m 500000] [--n-dosage 50000] [--m-dosage 20000] [--out DIR]

Cases: covariates = intercept + 10 and intercept + 20 random orthonormal columns (K = 11, 21), with ind.train = all rows and
a random 80 % of them.  Per case: the device time of the call (CUDA events, vector upload to the statistics,
bsg_univlinreg_last_ms), median and range over 5 calls after a warm-up call; the bytes of X read (one read of the selected
SNP-major lines per pass of at most 64 digit slices) and that rate against the H100 SXM data sheet's 3.35 TB/s; the
MACs issued on the tensor pipe (4 codes per byte x the pass's 8-slice tiles) against the data sheet's 1,979 dense int8
TOP/s; which of the two bounds it.  The baseline, on the same handle in the same run, is the route the engine had: K + 1
bed_cprodVec calls (X'y and X'u_k) plus the same algebra on the host, timed on the wall clock, with the largest
|score| difference between the two routes.  The CPU figure is the literal fp64 statistic (tests/gwas_ref.py) on a sample
of columns, extrapolated to m.  The GPU name, power limit and SM clock are read in the same run.
One JSON line to stdout (and DIR/bench_univlinreg.json).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_S = 3.35e12    # H100 SXM data sheet
INT8_MAC_S = 1979e12 / 2  # dense int8 TOP/s of the data sheet, as MACs
SEED = 20250924 + 4       # configs[4]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def passes_tiles(K):
    """8-slice tiles of each pass: y = 8 digit slices, each covariate vector 4, at most 64 slices per pass."""
    sizes, used = [], 64
    for v in range(K + 1):
        nd = 8 if v == 0 else 4
        if used + nd > 64:
            sizes.append(0)
            used = 0
        sizes[-1] += nd
        used += nd
    return [-(-s // 8) for s in sizes]


def orthonormal_covar(n, k, seed):
    q, _ = np.linalg.qr(np.random.default_rng(seed).normal(size=(n, k)))
    return q


def host_stats(S, cnt, U, y, nr):
    """The statistic from K + 1 plain products (the baseline's host algebra, centred form)."""
    K = U.shape[1]
    yc = y - y.mean()
    u1, uy = U.sum(axis=0), U.T @ yc
    sx = cnt[1] + 2.0 * cnt[2]
    sxx = cnt[1] + 4.0 * cnt[2]
    mx = sx / nr
    ssx = sxx - sx * mx
    T = S[1:] - np.outer(u1, mx)
    den = ssx - np.sum(T * T, axis=0)
    num = (S[0] - mx * yc.sum()) - uy @ T
    with np.errstate(invalid="ignore", divide="ignore"):
        b = num / den
        rss = (yc @ yc - uy @ uy) - b * num
        se = np.sqrt(rss / (nr - K - 1) / den)
    bad = (cnt[3] > 0) | (den <= 0)
    b[bad] = np.nan
    se[bad] = np.nan
    return b / se


def case(B, X, ind_row, K, seed, reps, baseline=True, dos=False):
    nr = ind_row.size
    rng = np.random.default_rng(seed)
    covar = orthonormal_covar(nr, K - 1, seed) * np.sqrt(nr)
    y = rng.normal(size=nr)
    B.big_univLinReg(X, y, ind_train=ind_row, covar_train=covar)  # warm-up
    ms, wall = [], []
    for _ in range(reps):
        t0 = time.time()
        res = B.big_univLinReg(X, y, ind_train=ind_row, covar_train=covar)
        wall.append(time.time() - t0)
        ms.append(B.api.univlinreg_last_ms())
    m = X.ncol
    tiles = passes_tiles(K)
    nbytes_line = (X.nrow + 3) // 4 if not dos else X.nrow
    bytes_read = len(tiles) * m * nbytes_line
    macs = sum(tiles) * 8 * m * (-(-X.nrow // 512) * 512)
    med = float(np.median(ms)) / 1e3
    t_hbm, t_mma = bytes_read / HBM_BYTES_S, macs / INT8_MAC_S
    out = dict(K=K, nr=int(nr), passes=len(tiles), tiles=tiles, device_ms_median=float(np.median(ms)),
               device_ms_range=[float(min(ms)), float(max(ms))], wall_s_median=float(np.median(wall)),
               bytes_read=int(bytes_read), hbm_share=t_hbm / med, macs=int(macs), mma_share=t_mma / med,
               bound="HBM" if t_hbm >= t_mma else "tensor pipe (data sheet)", nan_columns=int(np.isnan(res.score).sum()))
    if baseline and not dos:
        U = B.api.univlinreg_covar_basis(covar, nr)
        t0 = time.time()
        S = np.stack([B.bed_cprodVec(X, y - y.mean(), ind_row=ind_row)] +
                     [B.bed_cprodVec(X, U[:, k], ind_row=ind_row) for k in range(U.shape[1])])
        cnt = B.bed_counts(X, ind_row=ind_row)
        score = host_stats(S, cnt, U, y, nr)
        tb = time.time() - t0
        ok = ~np.isnan(score) & ~np.isnan(res.score)
        out.update(baseline_wall_s=tb, baseline_calls=U.shape[1] + 1, speedup_vs_baseline_wall=tb / float(np.median(wall)),
                   max_abs_score_diff=float(np.max(np.abs(score[ok] - res.score[ok]))),
                   max_abs_score=float(np.max(np.abs(res.score[ok]))))
    return out


def cpu_figure(n, m_total, K, seed):
    from tests import gwas_ref as G

    rng = np.random.default_rng(seed)
    Xs = rng.binomial(2, 0.3, size=(n, 50)).astype(np.float64)
    U = G.covar_basis(rng.normal(size=(n, K - 1)), n)
    y = rng.normal(size=n)
    t0 = time.time()
    G.univlinreg_fp64(Xs, y, U)
    dt = time.time() - t0
    return dict(columns=50, n=n, K=K, seconds=dt, extrapolated_s=dt * m_total / 50)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=487_000)
    ap.add_argument("--m", type=int, default=500_000)
    ap.add_argument("--n-dosage", type=int, default=50_000)
    ap.add_argument("--m-dosage", type=int, default=20_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import bigsnpr_b200 as B

    res = dict(tool="bench_univlinreg", gpu=gpu_info(), cases=[])
    X = B.Bed.synthetic(a.n, a.m, seed=SEED)
    rng = np.random.default_rng(1)
    sub = np.sort(rng.choice(a.n, int(0.8 * a.n), replace=False)).astype(np.int32) + 1
    for K in (11, 21):
        for name, rows in (("all rows", X.rows_along()), ("80% of rows", sub)):
            c = case(B, X, rows, K, seed=K, reps=a.reps)
            c.update(matrix="configs[4] %d x %d" % (a.n, a.m), ind_train=name)
            res["cases"].append(c)
            print(json.dumps(c), file=sys.stderr)
    del X
    code256 = np.full(256, np.nan)
    code256[:201] = np.arange(201) / 100
    byt = rng.integers(0, 201, size=(a.n_dosage, a.m_dosage), dtype=np.uint8)
    F = B.Bed.from_fbm(byt, code256)
    del byt
    for K in (11, 21):
        c = case(B, F, F.rows_along(), K, seed=100 + K, reps=a.reps, dos=True)
        c.update(matrix="CODE_DOSAGE FBM %d x %d" % (a.n_dosage, a.m_dosage), ind_train="all rows")
        res["cases"].append(c)
        print(json.dumps(c), file=sys.stderr)
    res["cpu_fp64_restatement"] = cpu_figure(a.n, a.m, 11, 5)
    res["gpu_after"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_univlinreg.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
