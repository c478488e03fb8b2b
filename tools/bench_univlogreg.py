"""big_univLogReg on one GPU (bsg_univlogreg): a logistic GWAS with covariates over a 20,000-column slice of the UK
Biobank-shaped synthetic matrix of BASELINE.json configs[4] (487,000 rows; the generator is keyed by (seed, column), so
the slice is the first 20,000 columns of the full matrix), and over a CODE_DOSAGE FBM at n = 50,000.

    python tools/bench_univlogreg.py [--n 487000] [--m 20000] [--n-dosage 50000] [--m-dosage 20000] [--out DIR]

Cases: covariates = intercept + 11 and intercept + 21 random columns (U with K = 12 and 22 columns, so H is 13 x 13 and
23 x 23), with ind.train = all rows and a random 80 % of them; a case / control phenotype from a liability threshold on
two covariates and one SNP.  Per case: the device time of the IRLS (CUDA events, bsg_univlogreg_last_ms), median and
range over 5 calls after a warm-up call; the wall time of the call; the histogram of IRLS steps; the SNPs refitted on the
host and the host time of those refits; (observation x SNP x step) per second; the fp64 multiply-adds the sums need per
(observation, SNP, step) -- (K + 1)(K + 4) / 2 for H and r plus K + 1 for eta -- as a rate against the H100 SXM data
sheet's fp64 FMA (34 TFLOP/s) and fp64 tensor (67 TFLOP/s) peaks.  The CPU figure is the NumPy restatement
(tests/logreg_ref.py) on a sample of columns, extrapolated to m.  The GPU name, power limit and SM clock are read in the
same run.  One JSON line to stdout (and DIR/bench_univlogreg.json).
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

FP64_FMA_MAC_S = 34e12 / 2     # H100 SXM data sheet, fp64 (FMA pipe), as multiply-adds
FP64_TENSOR_MAC_S = 67e12 / 2  # fp64 tensor core
SEED = 20250924 + 4            # configs[4]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def phenotype(B, X, ind_row, covar, seed):
    rng = np.random.default_rng(seed)
    x = B.read_bed(X, ind_row, [7])[:, 0].astype(np.float64) if not X.dosage_scale else \
        B.bed_prodVec(X, np.ones(1), ind_row, np.array([7], dtype=np.int32))
    x = np.where(x < 0, 0, x)
    liab = 0.3 * (x - x.mean()) + 0.5 * covar[:, 0] / np.std(covar[:, 0]) + rng.normal(size=ind_row.size)
    return (liab > np.quantile(liab, 0.7)).astype(np.float64)


def case(B, X, ind_row, K, seed, reps):
    from bigsnpr_b200.api import logit_glm_fit

    nr = ind_row.size
    rng = np.random.default_rng(seed)
    covar = rng.normal(size=(nr, K - 1))
    y = phenotype(B, X, ind_row, covar, seed)
    B.big_univLogReg(X, y, ind_train=ind_row, covar_train=covar)  # warm-up
    ms, wall = [], []
    for _ in range(reps):
        t0 = time.time()
        res = B.big_univLogReg(X, y, ind_train=ind_row, covar_train=covar)
        wall.append(time.time() - t0)
        ms.append(B.api.univlogreg_last_ms())
    m = X.ncol
    ok = ~np.isnan(res.estim)
    steps = res.niter[ok & ~res.refitted]
    hist = {int(k): int(v) for k, v in zip(*np.unique(steps, return_counts=True))}
    # the refits again, timed alone (the same host code the call runs)
    U = B.api.univlinreg_covar_basis(covar, nr)
    t0 = time.time()
    for c in np.flatnonzero(res.refitted):
        x = B.api._decode_column(X, ind_row, int(c) + 1)
        logit_glm_fit(np.column_stack([U, x]), y)
    refit_s = time.time() - t0
    # device work: every SNP steps through the observations once per IRLS step (refitted SNPs: maxiter steps)
    total_steps = int(steps.sum()) + int(res.refitted.sum()) * 20
    obs_snp_steps = float(nr) * total_steps
    P = K + 1
    macs = obs_snp_steps * (P * (P + 3) / 2 + P)
    med = float(np.median(ms)) / 1e3
    return dict(K=K, nr=int(nr), m=int(m), device_ms_median=float(np.median(ms)),
                device_ms_range=[float(min(ms)), float(max(ms))], wall_s_median=float(np.median(wall)),
                niter_histogram=hist, refitted=int(res.refitted.sum()), refit_host_s=refit_s,
                nan_columns=int((~ok).sum()), obs_snp_steps_per_s=obs_snp_steps / med, fp64_macs=macs,
                fp64_mac_rate=macs / med, share_of_fma_peak=macs / med / FP64_FMA_MAC_S,
                share_of_tensor_peak=macs / med / FP64_TENSOR_MAC_S)


def cpu_figure(n, m_total, K, seed):
    from tests import logreg_ref as L

    rng = np.random.default_rng(seed)
    Xs = rng.binomial(2, 0.3, size=(n, 20)).astype(np.float64)
    covar = rng.normal(size=(n, K - 1))
    y = (rng.random(n) < 0.3).astype(np.float64)
    U = L.covar_basis(covar, n)
    g0 = L.glm_fit(U, y)[0]
    t0 = time.time()
    L.irls(Xs, y, U, g0)
    dt = time.time() - t0
    return dict(columns=20, n=n, K=K, seconds=dt, extrapolated_s=dt * m_total / 20, threads=os.cpu_count())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=487_000)
    ap.add_argument("--m", type=int, default=20_000)
    ap.add_argument("--n-dosage", type=int, default=50_000)
    ap.add_argument("--m-dosage", type=int, default=20_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import bigsnpr_b200 as B

    res = dict(tool="bench_univlogreg", gpu=gpu_info(), cases=[])
    X = B.Bed.synthetic(a.n, a.m, seed=SEED)
    rng = np.random.default_rng(1)
    sub = np.sort(rng.choice(a.n, int(0.8 * a.n), replace=False)).astype(np.int32) + 1
    for K in (12, 22):
        for name, rows in (("all rows", X.rows_along()), ("80% of rows", sub)):
            c = case(B, X, rows, K, seed=K, reps=a.reps)
            c.update(matrix="configs[4] %d rows, first %d columns" % (a.n, a.m), ind_train=name)
            res["cases"].append(c)
            print(json.dumps(c), file=sys.stderr)
    del X
    code256 = np.full(256, np.nan)
    code256[:201] = np.arange(201) / 100
    byt = rng.integers(0, 201, size=(a.n_dosage, a.m_dosage), dtype=np.uint8)
    F = B.Bed.from_fbm(byt, code256)
    del byt
    for K in (12,):
        c = case(B, F, F.rows_along(), K, seed=100 + K, reps=a.reps)
        c.update(matrix="CODE_DOSAGE FBM %d x %d" % (a.n_dosage, a.m_dosage), ind_train="all rows")
        res["cases"].append(c)
        print(json.dumps(c), file=sys.stderr)
    res["cpu_numpy_restatement"] = cpu_figure(a.n, a.m, 12, 5)
    res["gpu_after"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_univlogreg.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
