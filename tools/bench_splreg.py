"""big_spLinReg / big_spLogReg on one GPU (bsg_splreg) over a slice of the LD-structured synthetic generator of
BASELINE.json configs[4] (keyed by (seed, column): the first m columns at n rows), against the C oracle
(tests/splreg_oracle.c, the same algorithm and arithmetic) on all host cores.

    python tools/bench_splreg.py [--n 100000] [--m 1000] [--m-cpu 100] [--reps 2] [--out DIR]

Workload: a phenotype with 1 % of the columns causal (normal effects, heritability 0.3 on the liability), 10 PCs from
bed_randomSVD as covariates, K = 10, alphas = (1, 0.01, 1e-4) (30 fits), bigstatsr's path defaults; the logistic
phenotype is the liability thresholded at 30 % cases.  Per family and call: the device time (CUDA events,
bsg_splreg_last_ms; every repetition listed), lambda steps and coordinate-descent passes per fit, and the stop messages.
The CPU figure is the C oracle on all cores (one fit per thread) over the first --m-cpu columns with the same rows, folds,
alphas and PCs, extrapolated linearly in columns to m (labelled as such).  The screening / descent split and the HBM
share of the screening pass are not instrumented (not measured).  The GPU name, power limit and SM clock and the host
core count are read in the same run.  Progress goes to stderr; one JSON line to stdout (and DIR/bench_splreg.json).
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

SEED = 20250924 + 4  # configs[4]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def log(msg):
    print(msg, file=sys.stderr, flush=True)


def run(B, fn, X, y, pcs, reps):
    dev = []
    for _ in range(reps):
        mod = fn(X, y, covar_train=pcs, K=10, alphas=(1.0, 0.01, 1e-4))
        dev.append(B.api.splreg_last_ms() / 1e3)
        log("  call: %.2f s of device time" % dev[-1])
    steps = mod.nb_lambda.reshape(-1)
    passes = np.array([p["passes"].sum() for row in mod.path for p in row])
    return dict(device_s=dev, lambda_steps_per_fit=dict(min=int(steps.min()), median=float(np.median(steps)),
                max=int(steps.max())), passes_per_fit=dict(min=int(passes.min()), median=float(np.median(passes)),
                max=int(passes.max())), messages=sorted(set(m for row in mod.message for m in row)),
                validation_loss=[float(v) for v in mod.validation_loss], nb_var=[int(v) for v in mod.nb_var],
                best_alpha=float(mod.alphas[mod.best_alpha])), mod


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--m", type=int, default=1_000)
    ap.add_argument("--m-cpu", type=int, default=100)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import bigsnpr_b200 as B

    X = B.Bed.synthetic(a.n, a.m, seed=SEED, ld_rho=0.9, ld_block=50)
    svd = B.bed_randomSVD(X, k=10)
    pcs = svd["u"] * svd["d"]
    rng = np.random.default_rng(1)
    causal = np.sort(rng.choice(a.m, max(1, a.m // 100), replace=False)) + 1
    Xc = B.read_bed(X, X.rows_along(), causal).astype(np.float64)
    g = (Xc - Xc.mean(0)) @ rng.normal(size=causal.size)
    g = g / np.std(g) * np.sqrt(0.3)
    liab = g + rng.normal(size=a.n) * np.sqrt(0.7)
    y01 = (liab > np.quantile(liab, 0.7)).astype(np.float64)
    res = dict(gpu=gpu_info(), host_cores=os.cpu_count(), n=a.n, m=a.m, K=10, alphas=[1, 0.01, 1e-4], covariates=10)
    log("matrix and PCs ready")
    res["linear"], mod = run(B, B.big_spLinReg, X, liab, pcs, a.reps)
    log("linear: %s" % json.dumps(res["linear"]))
    res["logistic"], _ = run(B, B.big_spLogReg, X, y01, pcs, a.reps)
    log("logistic: %s" % json.dumps(res["logistic"]))

    from tests import splreg_ref as S

    Xs = B.read_bed(X, X.rows_along(), np.arange(1, a.m_cpu + 1)).astype(np.float64)
    t0 = time.time()
    S.splreg(Xs, liab, 0, mod.ind_sets, 10, covar=pcs, alphas=(1.0, 0.01, 1e-4), engine="c")
    sec = time.time() - t0
    res["cpu_c_oracle"] = dict(what="tests/splreg_oracle.c on all %d host cores, linear, %d rows x first %d columns + "
                                    "10 PCs, K = 10, 3 alphas" % (os.cpu_count(), a.n, a.m_cpu), seconds=sec,
                               extrapolated_to_m_s=sec * a.m / a.m_cpu)
    log("cpu: %s" % json.dumps(res["cpu_c_oracle"]))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_splreg.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
