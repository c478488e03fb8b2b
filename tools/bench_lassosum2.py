"""snp_lassosum2 on one GPU (bsg_lassosum2): the default 30 x 4 (lambda, delta) grid over one chromosome-sized LD matrix, in
both SFBM storage forms.

    python tools/bench_lassosum2.py [--n 10000] [--m 90000] [--size 2000] [--cpu-points 8] [--out DIR]

The matrix is bed_cor of an LD-structured synthetic chromosome (m SNPs, n samples, a window of `size` SNPs each side),
built on the device.  Sumstats are simulated from it: beta = R b + e / sqrt(N) with sparse causal effects b and per-SNP
n_eff.  Per form: the wall time of as_SFBM (host storage build plus staging) and of the snp_lassosum2 call (after a
warm-up on a slice), and the device seconds of every grid point.  Counted work comes from the CPU oracle
(tests/lassosum2_oracle.c) on a stated subset of grid points (evenly spaced, plus the GPU's slowest point): sweeps, column updates (coordinates that
moved) and the corr bytes those updates read.  The oracle runs those points in parallel, one per core; the all-core CPU
figure for the whole grid is extrapolated as (sum of their times) x (120 / points) / cores, which assumes perfect load
balance; the slowest sampled point's time (the GPU's slowest point is sampled) is reported beside it as a lower bound for any all-core run.  The GPU columns of
those points must equal the oracle's bit for bit.  GPU name, power limit and SM clock are read in the same run.  One JSON
line to stdout (and DIR/bench_lassosum2.json).
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


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def simulated_sumstats(corr, m, seed, n_eff=50000):
    """beta = R b + e / sqrt(N): the full symmetric R from the upper CSC, 0.5 % causal SNPs, N 60-100 % of n_eff."""
    import scipy.sparse as sp

    p, i, x = corr
    U = sp.csc_matrix((x, i, p), shape=(m, m))
    rng = np.random.default_rng(seed)
    b = np.zeros(m)
    causal = rng.choice(m, m // 200, replace=False)
    b[causal] = rng.normal(size=causal.size) * np.sqrt(0.3 / causal.size)
    Rb = U @ b + U.T @ b - U.diagonal() * b
    N = np.round(n_eff * rng.uniform(0.6, 1.0, m))
    se = 1 / np.sqrt(N)
    return {"beta": Rb + rng.normal(size=m) * se, "beta_se": se, "n_eff": N}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10000)
    ap.add_argument("--m", type=int, default=90000)
    ap.add_argument("--size", type=int, default=2000, help="window, in SNPs each side (positions 1 kb apart)")
    ap.add_argument("--maxiter", type=int, default=1000)
    ap.add_argument("--cpu-points", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import bigsnpr_b200 as B
    from bigsnpr_b200 import api
    from tests import lassosum2_ref as L

    n, m = args.n, args.m
    res = {"n": n, "m": m, "window_snps_each_side": args.size, "grid": "30 lambda x 4 delta (defaults)",
           "maxiter": args.maxiter, "gpu_start": gpu_info()}
    g = B.Bed.synthetic(n, m, seed=21, ld_rho=0.9, ld_block=50)
    t0 = time.time()
    corr = B.bed_cor(g, size=args.size)
    res["bed_cor_s"] = round(time.time() - t0, 2)
    g.close()
    df = simulated_sumstats(corr, m, 4)
    res["nnz_upper"] = int(corr[0][-1])

    # warm-up: a 2,000-SNP slice, a short grid
    ps = corr[0][:2001]
    sl = (ps, corr[1][:ps[-1]], corr[2][:ps[-1]])
    sf = B.as_SFBM(sl)
    B.snp_lassosum2(sf, {k: v[:2000] for k, v in df.items()}, nlambda=4, maxiter=20)
    sf.close()

    kw = dict(maxiter=args.maxiter)
    spaced = np.linspace(0, 119, args.cpu_points).round().astype(int)
    bh, sc, lam, dp1, gl, gd = L.grid_inputs(df)
    for compact in (False, True):
        key = "compact" if compact else "non_compact"
        t0 = time.time()
        st = api.sfbm_storage(corr, compact=compact)
        t_host = time.time() - t0
        t0 = time.time()
        sf = api.SFBM(st[0], st[0], st[1], st[2], st[3])
        t_stage = time.time() - t0
        t0 = time.time()
        out = B.snp_lassosum2(sf, df, **kw)
        wall = time.time() - t0
        sf.close()
        gp = out.grid_param
        nnz = int(st[1][-1])
        bytes_per_value = 12 if not compact else 8  # int32 row + fp64 value, or the value alone
        r = {"nnz": nnz, "device_bytes": nnz * bytes_per_value + 8 * (m + 1) + (4 * m if compact else 0),
             "as_SFBM_host_build_s": round(t_host, 2), "as_SFBM_staging_s": round(t_stage, 2),
             "lassosum2_wall_s": round(wall, 3), "point_device_s": [round(float(t), 4) for t in gp["time"]],
             "slowest_point": int(np.argmax(gp["time"])), "slowest_point_s": round(float(np.max(gp["time"])), 3),
             "num_iter": gp["num_iter"].tolist(), "diverged_points": int(np.isnan(np.asarray(out)).any(0).sum())}
        # the oracle on the subset of points (the evenly spaced ones and the GPU's slowest): counts, CPU time, bit-identity
        pts = np.union1d(spaced, [int(np.argmax(gp["time"]))])
        even = np.isin(pts, spaced)
        la, dp = np.asfortranarray(lam[:, pts]), np.asfortranarray(dp1[:, pts])
        t0 = time.time()
        ncpu = os.cpu_count() or 1
        beta, it, mv, ent, secs = L.lassosum2(st, bh, np.arange(m), la, dp, 200e3, args.maxiter, 1e-5,
                                                              nthreads=min(ncpu, pts.size), counts=True)
        r["cpu_subset"] = {
            "points": pts.tolist(), "wall_s": round(time.time() - t0, 2), "point_s": [round(float(s), 3) for s in secs],
            "sweeps": it.tolist(), "column_updates": mv.tolist(),
            "corr_bytes_read": [int(e) * bytes_per_value for e in ent],
            "gpu_point_s": [round(float(gp["time"][q]), 4) for q in pts],
            "identical": bool(np.array_equal(np.asarray(out)[:, pts], beta * sc[:, None], equal_nan=True)
                              and np.array_equal(gp["num_iter"][pts], it))}
        # assumes perfect balance over the cores; the sampled points ran concurrently, so their times include memory
        # contention and are not pure single-core times.  No all-core run can end before its slowest point does.
        r["cpu_all_core_extrapolated_s"] = round(float(secs[even].sum()) * 120 / spaced.size / ncpu, 2)
        r["cpu_lower_bound_slowest_sampled_point_s"] = round(float(secs.max()), 2)
        r["cpu_cores"] = ncpu
        res[key] = r
        del st
    res["gpu_end"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_lassosum2.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
