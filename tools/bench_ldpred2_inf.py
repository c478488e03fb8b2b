"""snp_ldpred2_inf on one GPU (bsg_sfbm_solve): the conjugate-gradient solve over one chromosome-sized LD matrix, in both
SFBM storage forms, with h2 from snp_ldsc2.

    python tools/bench_ldpred2_inf.py [--n 10000] [--m 90000] [--size 2000] [--out DIR]

The matrix and sumstats are those of tools/bench_lassosum2.py (bed_cor of an LD-structured synthetic chromosome of m SNPs
and n samples, a window of `size` SNPs each side; beta = R b + e / sqrt(N)).  h2 comes from snp_ldsc2 on the SFBM; the
solve then also runs at 0.3 x and 1.4 x that h2 (a larger and a smaller diagonal: slower and faster convergence).  Per
solve: wall time of the sp_solve_sym call, iterations, the device time of its iterations (CUDA events around them,
bsg_sfbm_last_solve_ms) and per iteration, the stored-matrix bytes one iteration reads (12 B per value non-compact: int32
row + fp64 value, 8 B compact, + the offsets), that figure over the time per iteration and its share of the H100 SXM data
sheet's 3.35 TB/s, whether x, iters and error equal the CPU oracle's (tests/spsolve_oracle.c) bit for bit, and the
oracle's all-core wall time on the same host.  GPU name, power limit and SM clock are read in the same run.  One JSON
line to stdout (and DIR/bench_ldpred2_inf.json).
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM_BPS = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10000)
    ap.add_argument("--m", type=int, default=90000)
    ap.add_argument("--size", type=int, default=2000, help="window, in SNPs each side (positions 1 kb apart)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import bigsnpr_b200 as B
    from bigsnpr_b200 import _lib, api
    from bench_lassosum2 import gpu_info, simulated_sumstats
    from tests import spsolve_ref as S

    n, m = args.n, args.m
    res = {"n": n, "m": m, "window_snps_each_side": args.size, "tol": 1e-10, "maxiter": "10 m",
           "gpu_start": gpu_info()}
    g = B.Bed.synthetic(n, m, seed=21, ld_rho=0.9, ld_block=50)
    t0 = time.time()
    corr = B.bed_cor(g, size=args.size)
    res["bed_cor_s"] = round(time.time() - t0, 2)
    g.close()
    df = simulated_sumstats(corr, m, 4)
    res["nnz_upper"] = int(corr[0][-1])
    N = df["n_eff"]
    scale = np.sqrt(N * df["beta_se"] ** 2 + df["beta"] ** 2)
    beta_hat = df["beta"] / scale

    # warm-up: a 2,000-SNP slice
    ps = corr[0][:2001]
    sf = B.as_SFBM((ps, corr[1][:ps[-1]], corr[2][:ps[-1]]))
    B.snp_ldpred2_inf(sf, {k: v[:2000] for k, v in df.items()}, 0.3)
    sf.close()

    ncpu = os.cpu_count() or 1
    for compact in (False, True):
        key = "compact" if compact else "non_compact"
        st = api.sfbm_storage(corr, compact=compact)
        sf = api.SFBM(st[0], st[0], st[1], st[2], st[3])
        t0 = time.time()
        ldsc = B.snp_ldsc2(sf, df)
        r = {"snp_ldsc2_s": round(time.time() - t0, 3), "ldsc_int_h2": [float(v) for v in ldsc]}
        nnz = int(st[1][-1])
        bytes_iter = nnz * (8 if compact else 12) + 8 * (m + 1) + (4 * m if compact else 0)
        r["nnz"], r["matrix_bytes_per_iteration"] = nnz, bytes_iter
        solves = []
        for mult in (1.0, 0.3, 1.4):
            h2 = float(ldsc[1]) * mult
            d = m / (h2 * N)
            t0 = time.time()
            x, it, err = api._sp_solve(sf, beta_hat, d, 1e-10, None)
            wall = time.time() - t0
            ms = _lib.lib().bsg_sfbm_last_solve_ms(sf._h)
            x0, it0, err0, cpu_s = S.solve(st, beta_hat, d, 1e-10, None, nthreads=ncpu, timed=True)
            per_it = ms / 1e3 / max(it + 1, 1)  # the breaking iteration runs too
            solves.append({
                "h2": h2, "h2_multiplier": mult, "iterations": it, "error": err, "wall_s": round(wall, 4),
                "device_s": round(ms / 1e3, 4), "device_s_per_iteration": per_it,
                "matrix_GBps": round(bytes_iter / per_it / 1e9, 1),
                "share_of_3.35TBps": round(bytes_iter / per_it / HBM_BPS, 3),
                "identical_to_oracle": bool(x.tobytes() == x0.tobytes() and it == it0
                                            and np.float64(err).tobytes() == np.float64(err0).tobytes()),
                "cpu_oracle_all_core_s": round(cpu_s, 2), "cpu_cores": ncpu})
        r["solves"] = solves
        beta_inf = B.snp_ldpred2_inf(sf, df, float(ldsc[1]))
        r["ldpred2_inf_equals_scaled_solve"] = bool(
            beta_inf.tobytes() == (api._sp_solve(sf, beta_hat, m / (float(ldsc[1]) * N), 1e-10, None)[0] * scale).tobytes())
        sf.close()
        res[key] = r
        del st
    res["gpu_end"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_ldpred2_inf.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
