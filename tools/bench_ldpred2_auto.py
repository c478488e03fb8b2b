"""snp_ldpred2_auto on one GPU (bsg_ldpred2_auto): 1 chain (the default vec_p_init) and 30 chains
(seq_log(1e-4, 0.2, 30)) at the default burn_in = 500 and num_iter = 200, over the LD matrix of bench_lassosum2, in both
SFBM storage forms.

    python tools/bench_ldpred2_auto.py [--n 10000] [--m 90000] [--size 2000] [--cpu-chains 4] [--out DIR]

The matrix and the simulated sumstats are bench_lassosum2's (bed_cor of an LD-structured synthetic chromosome, m SNPs,
a window of `size` SNPs each side; beta = R b + e / sqrt(N)); h2_init is snp_ldsc2's estimate on it.  The chains run
with allow_jump_sign = FALSE and shrink_corr = 0.95, the reference's remedies against divergence: with the defaults,
every chain diverges on this matrix (the window-cut correlation matrix is not positive definite), on the device and in
the oracle alike, and stops before its last sweep.  `sweeps_run` counts each chain's completed sweeps.  Per form and run:
the wall time of the call and each chain's device seconds, and device ms per chain-sweep over the sweeps it ran.  Counted work comes from
the CPU oracle (tests/ldpred2_auto_oracle.c) on a stated subset of the chains (the 1-chain run's chain; for 30 chains,
`cpu-chains` evenly spaced ones, run in parallel, one per core): column updates ("moves") per sweep and the corr bytes
they read.  The all-core CPU time of the 30 chains is extrapolated as (sum of the subset's times) x 30 / subset / cores,
assuming perfect balance.  The GPU outputs of those chains must equal the oracle's bit for bit.  GPU name, power limit
and SM clock are read in the same run.  One JSON line to stdout (and DIR/bench_ldpred2_auto.json).
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_lassosum2 import gpu_info, simulated_sumstats  # noqa: E402


def same_bytes(a, b):
    """identical bytes, NaN entries compared as NaN"""
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10000)
    ap.add_argument("--m", type=int, default=90000)
    ap.add_argument("--size", type=int, default=2000, help="window, in SNPs each side (positions 1 kb apart)")
    ap.add_argument("--burn-in", type=int, default=500)
    ap.add_argument("--num-iter", type=int, default=200)
    ap.add_argument("--cpu-chains", type=int, default=4)
    ap.add_argument("--n-eff", type=float, default=50000, help="GWAS sample size of the simulated sumstats")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import bigsnpr_b200 as B
    from bigsnpr_b200 import api
    from tests import ldpred2_auto_ref as R

    n, m = args.n, args.m
    res = {"n": n, "m": m, "n_eff_max": args.n_eff, "window_snps_each_side": args.size, "burn_in": args.burn_in, "num_iter": args.num_iter,
           "allow_jump_sign": False, "shrink_corr": 0.95, "gpu_start": gpu_info()}
    g = B.Bed.synthetic(n, m, seed=21, ld_rho=0.9, ld_block=50)
    corr = B.bed_cor(g, size=args.size)
    g.close()
    df = simulated_sumstats(corr, m, 4, n_eff=args.n_eff)
    N = df["n_eff"]
    sd = 1 / np.sqrt(N * df["beta_se"] ** 2 + df["beta"] ** 2)
    bh, lv = df["beta"] * sd, 2 * np.log(sd)
    st0 = api.sfbm_storage(corr)
    sf = api.SFBM(st0[0], st0[0], st0[1], st0[2], st0[3])
    h2 = float(B.snp_ldsc2(sf, df, blocks=None)[1])
    res["h2_init_ldsc2"] = h2
    # warm-up: a 2,000-SNP slice, a few sweeps
    ps = corr[0][:2001]
    sl = B.as_SFBM((ps, corr[1][:ps[-1]], corr[2][:ps[-1]]))
    B.snp_ldpred2_auto(sl, {k: v[:2000] for k, v in df.items()}, h2, burn_in=5, num_iter=5, seed=1)
    sl.close()
    sf.close()
    mean_ld = None
    ncpu = os.cpu_count() or 1
    res["cpu_cores"] = ncpu
    for compact in (False, True):
        key = "compact" if compact else "non_compact"
        st = st0 if not compact else api.sfbm_storage(corr, compact=True)
        sf = api.SFBM(st[0], st[0], st[1], st[2], st[3])
        if mean_ld is None:
            mean_ld = float(np.mean(B.ld_scores_sfbm(sf)))
        bytes_per_value = 12 if not compact else 8  # int32 row + fp64 value, or the value alone
        out = {}
        for label, p_init in (("1_chain", np.array([0.1])), ("30_chains", api.seq_log(1e-4, 0.2, 30))):
            p_run = np.sort(p_init)[::-1]  # order(-vec_p_init)
            s = api.mrg32k3a_seed(2024)
            states = []
            for _ in p_run:
                states.append(s)
                s = api.mrg32k3a_next_stream(s)
            states = np.array(states)
            t0 = time.time()
            r = api._ldpred2_auto_call(sf, bh, N, lv, np.arange(m), p_run, h2, args.burn_in, args.num_iter,
                                       args.num_iter + 1, True, 0.95, True, np.array([1e-5, 1.0]), np.array([-0.5, 1.5]),
                                       mean_ld, states, sample=False)
            wall = time.time() - t0
            sub = np.array([0]) if p_run.size == 1 else np.unique(np.linspace(0, p_run.size - 1, args.cpu_chains).round()
                                                                   .astype(int))
            t0 = time.time()
            o = R.ldpred2_auto(st, bh, N, lv, np.arange(m), p_run[sub], h2, states[sub], burn_in=args.burn_in,
                               num_iter=args.num_iter, mean_ld=mean_ld, alpha_bounds=(-0.5, 1.5), sample=False,
                               no_jump_sign=True, shrink_corr=0.95,
                               nthreads=min(ncpu, sub.size), counts=True)
            cpu_wall = time.time() - t0
            ident = all(same_bytes(r[k][:, sub], o[k])
                        for k in ("beta_est", "postp_est", "corr_est", "path_p_est", "path_h2_est", "path_alpha_est"))
            dev = r["time"]
            sweeps = (~np.isnan(r["path_p_est"])).sum(0)  # completed sweeps (a diverging one is not recorded)
            osw = sweeps[sub]
            out[label] = {
                "p_init": [float(v) for v in p_run], "wall_s": round(wall, 3),
                "chain_device_s": [round(float(v), 3) for v in dev],
                "device_ms_per_chain_sweep": round(float((dev / sweeps).mean()) * 1e3, 3),
                "slowest_chain_device_s": round(float(dev.max()), 3),
                "sweeps_run": sweeps.tolist(),
                "h2_est": [round(float(np.mean(r["path_h2_est"][-args.num_iter:, c])), 4) for c in range(p_run.size)],
                "p_est": [float(np.mean(r["path_p_est"][-args.num_iter:, c])) for c in range(p_run.size)],
                "cpu_subset": {"chains": sub.tolist(), "wall_s": round(cpu_wall, 2),
                               "chain_s": [round(float(v), 2) for v in o["seconds"]],
                               "moves_per_sweep": [round(float(v) / w, 1) for v, w in zip(o["moves"], osw)],
                               "corr_bytes_read_per_sweep": [int(v) * bytes_per_value // int(w) for v, w in zip(o["entries"], osw)],
                               "gpu_chain_s": [round(float(dev[c]), 3) for c in sub]},
                "cpu_all_core_extrapolated_s": round(float(o["seconds"].sum()) * p_run.size / sub.size / min(ncpu, p_run.size), 2),
                "identical": bool(ident)}
        sf.close()
        res[key] = out
    res["gpu_end"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_ldpred2_auto.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
