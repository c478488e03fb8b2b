"""snp_ldpred2_grid on one GPU (bsg_ldpred2_grid): the 168-point grid users run (p = seq_log(1e-5, 1, 21), h2 = h2_est x
(0.3, 0.7, 1, 1.4) with h2_est snp_ldsc2's estimate, sparse FALSE and TRUE) at the default burn_in = 50 and num_iter = 100,
on two LD matrices of the same 90,000 SNPs:

  - banded: bench_lassosum2's matrix (bed_cor of an LD-structured synthetic chromosome, a window of `size` SNPs each side),
    non-compact.  It is probably not positive definite: LDpred2-auto's chains diverge on it, and so do many points here.
  - blocks: the block-diagonal matrix with full bed_cor inside blocks of `block` SNPs, compact.  Each block is a Gram
    matrix, so the matrix is positive semi-definite: the LD matrices users feed LDpred2 after snp_ldsplit look like it,
    and its chains run every sweep.

    python tools/bench_ldpred2_grid.py [--n 10000] [--m 90000] [--size 2000] [--block 3000] [--cpu-points 4] [--out DIR]

Per matrix: the wall time of the call and each point's device seconds; the points that diverged.  Counted work comes
from the CPU oracle (tests/ldpred2_grid_oracle.c) on `cpu-points` evenly spaced points of the run order, one per core:
sweeps run, column updates ("moves") per sweep, device and oracle ms per point-sweep, and whether the GPU columns of
those points equal the oracle's bit for bit.  The all-core CPU time of the 168 points is extrapolated from the subset as
(mean oracle seconds per sweep over the subset) x (sweeps of all points, diverged ones counted as the subset's mean)
/ cores, assuming perfect balance.  GPU name, power limit and SM clock are read in the same run.  One JSON line to
stdout (and DIR/bench_ldpred2_grid.json).
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
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def block_diagonal(B, g, m, block):
    """The upper CSC (p, i, x) of diag(bed_cor(block_1), bed_cor(block_2), ...), every pair inside a block stored."""
    ps, idx, xs, off = [np.zeros(1, dtype=np.int64)], [], [], 0
    for s in range(0, m, block):
        e = min(m, s + block)
        p, i, x = B.bed_cor(g, ind_col=np.arange(s + 1, e + 1, dtype=np.int32), size=e - s)
        ps.append(np.asarray(p[1:], dtype=np.int64) + off)
        idx.append(np.asarray(i, dtype=np.int64) + s)
        xs.append(np.asarray(x, dtype=np.float64))
        off += int(p[-1])
    return np.concatenate(ps), np.concatenate(idx), np.concatenate(xs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10000)
    ap.add_argument("--m", type=int, default=90000)
    ap.add_argument("--size", type=int, default=2000, help="window of the banded matrix, in SNPs each side")
    ap.add_argument("--block", type=int, default=3000, help="block size of the block-diagonal matrix, in SNPs")
    ap.add_argument("--burn-in", type=int, default=50)
    ap.add_argument("--num-iter", type=int, default=100)
    ap.add_argument("--cpu-points", type=int, default=4)
    ap.add_argument("--n-eff", type=float, default=50000, help="GWAS sample size of the simulated sumstats")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import bigsnpr_b200 as B
    from bigsnpr_b200 import api
    from tests import ldpred2_grid_ref as G

    n, m = args.n, args.m
    res = {"n": n, "m": m, "n_eff_max": args.n_eff, "burn_in": args.burn_in, "num_iter": args.num_iter,
           "gpu_start": gpu_info()}
    g = B.Bed.synthetic(n, m, seed=21, ld_rho=0.9, ld_block=50)
    banded = B.bed_cor(g, size=args.size)
    df = simulated_sumstats(banded, m, 4, n_eff=args.n_eff)
    N = df["n_eff"]
    scale = np.sqrt(N * df["beta_se"] ** 2 + df["beta"] ** 2)
    bh = df["beta"] / scale
    st = api.sfbm_storage(banded)
    sf = api.SFBM(st[0], st[0], st[1], st[2], st[3])
    h2_est = float(B.snp_ldsc2(sf, df, blocks=None)[1])
    sf.close()
    h2_seq = np.round(h2_est * np.array([0.3, 0.7, 1.0, 1.4]), 4)
    p_seq = api.seq_log(1e-5, 1, 21)
    P, H, S = np.meshgrid(p_seq, h2_seq, [False, True], indexing="ij")
    o = api._ldpred2_grid_order(P.ravel(), H.ravel(), S.ravel())
    p_run, h2_run, s_run = P.ravel()[o], H.ravel()[o], S.ravel()[o]
    npt = p_run.size
    states = api._mrg_streams(2024, npt)
    res.update({"h2_ldsc2": h2_est, "h2_seq": h2_seq.tolist(), "points": int(npt)})
    # warm-up: a 2,000-SNP slice, a few sweeps
    ps = banded[0][:2001]
    sl = B.as_SFBM((ps, banded[1][:ps[-1]], banded[2][:ps[-1]]))
    api._ldpred2_grid_call(sl, bh[:2000], N[:2000], np.arange(2000), p_run[:4], h2_run[:4], s_run[:4], 2, 2, states[:4])
    sl.close()
    ncpu = os.cpu_count() or 1
    res["cpu_cores"] = ncpu
    sub = np.unique(np.linspace(0, npt - 1, args.cpu_points).round().astype(int))
    mats = (("banded", False, args.size), ("blocks", True, args.block))
    for key, compact, width in mats:
        if key == "blocks":
            corr = block_diagonal(B, g, m, args.block)
            st = api.sfbm_storage(corr, compact=True)
            del corr
        elif compact:
            st = api.sfbm_storage(banded, compact=True)
        sf = api.SFBM(st[0], st[0], st[1], st[2], st[3])
        t0 = time.time()
        r = api._ldpred2_grid_call(sf, bh, N, np.arange(m), p_run, h2_run, s_run, args.burn_in, args.num_iter, states)
        wall = time.time() - t0
        sf.close()
        dev = r["time"]
        diverged = np.isnan(r["beta_est"]).all(0)
        t0 = time.time()
        orc = G.ldpred2_grid(st, bh, N, np.arange(m), p_run[sub], h2_run[sub], s_run[sub], states[sub], args.burn_in,
                             args.num_iter, nthreads=min(ncpu, sub.size), counts=True)
        cpu_wall = time.time() - t0
        sw = orc["sweeps"].astype(np.float64)
        ident = all(same_bytes(r["beta_est"][:, c], orc["beta_est"][:, i]) for i, c in enumerate(sub))
        full_sweeps = args.burn_in + args.num_iter
        est_sweeps = np.where(diverged, sw.mean(), full_sweeps).sum()
        bytes_per_value = 8 if compact else 12  # the value, or an int32 row and the value
        res[key] = {
            "storage": "compact" if compact else "non_compact", "width_snps": width, "nnz": int(st[1][-1]),
            "wall_s": round(wall, 3), "device_s_total_max": round(float(dev.max()), 3),
            "point_device_s": [round(float(v), 3) for v in dev],
            "device_s_per_point_mean": round(float(dev.mean()), 4),
            "diverged_points": int(diverged.sum()),
            "cpu_subset": {
                "points": sub.tolist(), "p": [float(p_run[c]) for c in sub], "h2": [float(h2_run[c]) for c in sub],
                "sparse": [bool(s_run[c]) for c in sub], "sweeps_run": orc["sweeps"].tolist(),
                "moves_per_sweep": [round(float(v) / w, 1) for v, w in zip(orc["moves"], sw)],
                "corr_bytes_read_per_sweep": [int(v * bytes_per_value / w) for v, w in zip(orc["entries"], sw)],
                "gpu_ms_per_point_sweep": [round(float(dev[c]) / w * 1e3, 3) for c, w in zip(sub, sw)],
                "cpu_ms_per_point_sweep": [round(float(v) / w * 1e3, 3) for v, w in zip(orc["seconds"], sw)],
                "cpu_wall_s": round(cpu_wall, 2)},
            "cpu_all_core_extrapolated_s": round(float((orc["seconds"] / sw).mean() * est_sweeps / ncpu), 2),
            "identical": bool(ident)}
    g.close()
    res["gpu_end"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_ldpred2_grid.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
