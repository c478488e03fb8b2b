#!/usr/bin/env python
"""Timings of the other hot-path rows on shapes scaled from BASELINE.json configs[2] (snp_cor) and configs[3]
(bed_tcrossprodSelf), plus colstats/counts.  Prints one JSON line per op.  Not the driver's bench."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bigsnpr_b200 as B  # noqa: E402


def timeit(f, reps=1):
    import torch

    f()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        r = f()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cor-n", type=int, default=100000)
    ap.add_argument("--cor-m", type=int, default=20000)
    ap.add_argument("--size", type=int, default=500)
    ap.add_argument("--clump-n", type=int, default=50000)
    ap.add_argument("--clump-m", type=int, default=100000)
    ap.add_argument("--grm-n", type=int, default=10000)
    ap.add_argument("--grm-m", type=int, default=50000)
    ap.add_argument("--ld-rho", type=float, default=0.9, help="LD-structured data for the windowed rows (0 = i.i.d.)")
    ap.add_argument("--skip", default="", help="comma list of: cor, clump, grm")
    a = ap.parse_args()
    # --- snp_cor / ld_scores (configs[2] is 100,000 x 200,000, size 500: 9.99e7 pairs)
    skip = set(a.skip.split(","))
    g = B.Bed.synthetic(a.cor_n, a.cor_m, seed=20250927, layouts=B.LAYOUT_SNP_MAJOR, ld_rho=a.ld_rho)
    t, (p, i, x) = timeit(lambda: B.bed_cor(g, size=a.size))
    pairs = int(p[-1]) - a.cor_m
    print(json.dumps({"op": "bed_cor", "n": a.cor_n, "m": a.cor_m, "size": a.size, "pairs": pairs, "seconds": t,
                      "pairs_per_s": pairs / t, "useful_flops": 2.0 * a.cor_n * pairs,
                      "cfg3_extrapolated_s": t * 99874750 / max(pairs, 1)}), flush=True)
    t, ld = timeit(lambda: B.bed_ld_scores(g, size=a.size))
    print(json.dumps({"op": "bed_ld_scores", "n": a.cor_n, "m": a.cor_m, "size": a.size, "seconds": t}), flush=True)
    t, _ = timeit(lambda: B.bed_counts(g))
    print(json.dumps({"op": "bed_counts(all)", "seconds": t}), flush=True)
    g.close()
    # --- bed_clumping (thr.r2 = 0.2, size = 500 kb on a 1 kb grid: 500 SNPs either side)
    gc = B.Bed.synthetic(a.clump_n, a.clump_m, seed=20250929, ld_rho=a.ld_rho)
    chrom, pos = np.ones(a.clump_m, dtype=int), 1000.0 * np.arange(1, a.clump_m + 1)
    t, keep = timeit(lambda: B.bed_clumping(gc, infos_chr=chrom, infos_pos=pos))
    rec = {"op": "bed_clumping", "n": a.clump_n, "m": a.clump_m, "thr_r2": 0.2, "size_kb": 500, "seconds": t,
           "kept": int(keep.size), "window_pairs": int(a.clump_m) * 500 - 500 * 501 // 2}
    try:
        from oracle import ref

        mo = min(a.clump_m, 1500)
        o = ref.synth_bed(a.clump_n, mo, seed=20250929, ld_rho=a.ld_rho)
        t0 = time.perf_counter()
        ko = ref.bed_clumping(o, infos_chr=chrom[:mo], infos_pos=pos[:mo])
        tc = time.perf_counter() - t0
        rec.update({"cpu_oracle_cols": mo, "cpu_oracle_seconds": tc, "cpu_oracle_threads": 1,
                    "same_kept_on_sample": bool(np.array_equal(ko, B.bed_clumping(gc, infos_chr=chrom, infos_pos=pos,
                                                                                   exclude=np.arange(mo + 1, a.clump_m + 1))))})
    except Exception as e:  # pragma: no cover
        rec["cpu_oracle_error"] = repr(e)
    print(json.dumps(rec), flush=True)
    gc.close()
    # --- bed_tcrossprodSelf (configs[3] is 10,000 x 1,000,000)
    for na_rate in (0.0, 0.01):
        g = B.Bed.synthetic(a.grm_n, a.grm_m, seed=20250928, na_rate=na_rate)
        sc = B.bed_scaleBinom(g)
        fun = lambda *aa, **kw: sc  # noqa: E731
        t, (K, c, s) = timeit(lambda: B.bed_tcrossprodSelf(g, fun_scaling=fun))
        print(json.dumps({"op": "bed_tcrossprodSelf", "n": a.grm_n, "m": a.grm_m, "na_rate": na_rate, "seconds": t,
                          "useful_flops": float(a.grm_n) * (a.grm_n + 1) * a.grm_m,
                          "useful_tflops": float(a.grm_n) * (a.grm_n + 1) * a.grm_m / t / 1e12,
                          "cfg4_extrapolated_s": t * 1_000_000 / a.grm_m, "path": os.environ.get("BSG_GRM_DSYRK", "0"),
                          "slices": os.environ.get("BSG_GRM_SLICES", "8")}), flush=True)
        g.close()
    # the same matrix with a caller's scaling that puts 1 % of the columns in rare-variant weight classes (cohort
    # allele frequencies of 1e-3 and 1e-5): the columns are sorted by class and each class is folded in turn
    g = B.Bed.synthetic(a.grm_n, a.grm_m, seed=20250928)
    sc = B.bed_scaleBinom(g)
    c, s = np.array(sc["center"]), np.array(sc["scale"])
    rare = np.random.default_rng(1).choice(a.grm_m, a.grm_m // 100, replace=False)
    pc = np.where(np.arange(rare.size) % 2 == 0, 1e-3, 1e-5)
    c[rare], s[rare] = 2 * pc, np.sqrt(2 * pc * (1 - pc))
    W1 = 1.0 / (s * s)
    ncls = np.unique(np.floor(np.log2(W1.max() / W1) / 4)).size  # the class rule of bsg_la.cu tcrossprod_impl
    t, _ = timeit(lambda: B.bed_tcrossprodSelf(g, fun_scaling=lambda *aa, **kw: {"center": c, "scale": s}))
    print(json.dumps({"op": "bed_tcrossprodSelf", "n": a.grm_n, "m": a.grm_m, "na_rate": 0.0, "seconds": t,
                      "rare_columns": int(rare.size), "weight_classes": int(ncls), "gpu": _gpu_name(),
                      "power_limit_w": _power_limit()}), flush=True)
    g.close()


def _gpu_name():
    import torch

    return torch.cuda.get_device_name(0)


def _power_limit():
    """The enforced power limit of GPU 0 in W, read (not set) through nvidia-smi; None where it cannot be read."""
    import subprocess

    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:  # pragma: no cover
        return None


if __name__ == "__main__":
    main()
