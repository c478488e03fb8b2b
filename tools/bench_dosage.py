"""Dosage FBM.code256 products on one GPU: the byte-operand tensor-pipe kernels (bsg_dosage.cu) at 50,000 x 100,000.

    python tools/bench_dosage.py [--n 50000] [--m 100000] [--reps 20] [--out DIR]

Reports per product (X.y = k_dmvT, Xt.y = k_dmv; identity selection and a column list of every other SNP): device time
from CUDA events over `reps` launches after warm-up, bytes of the value copy read / time, and that rate as a fraction of
the H100 SXM data-sheet 3.35 TB/s.  Then bed_randomSVD(k = 10) with snp_scaleBinom scaling (wall time), the literal
fp64 loop over code256[byte] on a column sample in NumPy (the CPU baseline, extrapolated to the whole matrix), and the
GPU name, power limit and SM clock read in the same process.  Writes one JSON line to stdout (and DIR/bench_dosage.json).
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

CODE_DOSAGE = np.concatenate([[0, 1, 2, np.nan, 0, 1, 2], np.arange(201) * 0.01, np.full(48, np.nan)])
HBM_PEAK = 3.35e12


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000)
    ap.add_argument("--m", type=int, default=100000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import bigsnpr_b200 as B

    n, m = args.n, args.m
    rng = np.random.default_rng(7)
    t0 = time.time()
    G = np.empty((n, m), dtype=np.uint8, order="F")
    step = max(1, (1 << 28) // n)
    for j0 in range(0, m, step):  # codes 7..207: dosages 0.00..2.00
        j1 = min(m, j0 + step)
        G[:, j0:j1] = (7 + rng.integers(0, 201, size=(n, j1 - j0), dtype=np.uint8)).astype(np.uint8)
    t_gen = time.time() - t0
    t0 = time.time()
    g = B.Bed.from_fbm(G, code256=CODE_DOSAGE)
    t_stage = time.time() - t0
    assert g.dosage_scale == 100
    st = B.snp_scaleBinom()(g)
    c, s = st["center"], st["scale"]
    res = {"n": n, "m": m, "bytes_per_pass": n * m, "gen_s": round(t_gen, 1), "stage_s": round(t_stage, 1)}
    cols = np.arange(1, m + 1, 2, dtype=np.int32)
    for label, ic in (("identity", None), ("col_list", cols)):
        icol = np.arange(1, m + 1, dtype=np.int32) if ic is None else ic
        t_first = time.time()
        v = B.View(g, ind_col=icol, center=c[icol - 1], scale=s[icol - 1])  # the first view builds the value copy
        x = torch.tensor(rng.normal(size=icol.size), device="cuda")
        y = torch.tensor(rng.normal(size=n), device="cuda")
        ox = torch.empty(n, dtype=torch.float64, device="cuda")
        oy = torch.empty(icol.size, dtype=torch.float64, device="cuda")
        v.prodvec_dev(x.data_ptr(), ox.data_ptr())
        torch.cuda.synchronize()
        if label == "identity":
            res["first_view_and_product_incl_value_copy_s"] = round(time.time() - t_first, 2)
        for name, f in (("prodVec", lambda: v.prodvec_dev(x.data_ptr(), ox.data_ptr())),
                        ("cprodVec", lambda: v.cprodvec_dev(y.data_ptr(), oy.data_ptr()))):
            for _ in range(3):
                f()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                f()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.reps
            nbytes = n * icol.size
            res["%s_%s_ms" % (name, label)] = round(ms, 3)
            res["%s_%s_TBps" % (name, label)] = round(nbytes / (ms * 1e-3) / 1e12, 3)
            res["%s_%s_frac_of_3.35TBps" % (name, label)] = round(nbytes / (ms * 1e-3) / HBM_PEAK, 3)
        assert not torch.isnan(ox).any() and not torch.isnan(oy).any()
        v.close()
    res["gpu_during_products"] = gpu_info()
    t0 = time.time()
    svd = B.bed_randomSVD(g, fun_scaling=B.snp_scaleBinom(), k=10)
    res["randomSVD_k10_s"] = round(time.time() - t0, 2)
    res["randomSVD_nops"] = int(svd["nops"])
    # CPU baseline: the literal loop (code256[byte] - c) / s * x on a column sample, extrapolated to m columns
    samp = np.arange(0, m, max(1, m // 500))
    xs = rng.normal(size=samp.size)
    t0 = time.time()
    X = (CODE_DOSAGE[G[:, samp]] - c[samp]) / s[samp]
    _ = (X * xs[None, :]).sum(axis=1)
    t_cpu = time.time() - t0
    res["cpu_literal_prodVec_s_extrapolated"] = round(t_cpu * m / samp.size, 2)
    res["gpu_after_svd"] = gpu_info()
    g.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_dosage.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
