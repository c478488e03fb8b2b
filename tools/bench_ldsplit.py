"""snp_ldsplit on one GPU (bsg_ldsplit) over one chromosome-sized LD matrix, with the reference example's parameters.

    python tools/bench_ldsplit.py [--n 10000] [--m 90000] [--size 2000] [--no-cpu] [--out DIR]

The matrix is bed_cor of the LD-structured synthetic chromosome of tools/bench_lassosum2.py (m SNPs, n samples, a window
of `size` SNPs each side), built on the device.  Parameters: thr_r2 = 0.02, min_size = 100, max_size =
round(seq_log(m / 30, m / 5, 10)), max_K = 500, the defaults otherwise (examples/example-split-LD.R).  Reported: the
device time of building E and its allocated bytes, the layers run per max_size, the device time of the layers and per
layer, the allocated E bytes per layer time (an upper bound on the bytes read: a col's E stops early when the cost
exceeds max_cost), the whole-call wall time (after a warm-up on a slice).  The CPU oracle (tests/ldsplit_oracle.c, one
thread like the reference) runs the smallest max_size alone; its table must equal the GPU's for that max_size bit for
bit, and its time is a measurement of that max_size only.  GPU name, power limit and SM clock are read in the same run.
One JSON line to stdout (and DIR/bench_ldsplit.json).
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

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10000)
    ap.add_argument("--m", type=int, default=90000)
    ap.add_argument("--size", type=int, default=2000)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import bigsnpr_b200 as B
    from bigsnpr_b200 import api
    from tests import ldsplit_ref as R

    res = {"n": args.n, "m": args.m, "window_snps_each_side": args.size, "gpu_start": gpu_info()}
    g = B.Bed.synthetic(args.n, args.m, seed=21, ld_rho=0.9, ld_block=50)
    corr = B.bed_cor(g, size=args.size)
    g.close()
    m = len(corr[0]) - 1
    S = np.round(api.seq_log(m / 30, m / 5, 10)).astype(np.int32)
    kw = dict(thr_r2=0.02, min_size=100, max_size=S, max_K=500)
    res.update({"max_size": S.tolist(), "thr_r2": 0.02, "min_size": 100, "max_K": 500, "nnz_upper": int(corr[0][-1])})

    t0 = time.time()
    h = B.LDCorr(corr)
    res["stage_s"] = round(time.time() - t0, 2)
    # warm-up: a 3,000-SNP slice
    ps = corr[0][:3001]
    w = B.LDCorr((ps, corr[1][:ps[-1]], corr[2][:ps[-1]]))
    w.split(0.02, 100, [300, 600], max_K=50)
    w.close()

    t0 = time.time()
    table, layers, secs = h.split(**kw)
    wall = time.time() - t0
    ecap = 4 * sum(max(0, min(int(S.max()), c + 1) - 100 + 1) for c in range(m))
    nl = int(layers.max())
    per_layer = float(secs[1]) / max(1, nl - 1)
    res.update({"wall_s": round(wall, 3), "E_build_device_s": round(float(secs[0]), 4), "E_bytes_allocated": ecap,
                "layers_per_max_size": layers.tolist(), "layers_device_s": round(float(secs[1]), 4),
                "device_s_per_layer": round(per_layer, 6),
                "E_bytes_allocated_per_layer_s": round(ecap / per_layer / 1e9, 1) if per_layer > 0 else None,
                "share_of_datasheet_hbm_upper_bound": round(ecap / per_layer / HBM_BYTES_PER_S, 3) if per_layer > 0 else None,
                "paths_perc_device_s": round(float(secs[2]), 4),
                "rows_kept": 0 if table is None else int(table["n_block"].size)})
    again = h.split(**kw)[0]
    res["two_calls_identical"] = bool(table is None and again is None or
                                      all(np.array_equal(table[k], again[k]) for k in ("n_block", "cost", "perc_kept")))
    if not args.no_cpu:
        s0 = int(S.min())
        low = api.ldsplit_lower(corr)
        t0 = time.time()
        nlc = []
        want = R.snp_ldsplit(low, 0.02, 100, s0, max_K=500, layers=nlc)
        cpu = time.time() - t0
        got = h.split(0.02, 100, s0, max_K=500)[0]
        same = (want is None and got is None) or (
            got is not None and want is not None and all(got[k].tobytes() == np.asarray(want[k]).tobytes()
                                                         for k in ("n_block", "cost", "cost2", "perc_kept"))
            and all(np.array_equal(a, b) for a, b in zip(got["all_last"], want["all_last"])))
        res["cpu_one_thread_smallest_max_size"] = {"max_size": s0, "wall_s": round(cpu, 2), "layers": nlc[0],
                                                   "identical_to_gpu": bool(same)}
    h.close()
    res["gpu_end"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_ldsplit.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
