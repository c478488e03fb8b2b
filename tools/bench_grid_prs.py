"""snp_grid_PRS on one GPU (bsg_prs_grid): the C+T scores of the default 7 x 4 clumping grid of one LD-structured
chromosome (the workload of tools/bench_grid_clumping.py) at 50 p-value thresholds, at n = 50,000 and at UK Biobank's
n = 487,000 (same SNPs, same keep sets).

    python tools/bench_grid_prs.py [--n 50000] [--n-large 487000] [--m 40000] [--m-dosage 10000] [--out DIR]

A third workload: 10,000 CODE_DOSAGE SNPs at n = 50,000 with the keep sets restricted to them.
Per workload: the device time of the call (CUDA events, quantisation to the gathered output, bsg_prs_last_ms), median
and range over 5 calls after a warm-up call of the same shape, the median wall time of snp_grid_PRS, the bytes the kernel must read (sum over sets of the step-padded line
count x ceil(n / 4), x n for dosages) and that rate against the H100 SXM data sheet's 3.35 TB/s.  The device baseline is the existing
path: one column-list bed_prodVec per (set, step), added up on the host; its largest relative difference to the new
scores is reported (the two quantise differently, so equality is not expected).  The CPU figure is R's literal loop
(tests/prs_ref.py) on one keep set and 2,000 rows.  The GPU name, power limit and SM clock are read in the same run.
One JSON line to stdout (and DIR/bench_grid_prs.json).
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

HBM_BYTES_S = 3.35e12  # H100 SXM data sheet


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def padded_lines(sets, lpS, thr):
    from tests import prs_ref as P

    tot = 0
    for s in sets:
        st, _ = P.steps_of(lpS[s - 1], thr, s.size)
        for k in range(thr.size):
            tot += -(-int(np.sum(st == k)) // 32) * 32
    return tot


def baseline(B, g, sets, betas, lpS, thr, ind_row):
    """Cumulative scores from one bed_prodVec per non-empty (set, step): (seconds, calls, list of nr x nthr arrays)."""
    from tests import prs_ref as P

    out, calls = [], 0
    t0 = time.time()
    for s in sets:
        st, ordr = P.steps_of(lpS[s - 1], thr, s.size)
        last = np.zeros(ind_row.size)
        cols = np.empty((ind_row.size, thr.size))
        for k, i in enumerate(ordr):
            ind = np.flatnonzero(st == k)
            if ind.size:
                last = last + B.bed_prodVec(g, betas[s[ind] - 1], ind_row=ind_row, ind_col=s[ind])
                calls += 1
            cols[:, i] = last
        out.append(cols)
    return time.time() - t0, calls, out


def run(B, g, n, sets, keep, betas, lpS, thr, with_baseline, bytes_per_line=None, reps=5):
    """The whole call `reps` times after one warm-up call of the same shape: median and range of the device time."""
    from bigsnpr_b200 import _lib

    B.snp_grid_PRS(g, keep, betas, lpS, grid_lpS_thr=thr, type="float")  # warm-up, same shape
    ms, wall = [], []
    for _ in range(reps):
        t0 = time.time()
        res = B.snp_grid_PRS(g, keep, betas, lpS, grid_lpS_thr=thr, type="float")
        wall.append(time.time() - t0)
        ms.append(_lib.lib().bsg_prs_last_ms())
    med = float(np.median(ms))
    lines = padded_lines(sets, lpS, thr)
    nbytes = lines * (bytes_per_line or -(-n // 4))
    r = {"n": n, "sets": len(sets), "thresholds": int(thr.size), "columns": int(res.shape[1]),
         "entries": int(sum(s.size for s in sets)), "padded_lines": lines, "reps": reps,
         "device_ms_median": round(med, 2), "device_ms_min_max": [round(min(ms), 2), round(max(ms), 2)],
         "wall_s_median": round(float(np.median(wall)), 3), "bytes": nbytes,
         "TB_s": round(nbytes / (med * 1e-3) / 1e12, 3), "share_of_3.35TB_s": round(nbytes / (med * 1e-3) / HBM_BYTES_S, 3)}
    if with_baseline:
        ir = np.arange(1, n + 1, dtype=np.int32)
        sec, calls, base = baseline(B, g, sets, betas, lpS, thr, ir)
        dev = np.asarray(B.snp_grid_PRS(g, keep, betas, lpS, grid_lpS_thr=thr, type="double"))
        ref = np.concatenate(base, axis=1)
        r["baseline_prodvec_per_step_s"] = round(sec, 3)
        r["baseline_calls"] = calls
        r["baseline_max_rel_diff"] = float(np.max(np.abs(dev - ref)) / np.max(np.abs(ref)))
    del res
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000)
    ap.add_argument("--n-large", type=int, default=487000)
    ap.add_argument("--m", type=int, default=40000)
    ap.add_argument("--mb", type=float, default=250.0)
    ap.add_argument("--m-dosage", type=int, default=10000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import bigsnpr_b200 as B
    from tests import prs_ref as P

    n, m = args.n, args.m
    rng = np.random.default_rng(3)
    pos = np.round(np.linspace(1, args.mb * 1e6, m))
    lpS = -np.log10(rng.uniform(size=m))
    betas = rng.normal(size=m) * 0.01
    thr = 0.9999 * B.seq_log(max(0.1, lpS.min()), lpS.max(), 50)
    res = {"m": m, "span_Mb": args.mb, "grid": "7 thr.r2 x 4 base.size (defaults), 50 thresholds", "gpu_start": gpu_info()}

    g = B.Bed.synthetic(n, m, seed=5, ld_rho=0.9, ld_block=50)
    keep = B.snp_grid_clumping(g, np.ones(m, dtype=int), pos, lpS)
    sets = [np.asarray(s, dtype=np.int64) for s in keep[0]]
    res["small"] = run(B, g, n, sets, keep, betas, lpS, thr, True)

    # R's literal loop on one keep set and 2,000 rows, and the device on the same
    s0 = sets[len(sets) // 2]
    ir = np.arange(1, 2001)
    G = B.read_bed(g, ir, s0, na_val=3)
    t0 = time.time()
    want = P.literal(G, ir, np.arange(1, s0.size + 1), betas[s0 - 1], None, lpS[s0 - 1], thr)
    t_cpu = time.time() - t0
    got = np.asarray(B.snp_grid_PRS(g, [[s0]], betas, lpS, grid_lpS_thr=thr, ind_row=ir, type="double"))
    res["cpu_literal"] = {"rows": 2000, "entries": int(s0.size), "numpy_s": round(t_cpu, 3),
                          "max_rel_diff": float(np.max(np.abs(got - want)) / np.max(np.abs(want)))}
    g.close()

    gl = B.Bed.synthetic(args.n_large, m, seed=5, ld_rho=0.9, ld_block=50)
    res["large"] = run(B, gl, args.n_large, sets, keep, betas, lpS, thr, False)
    gl.close()

    # 10,000 CODE_DOSAGE SNPs at n = 50,000 (random dosages, no NA), the keep sets restricted to them; bytes per line = n
    md = args.m_dosage
    code = np.concatenate([[0, 1, 2, np.nan, 0, 1, 2], np.arange(201) * 0.01, np.full(48, np.nan)])
    raw = np.asfortranarray(rng.integers(7, 208, size=(n, md), dtype=np.uint8))
    gd = B.Bed.from_fbm(raw, code256=code)
    del raw
    assert gd.dosage_scale == 100
    dsets = [s[s <= md] for s in sets]
    dkeep = [dsets]
    res["dosage"] = run(B, gd, n, dsets, dkeep, betas[:md], lpS[:md], thr, False, bytes_per_line=n)
    res["dosage"]["m"] = md
    gd.close()
    res["gpu_end"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_grid_prs.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
