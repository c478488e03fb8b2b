"""snp_grid_clumping on one GPU (bsg_grid_clumping_chr): the default 7 x 4 grid on one LD-structured chromosome whose
largest window (50 Mb) holds thousands of SNPs, as hard calls and as a CODE_DOSAGE FBM built from them.

    python tools/bench_grid_clumping.py [--n 50000] [--m 40000] [--mb 250] [--m-dosage 10000] [--out DIR]

Per matrix: the whole call (wall, after a warm-up call on a slice), and from torch.profiler (CUPTI) in the same call the
device time of the pair pass (Gram or dosage tiles, their epilogue) and of the rounds (k_grid_round launches).  Counts:
pairs of the band, useful MACs (pairs x n), their rate as a share of the H100 SXM data-sheet dense INT8 rate (1,979 TOPS =
989.5e12 MAC/s), the number of rounds.  The CPU figure is the oracle's literal grid loop (tests/grid_ref.py: R/SCT.R over
clumping_chr_cached, one thread) on a subsample, next to the GPU on the same subsample.  The GPU name, power limit and SM
clock are read in the same run.  One JSON line to stdout (and DIR/bench_grid_clumping.json).
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
INT8_DENSE_MACS = 989.5e12  # H100 SXM data sheet: 1,979 dense INT8 TOPS


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def band_pairs(pos, size):
    """Pairs of the union window at `size` (integer positions: both tests agree)."""
    left = np.searchsorted(pos, pos - size, side="left")
    return int(np.sum(np.arange(pos.size) - left))


def profiled_call(B, g, chr_, pos, lp):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.time()
        res = B.snp_grid_clumping(g, chr_, pos, lp)
        wall = time.time() - t0
    pair_us, round_us, rounds = 0.0, 0.0, 0
    for ev in prof.key_averages():
        name = ev.key
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if "k_grid_round" in name:
            round_us += t
            rounds += ev.count
        elif any(k in name for k in ("k_dos_pairs", "k_dos_compact", "gram", "k_cor_from_sums", "k_compact", "k_line_counts")):
            pair_us += t
    return res, wall, pair_us / 1e3, round_us / 1e3, rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000)
    ap.add_argument("--m", type=int, default=40000)
    ap.add_argument("--mb", type=float, default=250.0)
    ap.add_argument("--m-dosage", type=int, default=10000)
    ap.add_argument("--cpu-n", type=int, default=5000)
    ap.add_argument("--cpu-m", type=int, default=2000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import bigsnpr_b200 as B
    from oracle import ref
    from tests import grid_ref

    n, m = args.n, args.m
    rng = np.random.default_rng(3)
    pos = np.round(np.linspace(1, args.mb * 1e6, m))
    lp = -np.log10(rng.uniform(size=m))
    size_max = 1000 * 500 / 0.01
    res = {"n": n, "m": m, "span_Mb": args.mb, "grid": "7 thr.r2 x 4 base.size (defaults)", "gpu_start": gpu_info()}

    g = B.Bed.synthetic(n, m, seed=5, ld_rho=0.9, ld_block=50)
    B.snp_grid_clumping(g, np.ones(m, dtype=int), pos, lp, ind_row=np.arange(1, 2001), exclude=np.arange(2001, m + 1))  # warm-up
    out, wall, pair_ms, round_ms, rounds = profiled_call(B, g, np.ones(m, dtype=int), pos, lp)
    pairs = band_pairs(pos, size_max)
    res["hard"] = {"whole_call_s": round(wall, 3), "pair_pass_ms": round(pair_ms, 1), "rounds_ms": round(round_ms, 1),
                   "round_launches": rounds, "pairs": pairs, "macs": pairs * n,
                   "pair_pass_share_of_dense_int8": round(pairs * n / (pair_ms * 1e-3) / INT8_DENSE_MACS, 4),
                   "kept_min_max": [min(len(k) for k in out[0]), max(len(k) for k in out[0])]}

    # dosages: hard calls of the first m_dosage columns, moved off the integers (codes 7 + 100 * value, |jitter| <= 0.2)
    md = args.m_dosage
    G = ref.decode_dense(ref.OracleBed.from_packed(g.export_packed(), n, m)).astype(np.int16)[:, :md]
    g.close()
    jit = rng.integers(-20, 21, size=G.shape, dtype=np.int16)
    Gd = np.asfortranarray((7 + np.clip(100 * np.minimum(G, 2) + jit, 0, 200)).astype(np.uint8))
    del G, jit
    gd = B.Bed.from_fbm(Gd, code256=CODE_DOSAGE)
    assert gd.dosage_scale == 100
    posd = pos[:md]
    B.snp_grid_clumping(gd, np.ones(md, dtype=int), posd, lp[:md], ind_row=np.arange(1, 2001),
                        exclude=np.arange(1001, md + 1))  # warm-up
    out, wall, pair_ms, round_ms, rounds = profiled_call(B, gd, np.ones(md, dtype=int), posd, lp[:md])
    pairs = band_pairs(posd, size_max)
    res["dosage"] = {"m": md, "span_Mb": round(posd[-1] / 1e6, 1), "whole_call_s": round(wall, 3),
                     "pair_pass_ms": round(pair_ms, 1), "rounds_ms": round(round_ms, 1), "round_launches": rounds,
                     "pairs": pairs, "macs": pairs * n,
                     "pair_pass_share_of_dense_int8": round(pairs * n / (pair_ms * 1e-3) / INT8_DENSE_MACS, 4),
                     "kept_min_max": [min(len(k) for k in out[0]), max(len(k) for k in out[0])]}
    gd.close()

    # CPU: the oracle's literal grid loop on a subsample of the dosage matrix, and the GPU on the same subsample
    cn, cm = args.cpu_n, args.cpu_m
    sub = np.asfortranarray(Gd[:cn, :cm])
    del Gd
    o = ref.OracleFBM(sub, CODE_DOSAGE)
    t0 = time.time()
    want, _ = grid_ref.snp_grid_clumping(o, np.ones(cm, dtype=int), posd[:cm], lp[:cm])
    t_cpu = time.time() - t0
    gs = B.Bed.from_fbm(sub, code256=CODE_DOSAGE)
    t0 = time.time()
    got = B.snp_grid_clumping(gs, np.ones(cm, dtype=int), posd[:cm], lp[:cm])
    t_gpu = time.time() - t0
    res["cpu_subsample"] = {"n": cn, "m": cm, "oracle_one_thread_s": round(t_cpu, 2), "gpu_s": round(t_gpu, 3),
                            "identical": all(np.array_equal(a, b) for a, b in zip(got[0], want[0]))}
    res["gpu_end"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_grid_clumping.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
