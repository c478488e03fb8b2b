"""SCT end to end on one GPU: snp_grid_clumping -> snp_grid_PRS(type="float") -> snp_grid_stacking, the last step being
big_spLinReg / big_spLogReg over the dense float score matrix (bsg_splreg_dense).

    python tools/bench_grid_stacking.py [--workloads chromosome,genome] [--timeout-chromosome S] [--timeout-genome S]
                                        [--m-cpu 50] [--out DIR]

Workloads (LD-structured synthetic genotypes, ld_rho = 0.9 in 50-SNP blocks; pseudo-chromosomes with increasing
positions at the SNP density of tools/bench_grid_clumping.py, 40,000 SNPs over 250 Mb):
  - chromosome: the 40,000-SNP chromosome of tools/bench_grid_clumping.py at n = 100,000 (28 keep sets x 50 thresholds =
    1,400 columns);
  - genome: 22 x 5,000 SNPs at n = 50,000 (22 x 28 x 50 = 30,800 columns).
Every row is a training row.  Phenotype: 1 % of the SNPs causal with normal effects, heritability 0.3 on the liability;
the continuous y is the liability, the binary y the liability above its 70 % quantile.  big_univLinReg on the continuous
y gives betas and lpS, then the default clumping grid, the float scores and stacking with K = 10 for both phenotypes
(linear and logistic): alpha = 1 alone first, then the default alphas (1, 0.01, 1e-4).

Per workload and family: the device time (bsg_splreg_last_ms: column statistics to the end of the last fit), the
staging time (host gather and upload of the float matrix, bsg_splreg_last_stage_ms), the wall time of the call, the
median lambda steps and coordinate-descent passes per fit, the stop messages and the staged bytes (4 x n x columns).  The
CPU figure is the C oracle (tests/splreg_oracle.c, all host cores, one fit per thread) on the first --m-cpu columns of
the chromosome workload's matrix, linear, alpha = 1, extrapolated linearly in columns (labelled as such).  Each
workload runs in a child process with its own time limit; the parts of one that does not finish in it are reported "not
measured", with the limit.  The GPU name, power limit and SM clock are read in the same run.  One JSON line to stdout (and
DIR/bench_grid_stacking.json).
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

WORKLOADS = {"chromosome": dict(n=100_000, chroms=1, m_chr=40_000), "genome": dict(n=50_000, chroms=22, m_chr=5_000)}
SPAN_PER_SNP = 250e6 / 40_000
ALPHAS = (1.0, 0.01, 1e-4)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def log(msg):
    print(msg, file=sys.stderr, flush=True)


def pipeline(B, n, chroms, m_chr):
    """the score matrix of the SCT pipeline and the two phenotypes"""
    m = chroms * m_chr
    g = B.Bed.synthetic(n, m, seed=31, ld_rho=0.9, ld_block=50)
    rng = np.random.default_rng(1)
    causal = np.sort(rng.choice(m, m // 100, replace=False)) + 1
    Xc = B.read_bed(g, g.rows_along(), causal).astype(np.float64)
    gen = (Xc - Xc.mean(0)) @ rng.normal(size=causal.size)
    gen = gen / np.std(gen) * np.sqrt(0.3)
    y = gen + rng.normal(size=n) * np.sqrt(0.7)
    y01 = (y > np.quantile(y, 0.7)).astype(np.float64)
    t = {}
    t0 = time.time()
    gw = B.big_univLinReg(g, y)
    t["gwas_s"] = time.time() - t0
    lp = -gw.predict()
    chr_ = np.repeat(np.arange(1, chroms + 1), m_chr)
    pos = np.tile(np.round(np.arange(1, m_chr + 1) * SPAN_PER_SNP), chroms)
    t0 = time.time()
    keep = B.snp_grid_clumping(g, chr_, pos, lp)
    t["clumping_s"] = time.time() - t0
    t0 = time.time()
    multi = B.snp_grid_PRS(g, keep, gw.estim, lp, type="float")
    t["prs_s"] = time.time() - t0
    g.close()
    return multi, y, y01, t


def stack(B, multi, y, alphas=ALPHAS):
    t0 = time.time()
    res = B.snp_grid_stacking(multi, y, alphas=alphas, K=10)
    wall = time.time() - t0
    mod = res["mod"]
    steps = mod.nb_lambda.reshape(-1)
    passes = np.array([p["passes"].sum() for row in mod.path for p in row])
    return dict(device_s=B.api.splreg_last_ms() / 1e3, staging_s=B.api.splreg_last_stage_ms() / 1e3, wall_s=wall,
                lambda_steps_per_fit=dict(min=int(steps.min()), median=float(np.median(steps)), max=int(steps.max())),
                passes_per_fit=dict(min=int(passes.min()), median=float(np.median(passes)), max=int(passes.max())),
                messages=sorted(set(m for row in mod.message for m in row)),
                validation_loss=[float(v) for v in mod.validation_loss], nb_var=[int(v) for v in mod.nb_var],
                best_alpha=float(mod.alphas[mod.best_alpha]), kept_columns=int(mod.ind_col.size),
                nonzero_snps=int(np.count_nonzero(res["beta.G"])))


def child(name, m_cpu, out):
    import bigsnpr_b200 as B

    w = WORKLOADS[name]
    multi, y, y01, t = pipeline(B, w["n"], w["chroms"], w["m_chr"])
    n, ncol = multi.shape
    res = dict(n=n, snps=w["chroms"] * w["m_chr"], chromosomes=w["chroms"], columns=ncol,
               staged_bytes=4 * n * ncol, pipeline=t)
    log("%s: %d x %d float scores" % (name, n, ncol))

    def save():  # after every stage, so that a run stopped by its time limit keeps what it measured
        with open(out, "w") as f:
            json.dump(res, f)

    save()
    # alpha = 1 alone first (10 fits, short working sets), then the default three alphas, whose near-ridge fits keep
    # every column in the working set
    for key, yy, al in (("linear_alpha1", y, (1.0,)), ("logistic_alpha1", y01, (1.0,)), ("linear", y, ALPHAS),
                        ("logistic", y01, ALPHAS)):
        log("  %s ..." % key)
        res[key] = stack(B, multi, yy, al)
        log("  %s: %.1f s device, %.1f s staging" % (key, res[key]["device_s"], res[key]["staging_s"]))
        save()
        if m_cpu and key == "linear_alpha1":
            from tests import splreg_ref as S

            sub = np.asarray(multi[:, :m_cpu], dtype=np.float64)
            t0 = time.time()
            S.splreg(sub, y, 0, S.folds_from_seed(n, 10, 1), 10, alphas=(1.0,), engine="c")
            sec = time.time() - t0
            res["cpu_c_oracle"] = dict(what="tests/splreg_oracle.c on all %d host cores, linear, alpha = 1, K = 10, "
                                            "%d rows x the first %d columns" % (os.cpu_count(), n, m_cpu),
                                       seconds=sec, extrapolated_to_all_columns_s=sec * ncol / m_cpu,
                                       note="linear extrapolation in columns, not measured at full width")
            save()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="chromosome,genome")
    ap.add_argument("--timeout-chromosome", type=float, default=1200)
    ap.add_argument("--timeout-genome", type=float, default=600)
    ap.add_argument("--m-cpu", type=int, default=50)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", default=None)
    ap.add_argument("--child-out", default=None)
    a = ap.parse_args()
    if a.child:
        child(a.child, a.m_cpu, a.child_out)
        return
    import tempfile

    res = dict(gpu_start=gpu_info(), host_cores=os.cpu_count(), alphas=list(ALPHAS), K=10, type="float")
    tmp = tempfile.mkdtemp(prefix="bench_grid_stacking_")
    for name in a.workloads.split(","):
        lim = getattr(a, "timeout_" + name)
        out = os.path.join(tmp, name + ".json")
        cmd = [sys.executable, os.path.abspath(__file__), "--child", name, "--child-out", out,
               "--m-cpu", str(a.m_cpu if name == "chromosome" else 0)]
        t0 = time.time()
        p = subprocess.Popen(cmd)
        rc = None
        while rc is None and time.time() - t0 < lim:
            try:
                rc = p.wait(timeout=min(60.0, max(1.0, lim - (time.time() - t0))))
            except subprocess.TimeoutExpired:
                log("  %s: %.0f s" % (name, time.time() - t0))
        if rc is None:
            p.kill()
            p.wait()
        res[name] = json.load(open(out)) if os.path.exists(out) else dict(WORKLOADS[name])
        if rc != 0:  # what the child saved before it stopped is kept; the rest is not measured
            res[name]["status"] = "stopped: %s; parts absent here are not measured" % (
                "did not finish within %.0f s" % lim if rc is None else "exit code %s" % rc)
            res[name]["elapsed_s"] = time.time() - t0
        log("%s done in %.0f s" % (name, time.time() - t0))
    res["gpu_end"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_grid_stacking.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
