import os, sys, time, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import bigsnpr_b200 as B
n, m, size = int(os.environ.get("N", 100000)), int(os.environ.get("M", 20000)), 500
g = B.Bed.synthetic(n, m, seed=20250927, na_rate=float(os.environ.get("NA", "0")), layouts=B.LAYOUT_SNP_MAJOR)
for _ in range(2):
    torch.cuda.synchronize(); t = time.perf_counter(); ld = B.bed_ld_scores(g, size=size); torch.cuda.synchronize(); t_ld = time.perf_counter() - t
print(json.dumps({"na": os.environ.get("NA", "0"), "ld_seconds": t_ld, "ld_sum": float(ld.sum())}))
