"""Times mulls_coarse_reg_ransac (CRegistration::coarse_reg_ransac, cregistration.hpp:604-661) against the CPU
restatement (tests/harness/ransac_oracle.cpp) and writes records/h100_ransac_bench.json.

Sizes: N in {1 000, 4 000, 16 000} correspondences (feature_corr_num 1000, the 16-beam flagfile's 4000, and a large
block) x inlier ratio in {2 %, 10 %, 50 %}, max_iter_num 20 000, noise_bound 0.2. Per entry:
  - GPU call: a host clock around the whole call from pageable rows to tran_mat (copies, every kernel, the host-side
    sample stream and k walk), median of 7 after a warm-up;
  - the restatement on one thread, one run (it is sequential, as PCL's rejector is; there is no 6-thread variant);
  - whether the GPU's status, matrix bits, inlier count and hypothesis count equal the restatement's, in this run.
Kernel times come from torch.profiler in a separate pass, after the timed one. The card's name, power limit and
maximum SM clock are read in the same call.

    python scripts/gpu_ransac_bench.py [--out records/h100_ransac_bench.json] [--quick]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from mulls_b200.registration import Context  # noqa: E402
from test_ransac import oracle_ransac, scene  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def med_ms(fn, reps=7):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), [round(t, 3) for t in ts]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "h100_ransac_bench.json"))
    ap.add_argument("--quick", action="store_true", help="N = 1000 only")
    a = ap.parse_args()
    sizes = [1000] if a.quick else [1000, 4000, 16000]
    ratios = [0.02, 0.1, 0.5]
    ctx = Context(0, 1, 4096, max(sizes))
    rec = {"card": card(), "max_iter_num": 20000, "noise_bound": 0.2, "entries": []}
    scenes = {}
    for n in sizes:
        for r in ratios:
            t, s, _ = scene(n, r, 500 + n + int(r * 100))
            scenes[(n, r)] = (t, s)
            t0 = time.perf_counter()
            exp = oracle_ransac(t, s)
            cpu_ms = (time.perf_counter() - t0) * 1e3
            got = ctx.coarse_reg_ransac(t, s, tran_mat=np.full((4, 4), 7.0))
            equal = (got[0], got[2], got[3]) == (exp["status"], exp["n_inliers"], exp["n_hyp"]) and \
                np.array_equal(got[1].view(np.uint64), exp["T"].view(np.uint64))
            gpu_ms, all_ms = med_ms(lambda: ctx.coarse_reg_ransac(t, s))
            e = {"n": n, "inlier_ratio": r, "status": got[0], "n_inliers": got[2], "n_hypotheses": got[3],
                 "gpu_call_ms_median": round(gpu_ms, 3), "gpu_call_ms": all_ms, "restatement_1_thread_ms": round(cpu_ms, 1),
                 "equal_to_restatement": bool(equal)}
            rec["entries"].append(e)
            print(json.dumps(e), flush=True)
    # kernel times, separate pass
    import torch
    from torch.profiler import ProfilerActivity, profile

    kern = {}
    for (n, r), (t, s) in scenes.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ctx.coarse_reg_ransac(t, s)
            torch.cuda.synchronize()
        k = {}
        for ev in prof.key_averages():
            if "ransac" in ev.key:
                k[ev.key.split("(")[0]] = {"calls": ev.count, "total_us": round(ev.device_time_total, 1)}
        kern[f"{n}_{r}"] = k
    rec["kernels_us"] = kern
    ctx.close()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("card:", rec["card"], "all equal:", all(e["equal_to_restatement"] for e in rec["entries"]))


if __name__ == "__main__":
    main()
