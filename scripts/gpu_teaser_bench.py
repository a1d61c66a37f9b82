"""Times mulls_coarse_reg_teaser (CRegistration::coarse_reg_teaser, cregistration.hpp:664-759) against the CPU
restatement (tests/harness/teaser_oracle.cpp) and writes records/h100_teaser_bench.json.

Inputs, through the device NCC matching:
  - the loop pair 000000 / 000015 in best-n mode with corr_num 1 000 (test/mulls_slam.cpp's --feature_corr_num) and
    4 000 at noise_bound 0.6 (pca_neigh_r), and in plain mode (script/run_mulls_reg.sh: --fixed_num_corr_on=false
    --reciprocal_corr_on=false) at noise_bound 1.0 (4 x keypoint_nms_radius);
  - the consecutive scans 000000 / 000001 in best-n mode with corr_num 1 000 and in reciprocal mode, noise_bound 0.6;
  - a synthetic set of 8 000 correspondences at 10 % inliers, noise_bound 0.2.
Per entry:
  - the call's device span (CUDA events around everything it enqueues: copies, kernels, the host waits between search
    launches), median of 9 after a warm-up, and a host clock around the whole call;
  - the kernel time split into the graph (k_tm_graph), the clique (core numbers, greedy bound, pruning and the search)
    and GNC plus voting, from torch.profiler in a separate pass;
  - the restatement on one thread, one run, and whether status, matrix bits and counts equal it in this run.
The card's name, power limit and maximum SM clock are read in the same call.

    python scripts/gpu_teaser_bench.py [--out records/h100_teaser_bench.json]
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
from test_ransac import scene  # noqa: E402
from test_teaser import oracle_teaser, teaser_oracle_lib  # noqa: E402

PHASES = {"k_tm_graph": "graph", "k_tm_hindex": "clique", "k_tm_greedy": "clique", "k_tm_compact": "clique",
          "k_tm_search": "clique", "k_tm_gnc": "gnc_vote", "k_tm_vote": "gnc_vote"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "h100_teaser_bench.json"))
    a = ap.parse_args()
    from test_gpu_ransac import vertex_clouds

    ctx = Context(0, 1, 40000, 40000)
    sets = []
    t, s = vertex_clouds(0, 15)
    for k in (1000, 4000):
        ti, si = ctx.ncc_correspondences(t, s, True, k, False)
        sets.append((f"demo_000000_000015_best{k}", t[ti], s[si], 0.6))
    ti, si = ctx.ncc_correspondences(t, s, False, 0, False)
    sets.append(("demo_000000_000015_plain", t[ti], s[si], 1.0))
    t, s = vertex_clouds(0, 1)
    ti, si = ctx.ncc_correspondences(t, s, True, 1000, False)
    sets.append(("demo_000000_000001_best1000", t[ti], s[si], 0.6))
    ti, si = ctx.ncc_correspondences(t, s, False, 0, True)
    sets.append(("demo_000000_000001_reciprocal", t[ti], s[si], 0.6))
    t, s, _ = scene(8000, 0.1, 5)
    sets.append(("synthetic_8000_10pct", t, s, 0.2))
    rec = {"card": card(), "entries": []}
    teaser_oracle_lib()  # built before the first timed run
    import torch
    from torch.profiler import ProfilerActivity, profile

    for name, t, s, nb in sets:
        t0 = time.perf_counter()
        exp = oracle_teaser(t, s, noise_bound=nb)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        status, T, info = ctx.coarse_reg_teaser(t, s, noise_bound=nb, tran_mat=np.full((4, 4), 7.0))
        launches = info.pop("search_launches")
        na, nb_ = np.isnan(T), np.isnan(exp["T"])
        equal = (status, info) == (exp["status"], exp["info"]) and np.array_equal(na, nb_) and \
            np.array_equal(T[~na].view(np.uint64), exp["T"][~nb_].view(np.uint64))
        dev, host = [], []
        for _ in range(10):
            h0 = time.perf_counter()
            ctx.coarse_reg_teaser(t, s, noise_bound=nb)
            host.append((time.perf_counter() - h0) * 1e3)
            dev.append(ctx.stats()["ms_total"])
        dev, host = dev[1:], host[1:]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ctx.coarse_reg_teaser(t, s, noise_bound=nb)
            torch.cuda.synchronize()
        split = {"graph": 0.0, "clique": 0.0, "gnc_vote": 0.0}
        kernels = {}
        for ev in prof.key_averages():
            for k, ph in PHASES.items():
                if k in ev.key:
                    split[ph] += ev.device_time_total / 1e3
                    kernels[k] = {"calls": ev.count, "total_us": round(ev.device_time_total, 1)}
        e = {"set": name, "n": len(t), "noise_bound": nb, "status": status, "info": info, "search_launches": launches,
             "device_ms_median": round(float(np.median(dev)), 3), "device_ms": [round(x, 3) for x in dev],
             "host_ms_median": round(float(np.median(host)), 3), "kernel_ms_split": {k: round(v, 3) for k, v in split.items()},
             "kernels": kernels, "restatement_1_thread_ms": round(cpu_ms, 1), "equal_to_restatement": bool(equal)}
        rec["entries"].append(e)
        print(json.dumps(e), flush=True)
    ctx.close()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("card:", rec["card"], "all equal:", all(e["equal_to_restatement"] for e in rec["entries"]))


if __name__ == "__main__":
    main()
