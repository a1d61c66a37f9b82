"""Times mulls_ncc_correspondences (CRegistration::find_feature_correspondence_ncc, cregistration.hpp:409-601) against the
CPU restatement (tests/harness/ncc_oracle.cpp) and writes records/h100_ncc_bench.json.

Shapes: 1 000^2 (feature_corr_num's default scale), 4 000^2 (the 16-beam flagfile's 4 000), 16 000^2 and one asymmetric
shape; modes: plain, reciprocal, fixed with corr_num 1000 and 4000. Per entry:
  - GPU call: a host clock around the whole call (both copies, every kernel, the host walk), median of 7 after a warm-up;
  - the restatement at 1 and 6 threads (the reference fills its table on min(6, cores) threads), one run each; a
    single-thread run expected to take over a minute (the sort of every pair at 16 000^2) is "not measured";
  - whether the GPU's index pairs equal the restatement's, checked in this run.
Kernel times come from torch.profiler in a separate pass, after the timed one. The card's name, power limit and
maximum SM clock are read in the same call.

    python scripts/gpu_ncc_bench.py [--out records/h100_ncc_bench.json] [--quick]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from mulls_b200.registration import Context  # noqa: E402
from test_ncc import kpts, ncc_oracle_lib, oracle_ncc  # noqa: E402

MODES = [("plain", False, 2000, False), ("reciprocal", False, 2000, True), ("fixed1000", True, 1000, False),
         ("fixed4000", True, 4000, False)]


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


def one_ms(fn):
    t0 = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t0) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "h100_ncc_bench.json"))
    ap.add_argument("--quick", action="store_true", help="1 000^2 and the asymmetric shape only")
    a = ap.parse_args()
    shapes = [(1000, 1000), (4000, 4000), (16000, 16000), (2000, 8000)]
    if a.quick:
        shapes = [(1000, 1000), (2000, 8000)]
    ctx = Context(0, 1, 4096, 20000)
    lib_dir = tempfile.mkdtemp(prefix="ncc_oracle_")
    ncc_oracle_lib(lib_dir)  # compiled here, outside every timed call
    rec = {"card": card(), "what": "mulls_ncc_correspondences vs tests/harness/ncc_oracle.cpp", "entries": []}
    clouds = {}
    for nt, ns in shapes:
        rng = np.random.default_rng(nt * 7 + ns)
        t, s = kpts(nt, rng), kpts(ns, rng)
        clouds[(nt, ns)] = (t, s)
        oracle_ncc(t[:10], s[:10], False, 2000, False, threads=6, lib_dir=lib_dir)  # the OpenMP pool starts untimed
        for name, fixed, corr, recip in MODES:
            e = {"n_t": nt, "n_s": ns, "mode": name}
            gpu_ms, all_ms = med_ms(lambda: ctx.ncc_correspondences(t, s, fixed, corr, recip))
            got = ctx.ncc_correspondences(t, s, fixed, corr, recip)
            e["gpu_call_ms_median"], e["gpu_call_ms"] = round(gpu_ms, 3), all_ms
            e["n_pairs_out"] = int(len(got[0]))
            big_sort = fixed and nt * ns > 100_000_000
            ms6, exp = one_ms(lambda: oracle_ncc(t, s, fixed, corr, recip, threads=6, lib_dir=lib_dir))
            e["restatement_6_threads_ms"] = round(ms6, 1)
            if big_sort:
                e["restatement_1_thread_ms"] = "not measured"
            else:
                ms1, exp1 = one_ms(lambda: oracle_ncc(t, s, fixed, corr, recip, threads=1, lib_dir=lib_dir))
                e["restatement_1_thread_ms"] = round(ms1, 1)
                assert np.array_equal(exp1[0], exp[0]) and np.array_equal(exp1[1], exp[1])
            e["equal_to_restatement"] = bool(np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]))
            print(json.dumps(e), flush=True)
            rec["entries"].append(e)
    # kernel times, in a pass of their own
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile

        prof_out = {}
        for (nt, ns), (t, s) in clouds.items():
            for name, fixed, corr, recip in MODES:
                with profile(activities=[ProfilerActivity.CUDA]) as p:
                    ctx.ncc_correspondences(t, s, fixed, corr, recip)
                    torch.cuda.synchronize()
                k = {}
                for ev in p.key_averages():
                    if ev.device_type == torch.autograd.DeviceType.CUDA or "k_" in ev.key:
                        k[ev.key[:80]] = {"calls": ev.count, "us_total": round(ev.device_time_total, 1)}
                prof_out[f"{nt}x{ns} {name}"] = k
        rec["kernels_torch_profiler"] = prof_out
    except Exception as exc:  # the timed pass above stands on its own
        rec["kernels_torch_profiler"] = f"not measured: {exc}"
    rec["all_equal_to_restatement"] = all(e["equal_to_restatement"] for e in rec["entries"])
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", a.out, "all equal:", rec["all_equal_to_restatement"])
    ctx.close()


if __name__ == "__main__":
    main()
