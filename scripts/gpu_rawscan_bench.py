"""Raw-scan corrections on the GPU (mulls_vertical_intrinsic_calibration, mulls_timestamp_ratio in both modes,
mulls_motion_compensation for one cloud and for a five-cloud batch) against the CPU restatement
(tests/harness/rawscan_oracle.cpp, built into a temporary directory), at one scan's size (124 668 points,
test_rawscan.scan_like) and on a 1.9 M-point merged map (synth.make_merged_map, curvature = timestamps).
For every entry point and size, in one process:
  - a warm-up call, then R timed calls, each a host clock around the whole call (the H2D copy of the 48-byte rows, the
    kernels, the D2H copy of the changed column: the call synchronises before it returns); median and all;
  - the restatement on 1 thread and on 6 (the reference's OpenMP cap), median of R runs each, on copies of the rows;
  - how many output values differ from the restatement's (timestamps must not differ at all).
The card's name, power limit and max SM clock are read in the same call.
    python scripts/gpu_rawscan_bench.py [--reps 7] [--out file.json]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np

from mulls_b200 import synth
from mulls_b200.registration import Context
from test_rawscan import (TRANSFORMS, orc_batch_motion, orc_motion, orc_ratio, orc_vertical, rawscan_oracle_lib, rows_of,
                          scan_like)

F32 = np.float32


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip()


def timed(fn, reps):
    fn()  # warm-up
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def n_diff(a, b):
    a, b = np.asarray(a, F32).ravel(), np.asarray(b, F32).ravel()
    return int(((a.view(np.uint32) != b.view(np.uint32)) & ~(np.isnan(a) & np.isnan(b))).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    lib_dir = tempfile.mkdtemp(prefix="rawscan_oracle_")
    rawscan_oracle_lib(lib_dir)
    res = {"gpu": gpu_info(), "host_cpus": os.cpu_count(), "reps": a.reps, "rows": []}
    print(res["gpu"], flush=True)
    m = synth.make_merged_map(11, 16, n_points=120000)
    m[:, 9] = np.random.default_rng(3).uniform(0.0, 100.0, len(m)).astype(F32)
    clouds = {"scan": scan_like(124668, np.random.default_rng(8)), "merged_map": m}
    T = TRANSFORMS["small"]
    ctx = Context(0, 1, 16, len(m) + 16)
    for cname, rows in clouds.items():
        n = len(rows)
        ratio_rows = orc_ratio(rows, True, lib_dir=lib_dir)  # the motion compensation reads timestamp ratios
        parts = np.array_split(ratio_rows, 5)  # five feature clouds of the batch
        cases = {
            "vertical_intrinsic_calibration": (
                lambda: ctx.vertical_intrinsic_calibration(rows, 0.5)[0],
                lambda th: orc_vertical(rows, 0.5, threads=th, lib_dir=lib_dir)[0][:, :3]),
            "timestamp_ratio_timestamps": (
                lambda: ctx.timestamp_ratio(rows, True),
                lambda th: orc_ratio(rows, True, threads=th, lib_dir=lib_dir)[:, 9]),
            "timestamp_ratio_azimuth": (
                lambda: ctx.timestamp_ratio(rows, False, 90.0),
                lambda th: orc_ratio(rows, False, 90.0, threads=th, lib_dir=lib_dir)[:, 9]),
            "motion_compensation": (
                lambda: ctx.motion_compensation(ratio_rows, T),
                lambda th: orc_motion(ratio_rows, T, threads=th, lib_dir=lib_dir)[:, :3]),
            "batch_motion_compensation_5": (
                lambda: np.concatenate(ctx.motion_compensation(parts, T)),
                lambda th: np.concatenate([c[:, :3] for c in orc_batch_motion(parts + [rows_of(np.zeros((0, 3)))], T, False,
                                                                              threads=th, lib_dir=lib_dir)[:5]])),
        }
        for name, (gpu, cpu) in cases.items():
            wall = timed(gpu, a.reps)
            g = gpu()
            cpu_ms = {}
            for th in (1, 6):
                cpu_ms[th] = timed(lambda: cpu(th), a.reps)
            row = {"entry": name, "cloud": cname, "n_points": n,
                   "ms_gpu_call_median": round(float(np.median(wall)), 3), "ms_gpu_call_all": [round(v, 3) for v in wall],
                   "ms_cpu_1_thread_median": round(float(np.median(cpu_ms[1])), 3),
                   "ms_cpu_6_threads_median": round(float(np.median(cpu_ms[6])), 3),
                   "values_differing_from_restatement": n_diff(g, cpu(0)), "values": int(np.asarray(g).size)}
            row["gpu_faster_than_1_thread"] = row["ms_gpu_call_median"] < row["ms_cpu_1_thread_median"]
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
            dump(res, a.out)
    ctx.close()
    res["gpu_after"] = gpu_info()
    dump(res, a.out)
    shutil.rmtree(lib_dir, ignore_errors=True)


def dump(res, path):
    if path:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
