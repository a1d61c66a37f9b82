"""Statistical outlier filter (mulls_sor_filter, CFilter::sor_filter) on synthetic merged maps of about 2, 8 and 30 M
points (synth.make_merged_map: 16 sweeps of a drive, repeated along the street), mean_k = 20, n_std = 2.0.
For every size, in one process:
  - a warm-up call, then R timed calls, each a host clock around the whole call (H2D, ingest, kernels, D2H: the call
    synchronises before it returns);
  - a separate call under torch.profiler (CUDA activities): device time per phase (ingest kernels, k_sor_dist,
    k_sor_stats, k_sor_mark, the copies);
  - the CPU restatement (tests/harness/sor_oracle.cpp, built into a temporary directory) on the same cloud with every
    core, and with one thread ("reference-shaped": PCL runs the queries on one thread) on the sizes listed in
    --single-thread;
  - the GPU keep mask, mean distances and statistics against the restatement's.
The card's name, power limit and max SM clock are read in the same call.
    python scripts/gpu_sor_bench.py [--sizes 2,8,30] [--reps 5] [--oracle 2,8,30] [--single-thread 2] [--out file.json]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np

from mulls_b200 import synth
from mulls_b200.registration import Context

MEAN_K, N_STD = 20, 2.0
SOR = ("k_sor_dist", "k_sor_stats", "k_sor_mark")


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip()


def phase_of(name):
    if "Memcpy" in name or "memcpy" in name:
        return "D2H" if ("DtoH" in name or "Device -> Pageable" in name or "Device -> Pinned" in name) else (
            "H2D" if ("HtoD" in name or "-> Device" in name) else "copy")
    for k in SOR:
        if k in name:
            return k
    return "ingest"


def make_map(millions):
    copies = max(1, int(round(millions / 2.0)))
    return synth.make_merged_map(11, 16, n_points=120000, n_copies=copies)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="2,8,30")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle", default="2,8,30", help="sizes (M) on which the all-core oracle runs (and is compared)")
    ap.add_argument("--single-thread", default="2", help="sizes (M) on which the one-thread oracle runs too")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    sizes = [float(s) for s in a.sizes.split(",")]
    single = {float(s) for s in a.single_thread.split(",") if s}
    with_oracle = {float(s) for s in a.oracle.split(",") if s}
    # (test infrastructure: the CPU restatement the GPU result is compared with; its library goes to a temporary directory)
    from test_sor import oracle_sor_filter, sor_oracle_lib

    lib_dir = tempfile.mkdtemp(prefix="sor_oracle_")

    import torch
    from torch.profiler import ProfilerActivity, profile

    clouds = {s: make_map(s) for s in sizes}
    cap = max(len(c) for c in clouds.values())
    ctx = Context(0, 1, 4096, cap)
    res = {"gpu": gpu_info(), "mean_k": MEAN_K, "n_std": N_STD,
           "oracle_threads": sor_oracle_lib(lib_dir).orc_num_threads(), "sizes": []}
    print(res["gpu"], flush=True)
    for s in sizes:
        cloud = clouds[s]
        n = len(cloud)
        keep, dist, st = ctx.sor_filter(cloud, MEAN_K, N_STD)  # warm-up (also grows the hash pool if it must)
        wall = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            ctx.sor_filter(cloud, MEAN_K, N_STD)
            wall.append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ctx.sor_filter(cloud, MEAN_K, N_STD)
            torch.cuda.synchronize()
        phase = defaultdict(float)
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                phase[phase_of(ev.name)] += ev.time_range.elapsed_us() / 1000.0
        cpu_all = cpu_one = same = None
        if s in with_oracle:
            t0 = time.perf_counter()
            o = oracle_sor_filter(cloud, MEAN_K, N_STD, threads=0, lib_dir=lib_dir)
            cpu_all = (time.perf_counter() - t0) * 1e3
            same = bool(np.array_equal(keep, o[0]) and np.array_equal(dist.view(np.uint32), o[1].view(np.uint32)) and
                        all(np.float64(st[k]).tobytes() == np.float64(o[2][k]).tobytes() for k in ("mean", "stddev", "threshold")))
        if s in single:
            t0 = time.perf_counter()
            oracle_sor_filter(cloud, MEAN_K, N_STD, threads=1, lib_dir=lib_dir)
            cpu_one = (time.perf_counter() - t0) * 1e3
        row = {"size_m": s, "n_points": n, "n_kept": int(st["n_kept"]), "threshold": st["threshold"],
               "ms_call_median": float(np.median(wall)), "ms_call_all": [round(v, 3) for v in wall],
               "ms_device_phase": {k: round(v, 3) for k, v in sorted(phase.items())},
               "ms_cpu_oracle_all_cores": None if cpu_all is None else round(cpu_all, 1),
               "ms_cpu_oracle_one_thread": None if cpu_one is None else round(cpu_one, 1),
               "identical_to_oracle": same}
        res["sizes"].append(row)
        print(json.dumps(row), flush=True)
        dump(res, a.out)  # after every size: a partial run still leaves its numbers
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
