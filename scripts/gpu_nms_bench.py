"""Keypoint non-maximum suppression (mulls_non_max_suppress, CFilter::non_max_suppress in place, cfilter.hpp:1183-1240)
at the radius test/mulls_reg.cpp uses (0.25 x pca_neigh_r = 0.25 m) on:
  - the vertex clouds of the 16 demo scans (tests/golden/demo_chain.npz through the device front end with the
    parameters of test/mulls_reg.cpp, about 800 to 1 100 points each: the drivers' operating point);
  - those 16 clouds in one (submap-like, heavy suppression across chunks);
  - synthetic clouds of 20 000 and 120 000 points, about 8 points per r^3.
For every input, in one process: a warm-up call, then R timed calls, each with a host clock around the whole call (H2D,
kernels, D2H: the call synchronises before it returns) and the device span the library's CUDA events record
(mulls_get_stats ms_total); the CPU restatement (tests/harness/nms_oracle.cpp, one thread, built into a temporary
directory) on the same input, timed; and the kept indices against the restatement's. The card's name, power limit and
max SM clock are read in the same call.
    python scripts/gpu_nms_bench.py [--reps 20] [--out records/h100_nms_bench.json]"""
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

from mulls_b200.registration import Context

RADIUS = 0.25


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip()


def synthetic(n, seed):
    rng = np.random.default_rng(seed)
    edge = 0.6 * (n / 1000.0) ** (1 / 3)
    out = np.zeros((n, 12), np.float32)
    out[:, :3] = rng.uniform(-edge, edge, (n, 3))
    out[:, 7] = rng.uniform(0, 1, n)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    # (test infrastructure: the CPU restatement the GPU result is compared with; its library goes to a temporary directory)
    from test_ncc import _chain_mod
    from test_nms import nms_oracle_lib, oracle_nms

    lib_dir = tempfile.mkdtemp(prefix="nms_oracle_")
    nms_oracle_lib(lib_dir)  # compiled here, outside the timed calls
    mod = _chain_mod()
    gp, cp = mod.chain_params()
    z = np.load(os.path.join(ROOT, "tests", "golden", "demo_chain.npz"))
    ctx = Context(0, 1, 4096, 130000)
    inputs = []
    for k in range(16):
        raw = mod.decode_scan(z[f"scan{k}_dmm"], z[f"scan{k}_i"])
        inputs.append((f"demo_vertex_{k:06d}", ctx.extract_semantic_pts(raw, 0.0, gp, cp)["vertex"]))
    inputs.append(("demo_vertex_16_concatenated", np.concatenate([v for _, v in inputs])))
    inputs.append(("synthetic_20000", synthetic(20000, 1)))
    inputs.append(("synthetic_120000", synthetic(120000, 2)))
    res = {"gpu": gpu_info(), "radius": RADIUS, "reps": a.reps, "inputs": []}
    print(res["gpu"], flush=True)
    for name, rows in inputs:
        idx, _ = ctx.non_max_suppress(rows, RADIUS)  # warm-up
        wall, dev = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            ctx.non_max_suppress(rows, RADIUS)
            wall.append((time.perf_counter() - t0) * 1e3)
            dev.append(ctx.stats()["ms_total"])
        t0 = time.perf_counter()
        exp, _ = oracle_nms(rows, RADIUS, lib_dir=lib_dir)
        cpu = (time.perf_counter() - t0) * 1e3
        row = {"input": name, "n_points": len(rows), "n_kept": len(idx), "ms_call_host_median": round(float(np.median(wall)), 4),
               "ms_call_device_median": round(float(np.median(dev)), 4), "ms_cpu_restatement_one_thread": round(cpu, 3),
               "identical_to_restatement": bool(np.array_equal(idx, exp))}
        res["inputs"].append(row)
        print(json.dumps(row), flush=True)
    ctx.close()
    demo = [r for r in res["inputs"] if r["input"].startswith("demo_vertex_0")]
    res["demo_vertex_summary"] = {
        "n_points_range": [min(r["n_points"] for r in demo), max(r["n_points"] for r in demo)],
        "ms_call_host_median_of_medians": round(float(np.median([r["ms_call_host_median"] for r in demo])), 4),
        "ms_call_device_median_of_medians": round(float(np.median([r["ms_call_device_median"] for r in demo])), 4),
        "ms_cpu_restatement_median": round(float(np.median([r["ms_cpu_restatement_one_thread"] for r in demo])), 3)}
    res["all_identical"] = all(r["identical_to_restatement"] for r in res["inputs"])
    res["gpu_after"] = gpu_info()
    print(json.dumps(res["demo_vertex_summary"]), "all identical:", res["all_identical"], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    shutil.rmtree(lib_dir, ignore_errors=True)


if __name__ == "__main__":
    main()
