"""Point-wise GICP registration (mulls_omp_gicp_pcl, CRegistration::omp_gicp with using_voxel_gicp=False: PCL's
GeneralizedIterativeClosestPoint with its BFGS solver) on the workloads of records/h100_gicp_bench.json:
  - demo scans 000000 / 000001 of tests/golden/demo_chain.npz, raw (about 62 000 points a side) and voxel-downsampled on
    the device at 0.2 and 0.5 m;
  - synthetic structured pairs (tests/test_ndt.py's scene) of 20 000 and 120 000 source points against a 600 000-point
    target;
all with max_iter_num 20 (omp_gicp's default).
For every input, in one process: a warm-up call, then R timed calls with a host clock from the pageable rows to
Trans1_2 (the call synchronises before it returns), the device span of the library's CUDA events (mulls_get_stats
ms_total, which includes the host's BFGS between the evaluations and the small downloads), the kernel launches, the
outer iterations and the functor calls; per-kernel device times from a separate torch.profiler pass; and the CPU
restatement (tests/harness/gicp_pcl_oracle.cpp on one thread: the restatement, not the reference's OpenMP code) on the
same input, timed once, with its result compared bit for bit. The card's name, power limit and max SM clock are read in
the same call.
    python scripts/gpu_gicp_pcl_bench.py [--reps 5] [--out records/h100_gicp_pcl_bench.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
os.environ.setdefault("OMP_NUM_THREADS", "1")

import numpy as np

from mulls_b200.registration import Context


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip()


def workloads(ctx):
    from test_gpu_ndt import demo_pairs  # noqa: F401 (the demo scans)
    from test_ndt import moved, rot, structured_scene

    _, scans = demo_pairs()
    t, s = scans[0], scans[1]
    out = [("demo_0_1_raw", t, s, 1.0)]
    for v in (0.2, 0.5):
        pad = lambda c: np.c_[c, np.zeros((len(c), 4), np.float32)]
        out.append((f"demo_0_1_voxel{v}", ctx.voxel_downsample(pad(t), v)[:, :3].copy(),
                    ctx.voxel_downsample(pad(s), v)[:, :3].copy(), 1.0))
    tgt = structured_scene(600000, 31, extent=40.0)
    R, tr = rot(0.01, -0.01, 0.03), np.array([0.3, -0.2, 0.05])
    for n in (20000, 120000):
        src = moved(structured_scene(n, 32, extent=40.0), R.T, -R.T @ tr)
        out.append((f"synthetic_{n // 1000}k_src_600k_tgt", tgt, src, 1.0))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "h100_gicp_pcl_bench.json"))
    a = ap.parse_args()
    from test_gicp_pcl import oracle_gicp_pcl
    from test_ndt import bbox

    ctx = Context(0, 1, 700000, 700000)
    rec = dict(gpu=gpu_info(), reps=a.reps, workloads=[])
    for name, t, s, res in workloads(ctx):
        tb, sb = bbox(t), bbox(s)
        def call():
            return ctx.omp_gicp_pcl(t, s, tb, sb, max_iter_num=20, trace_cap=256)

        d = call()
        host, dev = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            d = call()
            host.append((time.perf_counter() - t0) * 1e3)
            dev.append(ctx.stats()["ms_total"])
        launches = ctx.stats()["kernel_launches"]
        import torch
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
        kernels = {}
        for e in prof.key_averages():
            if e.key.startswith(("_ZN5mulls", "void mulls", "mulls::", "void cub", "k_")) or "gicp" in e.key or "Select" in e.key or "cub" in e.key:
                kernels[e.key[:80]] = dict(count=e.count, ms_total=round(e.device_time_total / 1e3, 4))
        t0 = time.perf_counter()
        o = oracle_gicp_pcl(dict(tgt=t, src=s, tb=tb, sb=sb), max_iter=20, trace_cap=256)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        same = (d["code"] == o["code"] and d["iterations"] == o["iterations"] and np.array_equal(d["trans"], o["trans"])
                and np.float64(d["fitness"]).tobytes() == np.float64(o["fitness"]).tobytes())
        w = dict(name=name, n_target=len(t), n_source=len(s), n_target_filtered=d["n_target"], n_source_filtered=d["n_source"],
                 iterations=d["iterations"], converged=d["converged"], code=d["code"], fitness=d["fitness"],
                 functor_calls=int(d["trace"]["evaluations"].sum()), kernel_launches=launches,
                 host_ms_median=float(np.median(host)), device_ms_median=float(np.median(dev)),
                 device_ms_per_iteration=float(np.median(dev)) / max(d["iterations"], 1),
                 restatement_one_thread_ms=cpu_ms, equal_to_restatement=bool(same), kernels=kernels)
        rec["workloads"].append(w)
        print(json.dumps({k: v for k, v in w.items() if k != "kernels"}), flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
