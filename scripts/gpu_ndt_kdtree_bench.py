"""NDT registration with the KDTREE neighbourhood (mulls_omp_ndt_kdtree, CRegistration::omp_ndt with
use_direct_search = false) on scripts/gpu_ndt_bench.py's workloads: demo scans 000000 / 000001 raw and voxel-downsampled
on the device at 0.2 and 0.5 m, and synthetic structured pairs of 20 000 and 120 000 source points against a 600 000-point
target. For every input, in one process: a warm-up call, then R timed calls of KDTREE and of DIRECT7 (mulls_omp_ndt) on
the same inputs, alternating, each with a host clock from the pageable rows to Trans1_2 and the device span of the
library's CUDA events (mulls_get_stats ms_total); the iterations and kernel launches; per-kernel device times of one
KDTREE call from a separate torch.profiler pass; and the CPU restatement (tests/harness/ndt_kdtree_oracle.cpp on one thread:
the restatement, not the reference's OpenMP code) timed once, with its result compared bit for bit. The card's name,
power limit and max SM clock are read in the same call.
    python scripts/gpu_ndt_kdtree_bench.py [--reps 10] [--out records/h100_ndt_kdtree_bench.json]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
os.environ.setdefault("OMP_NUM_THREADS", "1")

import numpy as np

from gpu_ndt_bench import gpu_info, workloads
from mulls_b200.registration import Context


def timed(ctx, call, reps):
    host, dev = [], []
    d = None
    for _ in range(reps):
        t0 = time.perf_counter()
        d = call()
        host.append((time.perf_counter() - t0) * 1e3)
        dev.append(ctx.stats()["ms_total"])
    return d, host, dev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "h100_ndt_kdtree_bench.json"))
    a = ap.parse_args()
    from test_ndt import bbox
    from test_ndt_kdtree import oracle_kd

    ctx = Context(0, 1, 700000, 700000)
    rec = dict(gpu=gpu_info(), reps=a.reps, workloads=[])
    for name, t, s, res in workloads(ctx):
        tb, sb = bbox(t), bbox(s)
        kd = lambda: ctx.omp_ndt_kdtree(t, s, tb, sb, res, trace_cap=64)
        d7 = lambda: ctx.omp_ndt(t, s, tb, sb, res, trace_cap=64)
        kd(), d7()
        kh, kdv, dh, ddv = [], [], [], []
        for _ in range(a.reps):  # alternating
            d, h, v = timed(ctx, kd, 1)
            kh += h
            kdv += v
            launches = ctx.stats()["kernel_launches"]
            e, h, v = timed(ctx, d7, 1)
            dh += h
            ddv += v
            launches7 = ctx.stats()["kernel_launches"]
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            kd()
        kernels = {}
        for ev in prof.key_averages():
            if "ndt" in ev.key or "cub" in ev.key or ev.key.startswith(("_ZN5mulls", "void mulls", "mulls::", "k_")):
                kernels[ev.key[:80]] = dict(count=ev.count, ms_total=round(ev.device_time_total / 1e3, 4))
        t0 = time.perf_counter()
        o = oracle_kd(dict(tgt=t, src=s, tb=tb, sb=sb, res=res), trace_cap=64)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        same = (d["code"] == o["code"] and d["iterations"] == o["iterations"] and np.array_equal(d["trans"], o["trans"])
                and np.float64(d["fitness"]).tobytes() == np.float64(o["fitness"]).tobytes()
                and np.array_equal(d["trace"]["score"], o["trace"]["score"]))
        w = dict(name=name, n_target=len(t), n_source=len(s), n_target_filtered=d["n_target"], n_source_filtered=d["n_source"],
                 kdtree=dict(iterations=d["iterations"], code=d["code"], fitness=d["fitness"], kernel_launches=launches,
                             host_ms_median=float(np.median(kh)), device_ms_median=float(np.median(kdv)),
                             host_ms_min=float(np.min(kh)), host_ms_max=float(np.max(kh))),
                 direct7=dict(iterations=e["iterations"], code=e["code"], fitness=e["fitness"], kernel_launches=launches7,
                              host_ms_median=float(np.median(dh)), device_ms_median=float(np.median(ddv))),
                 restatement_one_thread_ms=cpu_ms, equal_to_restatement=bool(same), kernels=kernels)
        rec["workloads"].append(w)
        print(json.dumps({k: v for k, v in w.items() if k != "kernels"}), flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
