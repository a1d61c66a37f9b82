"""Batched NDT registration (mulls_omp_ndt_batch) against its two alternatives, in pairs per second:
  - batch:   one mulls_omp_ndt_batch call over the P pairs;
  - serial:  P mulls_omp_ndt calls one after the other on one context;
  - threads: P contexts driven from P host threads, one mulls_omp_ndt call each (concurrency left to the caller).
Workloads: the 15 consecutive pairs of tests/golden/demo_chain.npz, raw (about 62 000 points a side) and voxel-downsampled
on the device at 0.5 m, and the synthetic pairs of scripts/gpu_ndt_bench.py (20 000 source points against a 600 000-point
target, a different motion per pair) at P = 2 and 4. Each round runs the three ways in turn (the order rotates from
round to round), host clock around each, which ends in a device synchronise; the median over the rounds is reported.
Every result of every way is compared bit for bit with the serial calls. Then, on the workloads of
records/h100_ndt_bench.json, the single call against the batch call with P = 1, alternating. Kernel times come from a
separate torch.profiler pass over one batch call per workload. The card's name, power limit and max SM clock are read
in the same process.
    python scripts/gpu_ndt_batch_bench.py [--rounds 7] [--out records/h100_ndt_batch_bench.json]"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np

from mulls_b200.registration import Context


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip()


def workloads(ctx):
    from test_gpu_ndt import demo_pairs
    from test_ndt import moved, rot, structured_scene

    _, scans = demo_pairs()
    pad = lambda c: np.c_[c, np.zeros((len(c), 4), np.float32)]
    down = [ctx.voxel_downsample(pad(s), 0.5)[:, :3].copy() for s in scans]
    out = [("demo_chain_15_raw", [(scans[k], scans[k + 1]) for k in range(15)]),
           ("demo_chain_15_voxel0.5", [(down[k], down[k + 1]) for k in range(15)])]
    tgt = structured_scene(600000, 31, extent=40.0)
    base = structured_scene(20000, 32, extent=40.0)
    syn = []
    for i in range(4):
        R, tr = rot(0.01 * (i + 1), -0.01, 0.03), np.array([0.3, -0.2 + 0.1 * i, 0.05])
        syn.append((tgt, moved(base, R.T, -R.T @ tr)))
    out += [("synthetic_20k_src_600k_tgt_P2", syn[:2]), ("synthetic_20k_src_600k_tgt_P4", syn)]
    return out


def same(a, b):
    return (a["code"] == b["code"] and a["iterations"] == b["iterations"] and a["n_source"] == b["n_source"]
            and a["n_target"] == b["n_target"] and np.array_equal(a["trans"].view(np.uint64), b["trans"].view(np.uint64))
            and np.float64(a["fitness"]).tobytes() == np.float64(b["fitness"]).tobytes()
            and np.array_equal(a["trace"]["score"].view(np.uint64), b["trace"]["score"].view(np.uint64)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "h100_ndt_batch_bench.json"))
    a = ap.parse_args()
    from test_ndt import bbox

    cap_pts = 700000
    ctx = Context(0, 15, cap_pts, cap_pts)
    rec = dict(gpu=gpu_info(), rounds=a.rounds, workloads=[], single_vs_batch1=[])
    wl = workloads(ctx)
    for name, pairs in wl:
        P = len(pairs)
        tb = [bbox(t) for t, _ in pairs]
        sb = [bbox(s) for _, s in pairs]
        cap = max(max(len(t), len(s)) for t, s in pairs)
        lanes = [Context(0, 1, cap, cap) for _ in range(P)]
        pool = ThreadPoolExecutor(P)

        def batch():
            return ctx.omp_ndt_batch([t for t, _ in pairs], [s for _, s in pairs], tb, sb, trace_cap=64)

        def serial():
            return [ctx.omp_ndt(t, s, tb[i], sb[i], trace_cap=64) for i, (t, s) in enumerate(pairs)]

        def threads():
            futs = [pool.submit(lanes[i].omp_ndt, t, s, tb[i], sb[i], trace_cap=64) for i, (t, s) in enumerate(pairs)]
            return [f.result() for f in futs]

        ways = dict(batch=batch, serial=serial, threads=threads)
        ref = serial()
        equal = {k: all(same(x, y) for x, y in zip(f(), ref)) for k, f in ways.items()}  # also the warm-up
        times = {k: [] for k in ways}
        order = list(ways)
        for r in range(a.rounds):
            for k in order[r % 3:] + order[:r % 3]:
                t0 = time.perf_counter()
                got = ways[k]()
                times[k].append(time.perf_counter() - t0)
                equal[k] = equal[k] and all(same(x, y) for x, y in zip(got, ref))
        ctx.omp_ndt_batch([t for t, _ in pairs], [s for _, s in pairs], tb, sb)
        st = ctx.stats()
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            batch()
        kernels = {}
        for e in prof.key_averages():
            if "ndt" in e.key or "cub" in e.key or e.key.startswith(("_ZN5mulls", "void mulls", "mulls::", "k_")):
                kernels[e.key[:80]] = dict(count=e.count, ms_total=round(e.device_time_total / 1e3, 4))
        w = dict(name=name, pairs=P, n_source=[len(s) for _, s in pairs], n_target=[len(t) for t, _ in pairs],
                 iterations=[d["iterations"] for d in ref], codes=[d["code"] for d in ref],
                 equal_to_serial=equal, batch_kernel_launches=st["kernel_launches"], batch_device_ms=st["ms_total"],
                 pairs_per_s={k: P / float(np.median(v)) for k, v in times.items()},
                 ms_median={k: 1e3 * float(np.median(v)) for k, v in times.items()},
                 ms_min={k: 1e3 * float(np.min(v)) for k, v in times.items()}, kernels=kernels)
        w["batch_over_threads"] = w["pairs_per_s"]["batch"] / w["pairs_per_s"]["threads"]
        w["batch_over_serial"] = w["pairs_per_s"]["batch"] / w["pairs_per_s"]["serial"]
        rec["workloads"].append(w)
        print(json.dumps({k: v for k, v in w.items() if k != "kernels"}), flush=True)
        pool.shutdown()
        for c in lanes:
            c.close()
    # the single call against the batch call with P = 1, on the workloads of records/h100_ndt_bench.json
    from gpu_ndt_bench import workloads as single_workloads

    for name, t, s, res in single_workloads(ctx):
        tb, sb = bbox(t), bbox(s)
        one = lambda: ctx.omp_ndt(t, s, tb, sb, res, trace_cap=64)
        bat = lambda: ctx.omp_ndt_batch([t], [s], [tb], [sb], res, trace_cap=64)[0]
        eq = same(one(), bat())
        ts = dict(single=[], batch1=[])
        for r in range(2 * a.rounds):
            for k, f in ((("single", one), ("batch1", bat)) if r % 2 == 0 else (("batch1", bat), ("single", one))):
                t0 = time.perf_counter()
                f()
                ts[k].append(time.perf_counter() - t0)
        w = dict(name=name, equal=bool(eq), ms_median={k: 1e3 * float(np.median(v)) for k, v in ts.items()},
                 ms_min={k: 1e3 * float(np.min(v)) for k, v in ts.items()})
        rec["single_vs_batch1"].append(w)
        print(json.dumps(w), flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
