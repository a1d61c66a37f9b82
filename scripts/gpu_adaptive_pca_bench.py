"""Cost of distance-adaptive PCA neighbourhoods (use_distance_adaptive_pca, pca.hpp:310-326, unit 30 as
classify_nground_pts passes it) on the GPU: mulls_classify_nground on 20 000 unground points (neighbor_k 50, kitti-urban
thresholds) and mulls_extract_semantic_pts on a synthetic 64-beam scan, adaptive off and on, alternated call by call.
Wall clock around the C-ABI call (host rows in, host clouds out) and device time from the library's CUDA events. Each
configuration is checked once against its CPU restatement (the oracle for off, the adaptive restatement for on).

    python scripts/gpu_adaptive_pca_bench.py [--reps N] [--out file.json]"""
import argparse
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
sys.path.insert(0, "tests")
from mulls_b200 import abi  # noqa: E402
from mulls_b200.registration import Context  # noqa: E402
from oracle import oracle  # noqa: E402
from test_adaptive_pca import orc_classify_adaptive  # noqa: E402
from test_classify import kitti_params, unground_cloud  # noqa: E402
from test_ground import params as ground_params  # noqa: E402
from test_ground import raw_scan  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def same(a, b, keys):
    return all(a[k].shape == b[k].shape and np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)) for k in keys)


def timed(ctx, fn, variants, reps):
    """alternate the variants call by call; median wall / device ms per variant"""
    wall = {v: [] for v in variants}
    dev = {v: [] for v in variants}
    for v in variants:  # warm-up
        fn(variants[v])
    for _ in range(reps):
        for v, arg in variants.items():
            t0 = time.perf_counter()
            fn(arg)
            wall[v].append((time.perf_counter() - t0) * 1e3)
            dev[v].append(ctx.stats()["ms_total"])
    return {v: {"wall_ms_median": float(np.median(wall[v])), "wall_ms_min": float(np.min(wall[v])),
                "device_ms_median": float(np.median(dev[v])), "device_ms_min": float(np.min(dev[v]))} for v in variants}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    ctx = Context(0, 1, 16, 200000)
    res = {"gpu": gpu_info(), "reps": a.reps}

    # classify_nground_pts: 20 000 of the unground points, neighbor_k 50, kitti-urban thresholds
    ung = unground_cloud()
    off = kitti_params(neighbor_k=50, unground_down_fixed_num=20000)
    on = kitti_params(neighbor_k=50, unground_down_fixed_num=20000, use_distance_adaptive_pca=1, pca_unit_distance=30.0)
    g_off, g_on = ctx.classify_nground(ung, off), ctx.classify_nground(ung, on)
    res["classify"] = {
        "input_pts": int(ung.shape[0]), "pca_pts": 20000, "neighbor_k": 50, "radius": 0.7, "pca_down_rate": 2,
        "identical_off_vs_oracle": same(g_off, oracle.classify_nground(ung, off), abi.OUT_NAMES),
        "identical_on_vs_restatement": same(g_on, orc_classify_adaptive(ung, on), abi.OUT_NAMES),
        "sizes_off": {k: int(g_off[k].shape[0]) for k in abi.OUT_NAMES},
        "sizes_on": {k: int(g_on[k].shape[0]) for k in abi.OUT_NAMES},
        "times": timed(ctx, lambda p: ctx.classify_nground(ung, p), {"off": off, "on": on}, a.reps),
    }
    print("classify", json.dumps(res["classify"]), flush=True)

    # extract_semantic_pts on a synthetic 64-beam scan: voxel 0.05 m, ground filter, classification (r 0.7, k 25, stride 2)
    raw, _ = raw_scan()
    gp = ground_params()
    cps = {}
    for name, adaptive in (("off", 0), ("on", 1)):
        cp = abi.default_classify_params()
        cp.neighbor_searching_radius, cp.neighbor_k, cp.neigh_k_min, cp.pca_down_rate = 0.7, 25, 7, 2
        cp.fixed_num_downsampling, cp.unground_down_fixed_num, cp.random_seed = 1, 20000, 3
        cp.use_distance_adaptive_pca, cp.pca_unit_distance = adaptive, 30.0
        cps[name] = cp
    e_off, e_on = (ctx.extract_semantic_pts(raw, 0.05, gp, cps[v]) for v in ("off", "on"))
    down = oracle.voxel_downsample(raw, 0.05)
    og = oracle.fast_ground_filter(down, gp)
    res["extract"] = {
        "raw_pts": int(raw.shape[0]), "unground_pts": int(og["unground"].shape[0]),
        "identical_off_vs_oracle": same(e_off, oracle.classify_nground(og["unground"], cps["off"]), abi.OUT_NAMES),
        "identical_on_vs_restatement": same(e_on, orc_classify_adaptive(og["unground"], cps["on"]), abi.OUT_NAMES),
        "sizes_off": {k: int(v.shape[0]) for k, v in e_off.items()},
        "sizes_on": {k: int(v.shape[0]) for k, v in e_on.items()},
        "times": timed(ctx, lambda cp: ctx.extract_semantic_pts(raw, 0.05, gp, cp), cps, a.reps),
    }
    print("extract", json.dumps(res["extract"]), flush=True)
    ctx.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
