"""Where the ICP iteration's bookkeeping time goes: the bench batch (N distinct C2 pairs, seeds 1000.., resident in ONE
context, host launch loop) run R times under torch.profiler (CUDA activities). Prints the device time of k_resolve,
k_accumulate and k_solve per iteration (the n-th launch of a run is iteration n) and in total, next to what
k_accumulate has to do in that iteration: the live chunks it visits and the bytes it moves. Both are upper bounds:
iteration 0 is counted from the raw class sizes (the ingest's intersection filter may drop sources before it), and the
bytes assume that every kept source gathers a target.
    python scripts/gpu_bookkeeping_profile.py [--pairs 64] [--runs 5] [--lib LIB] [--out out.json]
LIB is a libmulls_b200.so to profile instead of this tree's (for example a build of the parent commit). The card's
name, power limit and clocks are printed with the numbers; with --out everything is also written there."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from collections import defaultdict
from concurrent.futures import ProcessPoolExecutor

import numpy as np

from mulls_b200 import abi, synth

KERNELS = ("k_resolve", "k_accumulate", "k_solve")
CHUNK = 128  # sources per chunk (kIterBlock)
# k_accumulate's bytes per source (DESIGN §4): the 1-byte flag of every live source; a kept source reads position,
# normal, match and distance (40 B), gathers its target if it passed (32 B, counted for every kept one) and writes its
# compacted copy and correspondence (44 B)
B_LIVE, B_KEPT = 1, 40 + 32 + 44


def _gen(a):
    p = synth.make_pair(a[0], a[1])
    return {"tgt": p["tgt"], "src": p["src"], "params": bytes(p["params"]), "init_guess": p["init_guess"]}


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip()


def short(name):
    return name.split("(")[0].replace("void ", "").replace("mulls::", "").split("<")[0]


ap = argparse.ArgumentParser()
ap.add_argument("--pairs", type=int, default=64)
ap.add_argument("--runs", type=int, default=5)
ap.add_argument("--lib", default=None)
ap.add_argument("--out", default=None)
args = ap.parse_args()
if args.lib:
    abi.LIB_PATH = os.path.abspath(args.lib)  # read when the library is first opened

with ProcessPoolExecutor(min(16, args.pairs)) as ex:
    pairs = list(ex.map(_gen, [(1000 + i, "c2") for i in range(args.pairs)]))
for p in pairs:
    p["params"] = abi.IcpParams.from_buffer_copy(p["params"])
ns = max(sum(len(s) for s in p["src"]) for p in pairs)
nt = max(sum(len(t) for t in p["tgt"]) for p in pairs)

import torch
from torch.profiler import ProfilerActivity, profile

from mulls_b200.registration import Context

ctx = Context(0, args.pairs, ns, nt)
ctx.set_tunable("use_graph", 0)  # host launch loop: one launch of each kernel per iteration
ctx.upload(pairs)
_, traces = ctx.run_resident(want_trace=True)
for _ in range(3):
    ctx.run_resident()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(args.runs):
        ctx.run_resident()
    torch.cuda.synchronize()
info = gpu_info()
ctx.close()

# per iteration: live sources (class sizes at its start; for iteration 0 the raw input sizes, an upper bound), live
# chunks, kept sources (class sizes after its compaction, from the trace)
n_iter = max(t["n_iter"] for t in traces)
live_src, live_chunks, kept_src = np.zeros(n_iter, np.int64), np.zeros(n_iter, np.int64), np.zeros(n_iter, np.int64)
for p, t in zip(pairs, traces):
    start = np.array([len(s) for s in p["src"]], np.int64)
    for i in range(t["n_iter"]):
        after = np.asarray(t["n_src"][i], np.int64)
        live_src[i] += start.sum()
        live_chunks[i] += ((start + CHUNK - 1) // CHUNK).sum()
        kept_src[i] += after.sum()
        start = after

starts = defaultdict(list)
for ev in prof.events():
    if ev.device_type == torch.autograd.DeviceType.CUDA and short(ev.name) in KERNELS:
        starts[short(ev.name)].append((ev.time_range.start, ev.time_range.elapsed_us() / 1000.0))
per_iter = {}
for k in KERNELS:
    evs = sorted(starts[k])
    per_run = len(evs) // args.runs
    assert per_run * args.runs == len(evs) and per_run > 0, (k, len(evs))
    ms = np.zeros(per_run)
    for idx, (_, dt) in enumerate(evs):
        ms[idx % per_run] += dt / args.runs
    per_iter[k] = ms
launches = len(per_iter["k_accumulate"])

print(f"GPU (name, power limit, max SM clock, SM clock after the runs): {info}")
print(f"{args.pairs} pairs, {args.runs} profiled runs, {launches} iterations launched per run, "
      f"library {abi.LIB_PATH}")
print(f"{'iter':>4} {'k_resolve':>10} {'k_accum':>10} {'k_solve':>10} {'chunks':>8} {'live src':>10} {'kept src':>10} "
      f"{'MB<=':>8} {'us/kchunk':>10} {'GB/s<=':>8}  (iteration 0: chunks and live sources are upper bounds)")
rows = []
for i in range(launches):
    a = per_iter["k_accumulate"][i]
    ch = int(live_chunks[i]) if i < n_iter else 0
    mb = (B_LIVE * live_src[i] + B_KEPT * kept_src[i]) / 1e6 if i < n_iter else 0.0
    row = {"iter": i, **{k: round(float(per_iter[k][i]), 4) for k in KERNELS}, "live_chunks": ch,
           "live_src": int(live_src[i]) if i < n_iter else 0, "kept_src": int(kept_src[i]) if i < n_iter else 0,
           "accumulate_MB_upper_bound": round(mb, 2), "counts_upper_bound": i == 0}
    rows.append(row)
    print(f"{i:4d} {per_iter['k_resolve'][i]:10.4f} {a:10.4f} {per_iter['k_solve'][i]:10.4f} {ch:8d} "
          f"{row['live_src']:10d} {row['kept_src']:10d} {mb:8.2f} {1e3 * a / max(ch, 1) * 1e3:10.3f} "
          f"{mb / max(a, 1e-9):8.1f}")
totals = {k: round(float(per_iter[k].sum()), 4) for k in KERNELS}
print("total ms per run: " + ", ".join(f"{k} {v:.3f}" for k, v in totals.items())
      + f"; k_accumulate + k_solve {totals['k_accumulate'] + totals['k_solve']:.3f}")
if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump({"gpu": info, "lib": abi.LIB_PATH, "n_pairs": args.pairs, "runs": args.runs, "per_iteration": rows,
                   "ms_per_run": totals}, f, indent=1)
