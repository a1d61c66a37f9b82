"""Where the ingest's time goes: the bench batch (N distinct C2 pairs, seeds 1000.., resident in ONE context) run R times
under torch.profiler (CUDA activities). Prints, per kernel name, the summed device time per run (the CUB radix-sort
kernels included), the ingest's share of it, and the library's own ms_ingest (CUDA events) of the same runs.
    python scripts/gpu_ingest_profile.py [N=64] [R=5] [out.json]
The card's name, power limit and clocks are printed with the numbers; with out.json everything is also written there."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from collections import defaultdict
from concurrent.futures import ProcessPoolExecutor

from mulls_b200 import abi, synth
from mulls_b200.registration import Context

n_pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 64
runs = int(sys.argv[2]) if len(sys.argv) > 2 else 5
out_path = sys.argv[3] if len(sys.argv) > 3 else None

# the kernels that run before the iteration loop (launch_ingest), CUB's sort kernels and the claim-table memset included
INGEST = ("k_state_init", "k_ingest", "k_pair_setup", "k_make_keys", "k_keepless", "k_digit_scan", "k_sort_pass",
          "k_seg_offsets", "k_cell_count", "k_gather", "k_hash", "DeviceRadixSort", "Memset")


def _gen(a):
    p = synth.make_pair(a[0], a[1])
    return {"tgt": p["tgt"], "src": p["src"], "params": bytes(p["params"]), "init_guess": p["init_guess"]}


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip()


def short(name):
    if "DeviceRadixSort" in name:
        return "cub::" + name[name.index("DeviceRadixSort"):].split("<")[0].split("(")[0]
    if "Memset" in name:
        return "Memset"
    return name.split("(")[0].replace("void ", "").replace("mulls::", "")


with ProcessPoolExecutor(min(16, n_pairs)) as ex:
    pairs = list(ex.map(_gen, [(1000 + i, "c2") for i in range(n_pairs)]))
for p in pairs:
    p["params"] = abi.IcpParams.from_buffer_copy(p["params"])
ns = max(sum(len(s) for s in p["src"]) for p in pairs)
nt = max(sum(len(t) for t in p["tgt"]) for p in pairs)
n_in = sum(sum(len(s) for s in p["src"]) + sum(len(t) for t in p["tgt"]) for p in pairs)

import torch
from torch.profiler import ProfilerActivity, profile

ctx = Context(0, n_pairs, ns, nt)
ctx.set_tunable("use_graph", 0)  # host launch loop: every kernel is a launch of its own
ctx.upload(pairs)
for _ in range(3):
    ctx.run_resident()
torch.cuda.synchronize()
ms_ingest = []
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(runs):
        ctx.run_resident()
        ms_ingest.append(ctx.stats()["ms_ingest"])
    torch.cuda.synchronize()
info_after = gpu_info()
ctx.close()

per_kernel = defaultdict(float)
calls = defaultdict(int)
for ev in prof.events():
    if ev.device_type == torch.autograd.DeviceType.CUDA:
        per_kernel[short(ev.name)] += ev.time_range.elapsed_us() / 1000.0 / runs  # us -> ms per run
        calls[short(ev.name)] += 1
ingest = {k: v for k, v in per_kernel.items() if any(t in k for t in INGEST)}
total = sum(per_kernel.values())
rows = sorted(per_kernel.items(), key=lambda kv: -kv[1])
print(f"GPU (name, power limit, max SM clock, SM clock after the runs): {info_after}")
print(f"{n_pairs} pairs, {n_in} input points, {runs} profiled runs")
print(f"{'kernel':<48} {'ms/run':>8} {'launches/run':>12}  ingest")
for k, v in rows:
    print(f"{k:<48} {v:8.3f} {calls[k] / runs:12.1f}  {'*' if k in ingest else ''}")
ing = sum(ingest.values())
print(f"device time per run: {total:.3f} ms summed over kernels; ingest kernels {ing:.3f} ms")
print(f"ms_ingest (library CUDA events, per run): {[round(v, 3) for v in ms_ingest]}")
if out_path:
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump({"gpu": info_after, "n_pairs": n_pairs, "n_input_points": n_in, "runs": runs,
                   "ms_per_run": {k: round(v, 4) for k, v in rows}, "ingest_kernels": sorted(ingest),
                   "ms_ingest_kernels_sum": round(ing, 4), "ms_kernels_sum": round(total, 4),
                   "ms_ingest_events": [round(v, 4) for v in ms_ingest]}, f, indent=1)
