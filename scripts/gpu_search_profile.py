"""k_search under the profiler: N distinct C2 pairs resident in ONE context, the whole path run R times.
    ncu --set full --clock-control none --import-source on -k regex:k_search -s <launches of run 1> -c 3 -o gpurun_out/prof \
        python scripts/gpu_search_profile.py 16 2
Without ncu it prints the per-iteration device time of the search kernel (CUDA events on the library's stream)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from mulls_b200 import synth
from mulls_b200.registration import Context

n_pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 16
runs = int(sys.argv[2]) if len(sys.argv) > 2 else 3
cfg = sys.argv[3] if len(sys.argv) > 3 else "c2"
from concurrent.futures import ProcessPoolExecutor
from mulls_b200 import abi
def _gen(a):
    p = synth.make_pair(a[0], a[1])
    return {"tgt": p["tgt"], "src": p["src"], "params": bytes(p["params"]), "init_guess": p["init_guess"]}
with ProcessPoolExecutor(min(32, n_pairs)) as ex:
    pairs = list(ex.map(_gen, [(1000 + i, cfg) for i in range(n_pairs)]))
for p in pairs:
    p["params"] = abi.IcpParams.from_buffer_copy(p["params"])
ns = max(sum(len(s) for s in p["src"]) for p in pairs)
nt = max(sum(len(t) for t in p["tgt"]) for p in pairs)
import torch
a = torch.empty(1 << 28, dtype=torch.uint8, device="cuda"); b = torch.empty_like(a)
for _ in range(3): b.copy_(a)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(10): b.copy_(a)
e1.record(); torch.cuda.synchronize()
print(f"box calibration: device copy {2 * a.numel() * 10 / e0.elapsed_time(e1) / 1e6:.0f} GB/s", flush=True)
del a, b
ctx = Context(0, n_pairs, ns + 16, nt + 16)
ctx.set_tunable("use_graph", 0)  # host launch loop: per-kernel CUDA events
ctx.upload(pairs)
for r in range(runs):
    res, _ = ctx.run_resident()
    st = ctx.stats()
    it = [round(v, 4) for v in st["ms_search_iter"][: int(st["search_launches"])]]
    print(f"run {r}: search {st['ms_search']:.3f} ms over {st['search_launches']} launches {it}; iterate {st['ms_iterate']:.3f} ms, "
          f"ingest {st['ms_ingest']:.3f} ms, total {st['ms_total']:.3f} ms; alg bytes {st['algorithmic_bytes'] / 1e6:.1f} MB -> "
          f"{st['algorithmic_bytes'] / 1e6 / st['ms_search']:.1f} GB/s; iters {[x['iters'] for x in res][:8]}", flush=True)
