"""Parent-vs-change A/B of the ICP loop paths: the same inputs through two builds of libmulls_b200.so, each build in its
own subprocess, the two alternating round by round.

    python scripts/gpu_loop_paths_ab.py PARENT_LIB [--rounds N] [--reps R] [--out FILE]

PARENT_LIB is the library built from the commit to compare against (for example into build/parent/); the other side
is this tree's mulls_b200/csrc/libmulls_b200.so. The cases cover every loop path:
  - cooperative: the 2.6k / 20k operating point of scripts/gpu_latency.py, one pair, the cooperative kernel (k_icp_loop);
  - graph: three C2 pairs resident on one context (about 2,800 source chunks, more than the cooperative kernel holds);
  - host loop: the same batch with use_graph = 0;
  - sharded: one C2 pair through mulls_icp_run_sharded at world size 1 (identity all-reduce), the host loop with hook.
Per case and side: a SHA-256 of the result and trace bytes, the integer fields of mulls_run_stats, and the median
device time (ms_total) of R untraced runs. Exits non-zero when the digests or integer stats differ between the sides.
"""
import argparse
import hashlib
import json
import os
import pickle
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
INT_STATS = ("kernel_launches", "algorithmic_bytes", "iterations", "search_launches")


def make_inputs(path):
    import numpy as np

    from mulls_b200 import abi, synth

    def downsample(clouds, counts, seed):  # as scripts/gpu_latency.py
        rng = np.random.default_rng(seed)
        out = []
        for c, k in zip(clouds, counts):
            idx = np.sort(rng.choice(len(c), size=min(k, len(c)), replace=False)) if len(c) else np.arange(0)
            out.append(np.ascontiguousarray(c[idx]))
        return out

    full = synth.make_pair(1000, "c2")
    small = dict(full)
    small["src"] = downsample(full["src"], (800, 400, 1200, 200, 0, 0), 1)
    small["tgt"] = downsample(full["tgt"], (9000, 2000, 7000, 2000, 0, 0), 2)
    p = abi.IcpParams.from_buffer_copy(full["params"])
    p.used_feature_type = b"111100"
    p.target_bound[:] = synth.cloud_bound(small["tgt"])
    small["params"] = p
    c2 = [synth.make_pair(s, "c2") for s in (1001, 1005, 1006)]
    plain = lambda q: dict(tgt=q["tgt"], src=q["src"], params=bytes(q["params"]), init_guess=q["init_guess"])  # noqa: E731
    with open(path, "wb") as f:
        pickle.dump({"small": plain(small), "c2": [plain(q) for q in c2]}, f)


def digest(results, traces):
    import numpy as np

    h = hashlib.sha256()
    for d in list(results) + list(traces):
        for k in sorted(d):
            h.update(k.encode())
            h.update(np.ascontiguousarray(np.asarray(d[k])).tobytes())
    return h.hexdigest()


def worker(lib, inputs, reps, out_path):
    from mulls_b200 import abi

    abi.LIB_PATH = lib  # read when the library is first opened
    from mulls_b200.registration import Context

    with open(inputs, "rb") as f:
        data = pickle.load(f)
    for q in [data["small"]] + data["c2"]:
        q["params"] = abi.IcpParams.from_buffer_copy(q["params"])
    c2 = data["c2"]
    n_c2 = max(max(sum(len(c) for c in q[side]) for q in c2) for side in ("src", "tgt"))
    out = {}

    def measure(name, ctx, run):
        res, tr = run(True)
        st = ctx.stats()
        for _ in range(3):
            run(False)
        ms = []
        for _ in range(reps):
            run(False)
            ms.append(ctx.stats()["ms_total"])
        out[name] = {"digest": digest(res, tr), "stats": {k: int(st[k]) for k in INT_STATS},
                     "codes": [r["code"] for r in res], "iters": [r["iters"] for r in res],
                     "ms_total_median": statistics.median(ms), "ms_total_min": min(ms)}

    ctx = Context(0, 1, 100000, 100000)
    measure("cooperative: 2.6k/20k operating point", ctx, lambda t: ctx.run_batch([data["small"]], want_trace=t))
    ctx.close()
    for mode, name in ((1, "graph: three C2 pairs, resident"), (0, "host loop: three C2 pairs, resident")):
        ctx = Context(0, len(c2), n_c2, n_c2)
        ctx.set_tunable("use_graph", mode)
        ctx.upload(c2)
        measure(name, ctx, lambda t: ctx.run_resident(want_trace=t))
        ctx.close()
    ctx = Context(0, 1, n_c2, n_c2)
    q = c2[0]
    base, glob = [0] * len(q["src"]), [len(c) for c in q["src"]]

    def sharded(t):
        r, tr = ctx.run_sharded(q, base, glob, lambda *a: 0, want_trace=t)
        return [r], ([tr] if tr is not None else [])

    measure("sharded: one C2 pair, world 1", ctx, sharded)
    ctx.close()
    with open(out_path, "w") as f:
        json.dump(out, f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("parent_lib")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", nargs=2, metavar=("INPUTS", "OUT"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args.parent_lib, args.worker[0], args.reps, args.worker[1])
    sides = {"parent": os.path.abspath(args.parent_lib),
             "change": os.path.join(ROOT, "mulls_b200", "csrc", "libmulls_b200.so")}
    runs = {s: [] for s in sides}
    with tempfile.TemporaryDirectory() as tmp:
        inputs = os.path.join(tmp, "inputs.pkl")
        make_inputs(inputs)
        for rnd in range(args.rounds):
            order = list(sides) if rnd % 2 == 0 else list(sides)[::-1]
            for side in order:
                res = os.path.join(tmp, f"{side}_{rnd}.json")
                subprocess.check_call([sys.executable, os.path.abspath(__file__), sides[side], "--reps", str(args.reps),
                                       "--worker", inputs, res])
                with open(res) as f:
                    runs[side].append(json.load(f))
                print(side, rnd, json.dumps({k: (v["ms_total_median"], v["stats"]) for k, v in runs[side][-1].items()}),
                      flush=True)
    ok = True
    report = {"cases": {}}
    for case in runs["parent"][0]:
        ref = runs["parent"][0][case]
        same = all(r[case]["digest"] == ref["digest"] and r[case]["stats"] == ref["stats"] for s in runs for r in runs[s])
        ok = ok and same
        report["cases"][case] = {
            "equal_results_traces_int_stats": same, "stats": ref["stats"], "codes": ref["codes"], "iters": ref["iters"],
            "ms_total_median_per_round": {s: [round(r[case]["ms_total_median"], 4) for r in runs[s]] for s in runs},
        }
    report["all_equal"] = ok
    text = json.dumps(report, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
