"""GPU checks of mulls_omp_ndt (CRegistration::omp_ndt, DIRECT7) against the CPU restatement
(tests/harness/ndt_oracle.cpp): on every CPU case of tests/test_ndt.py and on demo scan pairs 000000/000001 and 000000/000015
(raw, and voxel-downsampled on the device at 0.5 m) the device equals the restatement bit for bit: code, iterations, convergence, every Trans1_2
bit, the fitness bits and the per-iteration trace. Also: the refusals (KDTREE, capacity, NULL), known motion recovered,
the drop-in member against the library, and a batch uploaded again after an NDT call registers as before it (the call
replaces the resident batch)."""
import os

import numpy as np
import pytest

from mulls_b200 import synth
from mulls_b200.registration import Context, CRegistration
from test_ncc import ROOT, _chain_mod
from test_ndt import bbox, cases, oracle_ndt, rot

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, 1, 200000, 200000)
    yield c
    c.close()


def device_ndt(ctx, case, trace_cap=64):
    return ctx.omp_ndt(case["tgt"], case["src"], case.get("tb", bbox(case["tgt"])), case.get("sb", bbox(case["src"])),
                       case.get("res", 1.0), True, case.get("guess"), case.get("filter", True), case.get("thre", 10.0),
                       trace_cap=trace_cap)


def assert_bit_equal(d, o):
    for k in ("code", "iterations", "converged", "n_target", "n_source"):
        assert d[k] == o[k], (k, d[k], o[k])
    assert np.array_equal(np.float64(d["fitness"]).view(np.uint64), np.float64(o["fitness"]).view(np.uint64)), (d["fitness"], o["fitness"])
    assert np.array_equal(d["trans"].view(np.uint64), o["trans"].view(np.uint64)), (d["trans"], o["trans"])
    assert np.array_equal(d["trace"]["reversed"], o["trace"]["reversed"])
    for k in ("p", "step", "score"):
        assert np.array_equal(d["trace"][k].view(np.uint64), o["trace"][k].view(np.uint64)), k


@pytest.mark.parametrize("name", list(cases()))
def test_device_equals_restatement(ctx, name):
    c = cases()[name]
    assert_bit_equal(device_ndt(ctx, c), oracle_ndt(c))


def demo_pairs():
    mod = _chain_mod()
    z = np.load(os.path.join(ROOT, "tests", "golden", "demo_chain.npz"))
    scans = [np.ascontiguousarray(mod.decode_scan(z[f"scan{k}_dmm"], z[f"scan{k}_i"])[:, :3], np.float32) for k in range(16)]
    return [(0, 1), (0, 15)], scans


@pytest.mark.parametrize("voxel", [None, 0.5])
def test_demo_pairs_equal_restatement(ctx, voxel):
    pairs, scans = demo_pairs()
    for a, b in pairs:
        t, s = scans[a], scans[b]
        if voxel:
            t = ctx.voxel_downsample(np.c_[t, np.zeros((len(t), 4), np.float32)], voxel)[:, :3].copy()
            s = ctx.voxel_downsample(np.c_[s, np.zeros((len(s), 4), np.float32)], voxel)[:, :3].copy()
        c = dict(tgt=t, src=s)
        d, o = device_ndt(ctx, c), oracle_ndt(c)
        assert_bit_equal(d, o)
        assert d["n_source"] > 1000 and d["iterations"] >= 1


def test_known_motion(ctx):
    """the source is the target scene moved by (R, t)^-1 with 2 cm noise: Trans1_2 is within 0.06 m and 0.06 rad of
    (R, t). The walk never steps shorter than 0.05 (mixed m / rad), so its end can sit up to that far past the optimum."""
    d = device_ndt(ctx, cases()["motion"])
    R, t = rot(0.01, -0.015, 0.03), np.array([0.15, -0.1, 0.05])
    T = d["trans"]
    assert d["code"] == 1
    assert np.linalg.norm(T[:3, 3] - t) < 0.06
    assert np.arccos(np.clip((np.trace(T[:3, :3].T @ R) - 1) / 2, -1, 1)) < 0.06


def test_refusals(ctx):
    c = cases()["motion"]
    with pytest.raises(RuntimeError, match="error -103:"):  # MULLS_E_UNSUPPORTED
        ctx.omp_ndt(c["tgt"], c["src"], bbox(c["tgt"]), bbox(c["src"]), use_direct_search=False)
    small = Context(0, 1, 1000, 1000)
    try:
        with pytest.raises(RuntimeError, match="error -102:"):  # MULLS_E_CAPACITY
            small.omp_ndt(c["tgt"], c["src"], bbox(c["tgt"]), bbox(c["src"]))
    finally:
        small.close()
    from mulls_b200 import abi
    import ctypes as C
    res = abi.NdtResult()
    g = np.eye(4).ravel().copy()
    dp = C.POINTER(C.c_double)
    # NULL result, NULL guess, NULL bounds: MULLS_E_ARG
    assert ctx.lib.mulls_omp_ndt(ctx.handle, abi.CloudView(), abi.CloudView(), 1.0, 1, g.ctypes.data_as(dp), 1, 10.0,
                                 g.ctypes.data_as(dp), g.ctypes.data_as(dp), None, None, 0) == -101
    assert ctx.lib.mulls_omp_ndt(ctx.handle, abi.CloudView(), abi.CloudView(), 1.0, 1, None, 1, 10.0, g.ctypes.data_as(dp),
                                 g.ctypes.data_as(dp), C.byref(res), None, 0) == -101
    assert ctx.lib.mulls_omp_ndt(ctx.handle, abi.CloudView(), abi.CloudView(), 1.0, 1, g.ctypes.data_as(dp), 1, 10.0, None,
                                 g.ctypes.data_as(dp), C.byref(res), None, 0) == -101


def test_registration_after_ndt_unchanged(ctx):
    """mulls_omp_ndt replaces the resident batch (its fitness search builds the target's grid through the ingest, as
    mulls_sor_filter does): a batch uploaded again after the call registers exactly as before it"""
    pair = synth.make_pair(1000, "small")
    r0, _ = ctx.run_batch([pair], want_trace=True)
    device_ndt(ctx, cases()["motion"])
    r1, _ = ctx.run_batch([pair], want_trace=True)
    assert r0[0]["code"] == r1[0]["code"] and r0[0]["iters"] == r1[0]["iters"]
    assert np.array_equal(np.asarray(r0[0]["T"]), np.asarray(r1[0]["T"]))


def test_dropin_on_device(ctx):
    """the drop-in member (tests/stubs/ndt_caller.cpp replaying mulls_slam.cpp:634-636) returns what the library does"""
    import subprocess
    import tempfile

    from test_ndt import build_ndt_caller, rows
    pairs, scans = demo_pairs()
    t, s = scans[0], scans[1]
    d = device_ndt(ctx, dict(tgt=t, src=s))
    with tempfile.TemporaryDirectory() as td:
        exe = build_ndt_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0 and "failures 0" in out.stdout and "ran on a device: 1" in out.stdout, out.stdout + out.stderr
        tp, sp, op = (os.path.join(td, f) for f in ("t.bin", "s.bin", "o.bin"))
        rows(t).tofile(tp)
        rows(s).tofile(sp)
        r = subprocess.run([exe, tp, sp, op, "1.0"], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        o = np.fromfile(op, np.float64)
    assert int(o[0]) == d["code"]
    assert np.array_equal(o[1:].reshape(4, 4), d["trans"])


def test_cregistration_wrapper(ctx):
    c = cases()["guess"]
    reg = CRegistration(0, 50000, 50000)
    code, T = reg.omp_ndt(c["tgt"], c["src"], bbox(c["tgt"]), bbox(c["src"]), initial_guess=c["guess"])
    o = oracle_ndt(c)
    assert code == o["code"] and np.array_equal(T, o["trans"])
