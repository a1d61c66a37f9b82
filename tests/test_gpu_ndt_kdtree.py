"""GPU checks of mulls_omp_ndt_kdtree (omp_ndt with the KDTREE neighbourhood) against the CPU restatement
(tests/harness/ndt_kdtree_oracle.cpp): on every scene of tests/test_ndt_kdtree.py and on demo scan pairs 000000/000001 and
000000/000015 (raw, and voxel-downsampled on the device at 0.2 and 0.5 m) the device equals the restatement bit for bit:
code, iterations, convergence, n_target / n_source, every Trans1_2 bit, the fitness bits and every trace row. Also:
known motion recovered, the refusals, a batch registered after the call and b200::omp_ndt_kdtree against the library.
The dense_cube scene has lists longer than the 8 entries a call starts with, so it also covers their growth."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from mulls_b200 import abi, synth
from mulls_b200.registration import Context, CRegistration
from test_gpu_ndt import assert_bit_equal, demo_pairs
from test_ndt import bbox, cases, rot, rows
from test_ndt_kdtree import build_kdtree_caller, kd_case, kd_cases, oracle_kd

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, 1, 200000, 200000)
    yield c
    c.close()


def device_kd(ctx, case, trace_cap=64):
    return ctx.omp_ndt_kdtree(case["tgt"], case["src"], case.get("tb", bbox(case["tgt"])), case.get("sb", bbox(case["src"])),
                              case.get("res", 1.0), case.get("guess"), case.get("filter", True), case.get("thre", 10.0),
                              trace_cap=trace_cap)


@pytest.mark.parametrize("name", sorted(kd_cases()))
def test_device_equals_restatement(ctx, name):
    c = kd_case(name)
    assert_bit_equal(device_kd(ctx, c), oracle_kd(c))


@pytest.mark.parametrize("voxel", [None, 0.2, 0.5])
def test_demo_pairs_equal_restatement(ctx, voxel):
    pairs, scans = demo_pairs()
    for a, b in pairs:
        t, s = scans[a], scans[b]
        if voxel:
            t = ctx.voxel_downsample(np.c_[t, np.zeros((len(t), 4), np.float32)], voxel)[:, :3].copy()
            s = ctx.voxel_downsample(np.c_[s, np.zeros((len(s), 4), np.float32)], voxel)[:, :3].copy()
        c = dict(tgt=t, src=s)
        d, o = device_kd(ctx, c), oracle_kd(c)
        assert_bit_equal(d, o)
        assert d["n_source"] > 1000 and d["iterations"] >= 1


def test_known_motion(ctx):
    d = device_kd(ctx, cases()["motion"])
    R, t = rot(0.01, -0.015, 0.03), np.array([0.15, -0.1, 0.05])
    T = d["trans"]
    assert d["code"] == 1
    assert np.linalg.norm(T[:3, 3] - t) < 0.06
    assert np.arccos(np.clip((np.trace(T[:3, :3].T @ R) - 1) / 2, -1, 1)) < 0.06


def test_refusals(ctx):
    c = cases()["motion"]
    small = Context(0, 1, 1000, 1000)
    try:
        with pytest.raises(RuntimeError, match="error -102:"):  # MULLS_E_CAPACITY
            small.omp_ndt_kdtree(c["tgt"], c["src"], bbox(c["tgt"]), bbox(c["src"]))
    finally:
        small.close()
    with pytest.raises(RuntimeError, match="error -101:"):  # resolution <= 0: MULLS_E_ARG
        ctx.omp_ndt_kdtree(c["tgt"], c["src"], bbox(c["tgt"]), bbox(c["src"]), ndt_resolution=0.0)
    res = abi.NdtResult()
    g = np.eye(4).ravel().copy()
    dp = C.POINTER(C.c_double)
    f = ctx.lib.mulls_omp_ndt_kdtree
    assert f(ctx.handle, abi.CloudView(), abi.CloudView(), 1.0, g.ctypes.data_as(dp), 1, 10.0, g.ctypes.data_as(dp),
             g.ctypes.data_as(dp), None, None, 0) == -101
    assert f(ctx.handle, abi.CloudView(), abi.CloudView(), 1.0, None, 1, 10.0, g.ctypes.data_as(dp), g.ctypes.data_as(dp),
             C.byref(res), None, 0) == -101
    assert f(ctx.handle, abi.CloudView(), abi.CloudView(), -1.0, g.ctypes.data_as(dp), 1, 10.0, g.ctypes.data_as(dp),
             g.ctypes.data_as(dp), C.byref(res), None, 0) == -101
    # mulls_omp_ndt itself still refuses KDTREE
    with pytest.raises(RuntimeError, match="error -103:"):
        ctx.omp_ndt(c["tgt"], c["src"], bbox(c["tgt"]), bbox(c["src"]), use_direct_search=False)


def test_registration_after_kdtree_unchanged(ctx):
    """the call replaces the resident batch as mulls_omp_ndt does: a batch uploaded again registers exactly as before"""
    pair = synth.make_pair(1000, "small")
    r0, _ = ctx.run_batch([pair], want_trace=True)
    device_kd(ctx, cases()["motion"])
    r1, _ = ctx.run_batch([pair], want_trace=True)
    assert r0[0]["code"] == r1[0]["code"] and r0[0]["iters"] == r1[0]["iters"]
    assert np.array_equal(np.asarray(r0[0]["T"]), np.asarray(r1[0]["T"]))


def test_helper_on_device(ctx):
    """b200::omp_ndt_kdtree (tests/stubs/ndt_kdtree_caller.cpp replaying mulls_slam.cpp:634-636 with
    --ndt_searching_method=false) returns what the library does"""
    pairs, scans = demo_pairs()
    t, s = scans[0], scans[1]
    d = device_kd(ctx, dict(tgt=t, src=s))
    with tempfile.TemporaryDirectory() as td:
        exe = build_kdtree_caller(td)
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
    code, T = reg.omp_ndt_kdtree(c["tgt"], c["src"], bbox(c["tgt"]), bbox(c["src"]), initial_guess=c["guess"])
    o = oracle_kd(c)
    assert code == o["code"] and np.array_equal(T, o["trans"])
