"""GPU checks of mulls_omp_gicp_pcl (CRegistration::omp_gicp with using_voxel_gicp=False, point-wise GICP with PCL's
BFGS) against the CPU restatement (tests/harness/gicp_pcl_oracle.cpp): on every case of tests/test_gicp.py::cases()
and on demo scan pairs 000000/000001 and 000000/000015 (raw, and voxel-downsampled on the device at 0.5 m) the device
equals the restatement bit for bit: code, iterations, convergence, point counts, every Trans1_2 bit, the fitness bits
and every trace row. Also: max_iter_num 1, 5 and 20 reach the solver, known motion recovered, the refusals, a batch
uploaded again after the call registers as before it, a destroyed context gives back the call's scratch, and the shim
caller returns what the library does."""
import ctypes as C
import os

import numpy as np
import pytest

from mulls_b200 import synth
from mulls_b200.registration import Context, CRegistration
from test_gicp import cases
from test_gicp_pcl import REFUSED, oracle_gicp_pcl
from test_gpu_ndt import demo_pairs
from test_ndt import bbox, rot

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, 1, 200000, 200000)
    yield c
    c.close()


def device_gicp_pcl(ctx, case, max_iter=20, trace_cap=256):
    return ctx.omp_gicp_pcl(case["tgt"], case["src"], case.get("tb", bbox(case["tgt"])), case.get("sb", bbox(case["src"])),
                            max_iter_num=max_iter, initial_guess=case.get("guess"),
                            apply_intersection_filter=case.get("filter", False), fitness_score_thre=case.get("thre", 10.0),
                            trace_cap=trace_cap)


def assert_bit_equal(d, o):
    assert o["rc"] == 0
    for k in ("code", "iterations", "converged", "n_target", "n_source"):
        assert d[k] == o[k], (k, d[k], o[k])
    assert np.array_equal(np.float64(d["fitness"]).view(np.uint64), np.float64(o["fitness"]).view(np.uint64)), (d["fitness"], o["fitness"])
    assert np.array_equal(d["trans"].view(np.uint64), o["trans"].view(np.uint64)), (d["trans"], o["trans"])
    for k in ("n_corr", "inner_iterations", "status", "evaluations"):
        assert np.array_equal(d["trace"][k], o["trace"][k]), k
    for k in ("x", "delta"):
        assert np.array_equal(d["trace"][k].view(np.uint64), o["trace"][k].view(np.uint64)), k


@pytest.mark.parametrize("name", list(cases()))
def test_device_equals_restatement(ctx, name):
    c = cases()[name]
    assert_bit_equal(device_gicp_pcl(ctx, c), oracle_gicp_pcl(c))


@pytest.mark.parametrize("voxel", [None, 0.5])
def test_demo_pairs_equal_restatement(ctx, voxel):
    pairs, scans = demo_pairs()
    for a, b in pairs:
        t, s = scans[a], scans[b]
        if voxel:
            t = ctx.voxel_downsample(np.c_[t, np.zeros((len(t), 4), np.float32)], voxel)[:, :3].copy()
            s = ctx.voxel_downsample(np.c_[s, np.zeros((len(s), 4), np.float32)], voxel)[:, :3].copy()
        c = dict(tgt=t, src=s)
        d, o = device_gicp_pcl(ctx, c), oracle_gicp_pcl(c)
        assert_bit_equal(d, o)
        assert d["n_source"] > 1000 and d["iterations"] >= 1


def test_max_iter_reaches_the_solver(ctx):
    c = cases()["motion"]
    r = {}
    for k in (1, 5, 20):
        r[k] = device_gicp_pcl(ctx, c, max_iter=k)
        assert_bit_equal(r[k], oracle_gicp_pcl(c, max_iter=k))
    assert (r[1]["trace"]["inner_iterations"] == 1).all() and (r[5]["trace"]["inner_iterations"] == 5).any()
    for a, b in ((1, 5), (5, 20), (1, 20)):
        assert not np.array_equal(r[a]["trans"], r[b]["trans"]), (a, b)


def test_known_motion(ctx):
    d = device_gicp_pcl(ctx, cases()["motion"])
    R, t = rot(0.01, -0.015, 0.03), np.array([0.15, -0.1, 0.05])
    T = d["trans"]
    assert d["code"] == 1 and d["converged"]
    assert np.linalg.norm(T[:3, 3] - t) < 0.03
    assert np.arccos(np.clip((np.trace(T[:3, :3].T @ R) - 1) / 2, -1, 1)) < 0.01


def test_refusals(ctx):
    c = cases()["motion"]
    for name, mk in REFUSED.items():
        k = mk(c)
        with pytest.raises(RuntimeError, match="error -103:"):  # MULLS_E_UNSUPPORTED
            ctx.omp_gicp_pcl(k["tgt"], k["src"], bbox(k["tgt"]), bbox(k["src"]), apply_intersection_filter=k.get("filter", False))
    small = Context(0, 1, 1000, 1000)
    try:
        with pytest.raises(RuntimeError, match="error -102:"):  # MULLS_E_CAPACITY
            small.omp_gicp_pcl(c["tgt"], c["src"], bbox(c["tgt"]), bbox(c["src"]))
    finally:
        small.close()
    from mulls_b200 import abi
    res = abi.GicpPclResult()
    g = np.eye(4).ravel().copy()
    dp = C.POINTER(C.c_double)
    f = ctx.lib.mulls_omp_gicp_pcl
    assert f(ctx.handle, abi.CloudView(), abi.CloudView(), 20, g.ctypes.data_as(dp), 0, 10.0, g.ctypes.data_as(dp),
             g.ctypes.data_as(dp), None, None, 0) == -101
    assert f(ctx.handle, abi.CloudView(), abi.CloudView(), 20, g.ctypes.data_as(dp), 0, 10.0, g.ctypes.data_as(dp),
             g.ctypes.data_as(dp), C.byref(res), None, 4) == -101  # a trace capacity without a trace


def test_registration_after_gicp_pcl_unchanged(ctx):
    pair = synth.make_pair(1000, "small")
    r0, _ = ctx.run_batch([pair], want_trace=True)
    device_gicp_pcl(ctx, cases()["motion"])
    r1, _ = ctx.run_batch([pair], want_trace=True)
    assert r0[0]["code"] == r1[0]["code"] and r0[0]["iters"] == r1[0]["iters"]
    assert np.array_equal(np.asarray(r0[0]["T"]), np.asarray(r1[0]["T"]))


def test_shim_on_device(ctx):
    """lo::b200::omp_gicp_pcl (tests/stubs/gicp_pcl_caller.cpp replaying mulls_slam.cpp:637-639 with
    --voxel_gicp_on=false) returns what the library does"""
    import subprocess
    import tempfile

    from test_gicp_pcl import build_gicp_pcl_caller
    from test_ndt import rows
    pairs, scans = demo_pairs()
    t, s = scans[0], scans[1]
    with tempfile.TemporaryDirectory() as td:
        exe = build_gicp_pcl_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0 and "failures 0" in out.stdout and "ran on a device: 1" in out.stdout, out.stdout + out.stderr
        tp, sp, op = (os.path.join(td, f) for f in ("t.bin", "s.bin", "o.bin"))
        rows(t).tofile(tp)
        rows(s).tofile(sp)
        r = subprocess.run([exe, tp, sp, op, "15"], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        o = np.fromfile(op, np.float64)
    d = device_gicp_pcl(ctx, dict(tgt=t, src=s, filter=True), max_iter=15)
    assert int(o[0]) == d["code"]
    assert np.array_equal(o[1:].reshape(4, 4), d["trans"])


def test_cregistration_wrapper(ctx):
    c = cases()["guess"]
    reg = CRegistration(0, 50000, 50000)
    code, T = reg.omp_gicp_pcl(c["tgt"], c["src"], bbox(c["tgt"]), bbox(c["src"]), initial_guess=c["guess"])
    o = oracle_gicp_pcl(c)
    assert code == o["code"] and np.array_equal(T, o["trans"])


def test_context_memory_released():
    """a destroyed context gives back the scratch omp_gicp_pcl grew: four rounds of create, one call on a 200 000-point
    target, close leave the device's free memory where it was"""
    import torch

    from test_ndt import structured_scene
    tgt = structured_scene(200000, 5)
    src = tgt[::4].copy()

    def once():
        c = Context(0, 1, 250000, 250000)
        try:
            c.omp_gicp_pcl(tgt, src, bbox(tgt), bbox(src), max_iter_num=2)
        finally:
            c.close()

    once()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    for _ in range(4):
        once()
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info(0)[0]
    assert free0 - free1 < (32 << 20), (free0 - free1) / 2**20
