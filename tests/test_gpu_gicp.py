"""GPU checks of mulls_omp_gicp (CRegistration::omp_gicp, FastVGICP) against the CPU restatement
(tests/harness/gicp_oracle.cpp): on every CPU case of tests/test_gicp.py and on demo scan pairs 000000/000001 and
000000/000015 (raw, and voxel-downsampled on the device at 0.5 m, with voxel_size 1.0 and 0.5), seeded identically, the
device equals the restatement bit for bit: code, iterations, convergence, every Trans1_2 bit, the fitness bits, x0, the
per-iteration trace and the rand() state afterwards. Also: the refusals, known motion recovered, the ignored arguments,
the drop-in member against the library, a batch uploaded again after a GICP call registers as before it, and a
destroyed context gives back the scratch its GICP and NDT calls grew."""
import os

import numpy as np
import pytest

from mulls_b200 import synth
from mulls_b200.registration import Context, CRegistration
from test_gicp import LIBC, REFUSED, cases, draws_until, oracle_gicp
from test_gpu_ndt import demo_pairs
from test_ndt import bbox, rot

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, 1, 200000, 200000)
    yield c
    c.close()


def device_gicp(ctx, case, trace_cap=64, seed=1234, **kw):
    LIBC.srand(seed)
    d = ctx.omp_gicp(case["tgt"], case["src"], case.get("tb", bbox(case["tgt"])), case.get("sb", bbox(case["src"])),
                     using_voxel_gicp=True, voxel_size=case.get("res", 1.0), initial_guess=case.get("guess"),
                     apply_intersection_filter=case.get("filter", False), fitness_score_thre=case.get("thre", 10.0),
                     trace_cap=trace_cap, **kw)
    d["next_rand"] = LIBC.rand()
    d["draws"] = draws_until(seed, d["next_rand"])
    return d


def assert_bit_equal(d, o):
    assert o["rc"] == 0
    for k in ("code", "iterations", "converged", "n_target", "n_source", "next_rand", "draws"):
        assert d[k] == o[k], (k, d[k], o[k])
    assert np.array_equal(np.float64(d["fitness"]).view(np.uint64), np.float64(o["fitness"]).view(np.uint64)), (d["fitness"], o["fitness"])
    assert np.array_equal(d["trans"].view(np.uint64), o["trans"].view(np.uint64)), (d["trans"], o["trans"])
    assert np.array_equal(d["x0"].view(np.uint32), o["x0"].view(np.uint32))
    for k in ("n_corr", "random_step"):
        assert np.array_equal(d["trace"][k], o["trace"][k]), k
    for k in ("x", "delta"):
        assert np.array_equal(d["trace"][k].view(np.uint32), o["trace"][k].view(np.uint32)), k


@pytest.mark.parametrize("name", list(cases()))
def test_device_equals_restatement(ctx, name):
    c = cases()[name]
    assert_bit_equal(device_gicp(ctx, c), oracle_gicp(c))


@pytest.mark.parametrize("voxel", [None, 0.5])
@pytest.mark.parametrize("res", [1.0, 0.5])
def test_demo_pairs_equal_restatement(ctx, voxel, res):
    pairs, scans = demo_pairs()
    for a, b in pairs:
        t, s = scans[a], scans[b]
        if voxel:
            t = ctx.voxel_downsample(np.c_[t, np.zeros((len(t), 4), np.float32)], voxel)[:, :3].copy()
            s = ctx.voxel_downsample(np.c_[s, np.zeros((len(s), 4), np.float32)], voxel)[:, :3].copy()
        c = dict(tgt=t, src=s, res=res)
        d, o = device_gicp(ctx, c), oracle_gicp(c)
        assert_bit_equal(d, o)
        assert d["n_source"] > 1000 and d["iterations"] >= 1


def test_known_motion(ctx):
    d = device_gicp(ctx, cases()["motion"])
    R, t = rot(0.01, -0.015, 0.03), np.array([0.15, -0.1, 0.05])
    T = d["trans"]
    assert d["code"] == 1 and d["converged"]
    assert np.linalg.norm(T[:3, 3] - t) < 0.03
    assert np.arccos(np.clip((np.trace(T[:3, :3].T @ R) - 1) / 2, -1, 1)) < 0.01


def test_ignored_arguments(ctx):
    c = cases()["motion"]
    a = device_gicp(ctx, c)
    b = device_gicp(ctx, c, max_iter_num=1, dis_thre_unit=0.01)
    assert np.array_equal(a["trans"], b["trans"]) and a["iterations"] == b["iterations"]


def test_refusals(ctx):
    c = cases()["motion"]
    for name, mk in REFUSED.items():
        k = mk(c)
        LIBC.srand(7)
        with pytest.raises(RuntimeError, match="error -103:"):  # MULLS_E_UNSUPPORTED
            ctx.omp_gicp(k["tgt"], k["src"], bbox(k["tgt"]), bbox(k["src"]), voxel_size=k.get("res", 1.0),
                         apply_intersection_filter=k.get("filter", False))
        assert draws_until(7, LIBC.rand()) == 0, name  # a refused call draws nothing
    with pytest.raises(RuntimeError, match="error -103:"):
        ctx.omp_gicp(c["tgt"], c["src"], bbox(c["tgt"]), bbox(c["src"]), using_voxel_gicp=False)
    small = Context(0, 1, 1000, 1000)
    try:
        with pytest.raises(RuntimeError, match="error -102:"):  # MULLS_E_CAPACITY
            small.omp_gicp(c["tgt"], c["src"], bbox(c["tgt"]), bbox(c["src"]))
    finally:
        small.close()
    from mulls_b200 import abi
    import ctypes as C
    res = abi.GicpResult()
    g = np.eye(4).ravel().copy()
    dp = C.POINTER(C.c_double)
    assert ctx.lib.mulls_omp_gicp(ctx.handle, abi.CloudView(), abi.CloudView(), 1, 1.0, g.ctypes.data_as(dp), 0, 10.0,
                                  g.ctypes.data_as(dp), g.ctypes.data_as(dp), None, None, 0) == -101
    assert ctx.lib.mulls_omp_gicp(ctx.handle, abi.CloudView(), abi.CloudView(), 1, 0.0, g.ctypes.data_as(dp), 0, 10.0,
                                  g.ctypes.data_as(dp), g.ctypes.data_as(dp), C.byref(res), None, 0) == -101


def test_registration_after_gicp_unchanged(ctx):
    pair = synth.make_pair(1000, "small")
    r0, _ = ctx.run_batch([pair], want_trace=True)
    device_gicp(ctx, cases()["motion"])
    r1, _ = ctx.run_batch([pair], want_trace=True)
    assert r0[0]["code"] == r1[0]["code"] and r0[0]["iters"] == r1[0]["iters"]
    assert np.array_equal(np.asarray(r0[0]["T"]), np.asarray(r1[0]["T"]))


def test_dropin_on_device(ctx):
    """the drop-in member (tests/stubs/gicp_caller.cpp replaying mulls_slam.cpp:637-639) returns what the library does"""
    import subprocess
    import tempfile

    from test_gicp import build_gicp_caller
    from test_ndt import rows
    pairs, scans = demo_pairs()
    t, s = scans[0], scans[1]
    with tempfile.TemporaryDirectory() as td:
        exe = build_gicp_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0 and "failures 0" in out.stdout and "ran on a device: 1" in out.stdout, out.stdout + out.stderr
        tp, sp, op = (os.path.join(td, f) for f in ("t.bin", "s.bin", "o.bin"))
        rows(t).tofile(tp)
        rows(s).tofile(sp)
        r = subprocess.run([exe, tp, sp, op, "1.0"], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        o = np.fromfile(op, np.float64)
    # the caller's process starts from rand()'s default seed (1); the filter is on at the call site
    d = device_gicp(ctx, dict(tgt=t, src=s, filter=True), seed=1)
    assert int(o[0]) == d["code"]
    assert np.array_equal(o[1:].reshape(4, 4), d["trans"])


def test_cregistration_wrapper(ctx):
    c = cases()["guess"]
    reg = CRegistration(0, 50000, 50000)
    LIBC.srand(1234)
    code, T = reg.omp_gicp(c["tgt"], c["src"], bbox(c["tgt"]), bbox(c["src"]), initial_guess=c["guess"])
    o = oracle_gicp(c)
    assert code == o["code"] and np.array_equal(T, o["trans"])


def test_context_memory_released():
    """mulls_destroy frees the scratch omp_gicp and omp_ndt grow: creating a context, running both calls on a
    200 000-point target and closing it, four times, leaves the device's free memory where it was (each round grows
    about 50 MB of scratch, which a leak would lose for the rest of the process)"""
    import torch

    from test_ndt import structured_scene
    tgt = structured_scene(200000, 5)
    src = tgt[::4].copy()

    def once():
        c = Context(0, 1, 250000, 250000)
        try:
            LIBC.srand(1)
            c.omp_gicp(tgt, src, bbox(tgt), bbox(src))
            c.omp_ndt(tgt, src, bbox(tgt), bbox(src))
        finally:
            c.close()

    once()  # module loading and the runtime's own first allocations
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    for _ in range(4):
        once()
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info(0)[0]
    assert free0 - free1 < (32 << 20), (free0 - free1) / 2**20
