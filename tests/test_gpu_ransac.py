"""GPU checks of mulls_coarse_reg_ransac (CRegistration::coarse_reg_ransac, cregistration.hpp:604-661): status,
tran_mat bits, inlier count and hypothesis count of the CPU restatement (tests/harness/ransac_oracle.cpp) on every
correspondence set of tests/test_ransac.py (the two oscillating refinements included), on the real chain (vertex clouds
of demo scans 000000 / 000001 and 000000 / 000015 -> device NCC matching -> RANSAC), at
4 000 correspondences with every one of 20 001 hypotheses scored; refusals; the resident batch it leaves alone; and the
C++ drop-in on the device."""
import ctypes as C
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

from mulls_b200 import abi, synth
from mulls_b200.registration import Context, CRegistration
from test_ncc import ROOT, _chain_mod, real_vertex_clouds
from test_ransac import CASES, build_caller, oracle_ransac, scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, 1, 4096, 20000)
    yield c
    c.close()


def assert_equal_oracle(ctx, t, s, **kw):
    exp = oracle_ransac(t, s, **kw)
    status, T, n_inl, n_hyp = ctx.coarse_reg_ransac(t, s, tran_mat=np.full((4, 4), 7.0), **kw)
    assert (status, n_inl, n_hyp) == (exp["status"], exp["n_inliers"], exp["n_hyp"])
    assert np.array_equal(T.view(np.uint64), exp["T"].view(np.uint64)), (T, exp["T"])
    return status, n_hyp


@pytest.mark.parametrize("name,target,source,kw", CASES, ids=[c[0] for c in CASES])
def test_cases_equal_oracle(ctx, name, target, source, kw):
    assert_equal_oracle(ctx, target, source, **kw)


@functools.lru_cache(maxsize=None)
def vertex_clouds(a, b):
    """pc_vertex of demo scans a and b through the oracle's front end (0 / 1: consecutive scans, 0 / 15: the pair
    test/mulls_reg.cpp registers in the demo run)"""
    if (a, b) == (0, 1):
        return real_vertex_clouds()
    mod = _chain_mod()
    z = np.load(os.path.join(ROOT, "tests", "golden", "demo_chain.npz"))
    gp, cp = mod.chain_params()
    out = []
    for k in (a, b):
        raw = mod.decode_scan(z[f"scan{k}_dmm"], z[f"scan{k}_i"])
        out.append(np.ascontiguousarray(mod.oracle_features(raw, gp, cp)["vertex"], np.float32))
    return out[0], out[1]


@pytest.mark.parametrize("scans", [(0, 1), (0, 15)], ids=["000000_000001", "000000_000015"])
@pytest.mark.parametrize("corr_num", [1000, 4000])
def test_real_chain_equals_oracle(ctx, scans, corr_num):
    t, s = vertex_clouds(*scans)
    ti, si = ctx.ncc_correspondences(t, s, True, corr_num, True)
    assert len(ti) > 100
    assert_equal_oracle(ctx, t[ti], s[si])


def test_every_hypothesis_scored_at_4000():
    c = Context(0, 1, 4096, 20000)
    try:
        t, s, _ = scene(4000, 0.02, 21)
        _, n_hyp = assert_equal_oracle(c, t, s, max_iter_num=20000)
        assert n_hyp == 20001
    finally:
        c.close()


def test_20000_correspondences(ctx):
    t, s, _ = scene(20000, 0.1, 12)
    assert assert_equal_oracle(ctx, t, s)[0] == 1


def test_refusals_then_the_context_still_works():
    c = Context(0, 1, 1000, 1000)
    try:
        t, s, _ = scene(300, 0.5, 2)
        with pytest.raises(RuntimeError, match="-102"):
            c.coarse_reg_ransac(np.concatenate([t] * 4), np.concatenate([s] * 4))
        with pytest.raises(RuntimeError, match="-101"):
            c.coarse_reg_ransac(t, s[:299])
        lib = abi.load_library()
        T = np.full(16, 7.0)
        st, ni, nh = C.c_int(5), C.c_int(5), C.c_int(5)
        tv, sv = abi.cloud_view(abi.as_aos48(t)), abi.cloud_view(abi.as_aos48(s))
        dp = C.POINTER(C.c_double)
        assert lib.mulls_coarse_reg_ransac(c.handle, tv, sv, 0.2, 8, 20000, None, C.byref(st), C.byref(ni), C.byref(nh)) == abi.E_ARG
        for args in ((None, C.byref(ni), C.byref(nh)), (C.byref(st), None, C.byref(nh)), (C.byref(st), C.byref(ni), None)):
            assert lib.mulls_coarse_reg_ransac(c.handle, tv, sv, 0.2, 8, 20000, T.ctypes.data_as(dp), *args) == abi.E_ARG
        assert np.all(T == 7.0) and st.value == 5
        assert_equal_oracle(c, t, s)
    finally:
        c.close()


def test_resident_batch_is_left_alone():
    pair = synth.make_pair(1000, "small")
    t, s, _ = scene(700, 0.3, 5)
    c = Context(0, 1, 100000, 100000)
    try:
        c.upload([pair])
        r0, _ = c.run_resident()
        assert_equal_oracle(c, t, s)
        r1, _ = c.run_resident()  # no re-upload: the batch and its grid are still there
        assert np.array_equal(r0[0]["T"], r1[0]["T"]) and r0[0]["code"] == r1[0]["code"] and r0[0]["iters"] == r1[0]["iters"]
    finally:
        c.close()


@pytest.mark.parametrize("case", ["known_50pct", "n2", "noise_bound_zero"])
def test_dropin_on_the_device_returns_the_oracle_matrix(case):
    name, t, s, kw = next(c for c in CASES if c[0] == case)
    kw = dict(dict(noise_bound=0.2, min_inlier_num=8, max_iter_num=20000), **kw)
    marker = (100.0 + np.arange(16)).reshape(4, 4)
    exp = oracle_ransac(t, s, tran=marker, **kw)
    with tempfile.TemporaryDirectory() as td:
        exe = build_caller(td)
        paths = [os.path.join(td, f) for f in ("t.bin", "s.bin", "out.bin")]
        np.ascontiguousarray(t, np.float32).tofile(paths[0])
        np.ascontiguousarray(s, np.float32).tofile(paths[1])
        out = subprocess.run([exe] + paths + [repr(float(kw["noise_bound"])), str(kw["min_inlier_num"]), str(kw["max_iter_num"])],
                             capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stdout + out.stderr
        got = np.fromfile(paths[2], np.float64)
        base = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert int(got[0]) == exp["status"]
    assert np.array_equal(got[1:].reshape(4, 4).view(np.uint64), exp["T"].view(np.uint64))  # the marker on -1
    assert base.returncode == 0 and "ran on a device: 1" in base.stdout and "failures 0" in base.stdout, base.stdout


def test_python_mirror_keeps_tran_mat_on_failure():
    t, s, _ = scene(300, 0.5, 2)
    reg = CRegistration(0, 1000, 1000)
    guess = np.arange(16.0).reshape(4, 4)
    status, T = reg.coarse_reg_ransac(t[:5], s[:5], guess)
    assert status == -1 and np.array_equal(T, guess)
    status, T = reg.coarse_reg_ransac(t, s, guess)
    exp = oracle_ransac(t, s)
    assert status == exp["status"] == 1 and np.array_equal(T, exp["T"])
