"""GPU checks of mulls_ncc_correspondences (CRegistration::find_feature_correspondence_ncc, cregistration.hpp:409-601):
the index pairs of the CPU restatement (tests/harness/ncc_oracle.cpp), in order, on the adversarial and real keypoint
clouds of tests/test_ncc.py in every mode and at the sizes the drivers run; the fixed-number mode at the INT_MAX pair
bound against a closed form; refusals; the resident batch it leaves alone; and the C++ drop-in on the device."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from mulls_b200 import abi, synth
from mulls_b200.registration import Context, CRegistration
from test_ncc import CLOUDS, MODES, assert_same_pairs, build_ncc_caller, kpts, oracle_ncc, real_vertex_clouds

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, 1, 4096, 46341)
    yield c
    c.close()


@pytest.mark.parametrize("mode,fixed,corr,recip", MODES, ids=[m[0] for m in MODES])
@pytest.mark.parametrize("name,target,source", CLOUDS, ids=[c[0] for c in CLOUDS])
def test_adversarial_clouds_equal_oracle(ctx, name, target, source, mode, fixed, corr, recip):
    assert_same_pairs(ctx.ncc_correspondences(target, source, fixed, corr, recip), oracle_ncc(target, source, fixed, corr, recip))


@pytest.mark.parametrize("mode,fixed,corr,recip", MODES + [("fixed4000", True, 4000, False)], ids=[m[0] for m in MODES] + ["fixed4000"])
def test_real_vertex_clouds_equal_oracle(ctx, mode, fixed, corr, recip):
    t, s = real_vertex_clouds()
    got = ctx.ncc_correspondences(t, s, fixed, corr, recip)
    assert len(got[0]) > 0
    assert_same_pairs(got, oracle_ncc(t, s, fixed, corr, recip))


@pytest.mark.parametrize("corr_num", [-1, 0, 1, "M", "M+1"])
@pytest.mark.parametrize("name", ["random", "all_equal", "no_finite_distance", "integer_only"])
def test_fixed_corr_num_edges(ctx, name, corr_num):
    t, s = dict((c[0], (c[1], c[2])) for c in CLOUDS)[name]
    M = len(t) * len(s)
    k = {"M": M, "M+1": M + 1}.get(corr_num, corr_num)
    assert_same_pairs(ctx.ncc_correspondences(t, s, True, k, False), oracle_ncc(t, s, True, k, False))


@pytest.mark.parametrize("corr_num", [1000, 3000, 4000])
def test_fixed_4000_squared(ctx, corr_num):
    rng = np.random.default_rng(corr_num)
    t, s = kpts(4000, rng), kpts(4000, rng)
    assert_same_pairs(ctx.ncc_correspondences(t, s, True, corr_num, True), oracle_ncc(t, s, True, corr_num, True))


@pytest.mark.parametrize("recip", [False, True], ids=["plain", "reciprocal"])
def test_20000_squared(ctx, recip):
    rng = np.random.default_rng(20 + recip)
    t, s = kpts(20000, rng), kpts(20000, rng)
    got = ctx.ncc_correspondences(t, s, False, 2000, recip)
    assert_same_pairs(got, oracle_ncc(t, s, False, 2000, recip))
    assert len(got[0]) == 20000 or recip


def int_max_cloud(n):
    """target data[3] = i, source data[3] = j + 0.5, everything else equal but target row 0's intensity (0; every other
    intensity is 1): d(i, j) = |30 i - 30 j - 15| for i >= 1, 255 more for i = 0. The smallest distance, 15, is taken by
    (i, i - 1) and (i, i), i >= 1, in pair-index order"""
    t = np.zeros((n, 12), np.float32)
    s = np.zeros((n, 12), np.float32)
    t[:, 3] = np.arange(n)
    s[:, 3] = np.arange(n) + 0.5
    t[:, 8], s[:, 8] = 1.0, 1.0
    t[0, 8] = 0.0
    return t, s


def test_fixed_mode_at_the_int_max_bound(ctx):
    n = 46340  # n^2 = 2 147 395 600 <= INT_MAX
    t, s = int_max_cloud(n)
    got = ctx.ncc_correspondences(t, s, True, 1000, False)
    k = np.arange(1000)
    i = 1 + k // 2
    assert np.array_equal(got[0], i) and np.array_equal(got[1], i - 1 + k % 2)
    t, s = int_max_cloud(n + 1)  # 2 147 488 281 > INT_MAX
    with pytest.raises(RuntimeError, match="-101"):
        ctx.ncc_correspondences(t, s, True, 1000, False)
    got = ctx.ncc_correspondences(t, s, False, 2000, False)  # the other modes have no such bound
    assert np.array_equal(got[0], np.arange(n + 1)) and got[1][1] == 0 and got[1][0] == 0
    small = CLOUDS[0]
    assert_same_pairs(ctx.ncc_correspondences(small[1], small[2], True, 1000, False), oracle_ncc(small[1], small[2], True, 1000, False))


def test_too_few_keypoints_is_not_performed(ctx):
    rng = np.random.default_rng(4)
    assert ctx.ncc_correspondences(kpts(9, rng), kpts(500, rng)) is None
    assert ctx.ncc_correspondences(kpts(500, rng), kpts(9, rng), True, 100) is None
    ok, tc, sc = CRegistration(0, 1000, 1000).find_feature_correspondence_ncc(kpts(9, rng), kpts(50, rng), kpts(3, rng), kpts(3, rng))
    assert not ok and len(tc) == 3 and len(sc) == 3


def test_refusals_then_the_context_still_works():
    c = Context(0, 1, 1000, 1000)
    try:
        rng = np.random.default_rng(2)
        t, s = kpts(300, rng), kpts(200, rng)
        with pytest.raises(RuntimeError, match="-102"):
            c.ncc_correspondences(kpts(1001, rng), s)
        with pytest.raises(RuntimeError, match="-102"):
            c.ncc_correspondences(t, kpts(1001, rng), True, 10)
        lib = abi.load_library()
        ti, si = np.zeros(300, np.int32), np.zeros(300, np.int32)
        n, done = C.c_size_t(0), C.c_int(0)
        ip = C.POINTER(C.c_int32)
        tv, sv = abi.cloud_view(abi.as_aos48(t)), abi.cloud_view(abi.as_aos48(s))
        exp = oracle_ncc(t, s, False, 2000, False)
        rc = lib.mulls_ncc_correspondences(c.handle, tv, sv, 0, 2000, 0, ti.ctypes.data_as(ip), si.ctypes.data_as(ip),
                                           len(exp[0]) - 1, C.byref(n), C.byref(done))
        assert rc == abi.E_ARG and n.value == 0 and done.value == 0  # one short of the result
        rc = lib.mulls_ncc_correspondences(c.handle, tv, sv, 0, 2000, 0, None, None, 0, C.byref(n), C.byref(done))
        assert rc == abi.E_ARG
        rc = lib.mulls_ncc_correspondences(c.handle, tv, sv, 0, 2000, 0, ti.ctypes.data_as(ip), si.ctypes.data_as(ip), 300, None,
                                           C.byref(done))
        assert rc == abi.E_ARG
        rc = lib.mulls_ncc_correspondences(c.handle, tv, sv, 0, 2000, 0, ti.ctypes.data_as(ip), si.ctypes.data_as(ip),
                                           len(exp[0]), C.byref(n), C.byref(done))
        assert rc == 0 and done.value == 1 and n.value == len(exp[0])
        assert np.array_equal(ti[: n.value], exp[0]) and np.array_equal(si[: n.value], exp[1])
        for fixed, corr, recip in ((True, 500, False), (False, 2000, True)):
            assert_same_pairs(c.ncc_correspondences(t, s, fixed, corr, recip), oracle_ncc(t, s, fixed, corr, recip))
    finally:
        c.close()


def test_resident_batch_is_left_alone():
    pair = synth.make_pair(1000, "small")
    rng = np.random.default_rng(5)
    t, s = kpts(700, rng), kpts(650, rng)
    c = Context(0, 1, 100000, 100000)
    try:
        c.upload([pair])
        r0, _ = c.run_resident()
        for fixed, corr, recip in ((False, 2000, False), (False, 2000, True), (True, 1000, False)):
            assert_same_pairs(c.ncc_correspondences(t, s, fixed, corr, recip), oracle_ncc(t, s, fixed, corr, recip))
        r1, _ = c.run_resident()  # no re-upload: the batch and its grid are still there
        assert np.array_equal(r0[0]["T"], r1[0]["T"]) and r0[0]["code"] == r1[0]["code"] and r0[0]["iters"] == r1[0]["iters"]
    finally:
        c.close()


@pytest.mark.parametrize("fixed,corr,recip", [(False, 1000, False), (True, 1000, True), (True, 4000, False), (False, 2000, True)])
def test_dropin_on_the_device_appends_the_oracle_rows(fixed, corr, recip):
    t, s = real_vertex_clouds()
    ti, si = oracle_ncc(t, s, fixed, corr, recip)
    with tempfile.TemporaryDirectory() as td:
        exe = build_ncc_caller(td)
        paths = [os.path.join(td, f) for f in ("t.bin", "s.bin", "tc.bin", "sc.bin")]
        t.tofile(paths[0])
        s.tofile(paths[1])
        out = subprocess.run([exe] + paths + [str(int(fixed)), str(corr), str(int(recip))], capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stdout + out.stderr
        got_t = np.fromfile(paths[2], np.float32).reshape(-1, 12)
        got_s = np.fromfile(paths[3], np.float32).reshape(-1, 12)
        base = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert np.array_equal(got_t.view(np.uint32), t[ti].view(np.uint32))
    assert np.array_equal(got_s.view(np.uint32), s[si].view(np.uint32))
    assert base.returncode == 0 and "ran on a device: 1" in base.stdout and "failures 0" in base.stdout, base.stdout


def test_python_mirror_appends_rows():
    t, s = real_vertex_clouds()
    ti, si = oracle_ncc(t, s, False, 2000, True)
    pre = kpts(2, np.random.default_rng(1))
    ok, tc, sc = CRegistration(0, 1000, 20000).find_feature_correspondence_ncc(t, s, pre, pre)
    assert ok
    assert np.array_equal(tc.view(np.uint32), np.concatenate([pre, t[ti]]).view(np.uint32))
    assert np.array_equal(sc.view(np.uint32), np.concatenate([pre, s[si]]).view(np.uint32))
