"""GPU checks of mulls_coarse_reg_teaser (CRegistration::coarse_reg_teaser, cregistration.hpp:664-759): status,
tran_mat bits and every count of mulls_teaser_info but the launch count equal the CPU restatement's
(tests/harness/teaser_oracle.cpp) on every correspondence set of tests/test_teaser.py, on the real chain (vertex clouds
of demo scans 000000 / 000015 -> device NCC matching in best-n, reciprocal and plain mode -> TEASER++, and 000000 /
000001 in best-n 1 000 and reciprocal mode), at 8 000 correspondences and on a dense graph that needs several search
launches; a search that exhausts its budget (a random dense graph, and the plain set of the consecutive scans
000000 / 000001 at noise bound 0.6) ends with the documented error; refusals; the resident batch it leaves alone; and the C++ drop-in on the device."""
import ctypes as C
import os
import subprocess
import tempfile
import time

import numpy as np
import pytest

from mulls_b200 import abi, synth
from mulls_b200.registration import Context, CRegistration
from test_gpu_ransac import vertex_clouds
from test_ransac import build_caller, rows, scene
from test_teaser import CASES, oracle_teaser

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, 1, 40000, 40000)
    yield c
    c.close()


def same_bits(a, b):
    """equal bits, any NaN equal to any NaN (the device and the host need not make the same NaN)"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    na, nb_ = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb_) and np.array_equal(a[~na].view(np.uint64), b[~nb_].view(np.uint64))


def assert_equal_oracle(ctx, t, s, **kw):
    exp = oracle_teaser(t, s, **kw)
    status, T, info = ctx.coarse_reg_teaser(t, s, tran_mat=np.full((4, 4), 7.0), **kw)
    launches = info.pop("search_launches")
    assert (status, info) == (exp["status"], exp["info"]), ((status, info), (exp["status"], exp["info"]))
    assert same_bits(T, exp["T"]), (T, exp["T"])
    return status, info, launches


@pytest.mark.parametrize("name,target,source,kw", CASES, ids=[c[0] for c in CASES])
def test_cases_equal_oracle(ctx, name, target, source, kw):
    assert_equal_oracle(ctx, target, source, **kw)


def chain_corr(ctx, scans, mode):
    t, s = vertex_clouds(*scans)
    if mode == "reciprocal":
        ti, si = ctx.ncc_correspondences(t, s, False, 0, True)
    elif mode == "plain":  # script/run_mulls_reg.sh: --fixed_num_corr_on=false --reciprocal_corr_on=false
        ti, si = ctx.ncc_correspondences(t, s, False, 0, False)
    else:  # test/mulls_slam.cpp's best-n matching
        ti, si = ctx.ncc_correspondences(t, s, True, int(mode.split("_")[-1]), False)
    assert len(ti) > 100
    return t[ti], s[si]


CHAIN = [((0, 15), m) for m in ("best_n_1000", "best_n_4000", "reciprocal", "plain")] + \
    [((0, 1), m) for m in ("best_n_1000", "reciprocal")]


@pytest.mark.parametrize("scans,mode", CHAIN, ids=[f"{a:06d}_{b:06d}_{m}" for (a, b), m in CHAIN])
@pytest.mark.parametrize("noise_bound", [0.6, 1.0])
def test_real_chain_equals_oracle(ctx, scans, mode, noise_bound):
    assert_equal_oracle(ctx, *chain_corr(ctx, scans, mode), noise_bound=noise_bound)


def test_consecutive_scans_plain_exhaust_the_budget(ctx):
    """The plain matching of two consecutive scans at noise bound 0.6 leaves a graph whose clique number the exact
    search cannot prove within its budget (one CPU thread of the restatement takes minutes too). The call says so
    within the budget's time and leaves the context usable."""
    t, s = chain_corr(ctx, (0, 1), "plain")
    t0 = time.time()
    with pytest.raises(RuntimeError, match="-102.*MULLS_TEASER_SEARCH_LAUNCHES"):
        ctx.coarse_reg_teaser(t, s, noise_bound=0.6)
    assert time.time() - t0 < 40.0
    name, t2, s2, kw = CASES[0]
    assert_equal_oracle(ctx, t2, s2, **kw)


def test_8000_correspondences(ctx):
    t, s, _ = scene(8000, 0.1, 5)
    status, info, _ = assert_equal_oracle(ctx, t, s)
    assert status == 1 and info["clique_size"] == 800


def test_dense_graph_takes_several_search_launches(ctx):
    rng = np.random.default_rng(1)
    t, s = rows(rng.uniform(0, 1, (200, 3))), rows(rng.uniform(0, 1, (200, 3)))
    _, info, launches = assert_equal_oracle(ctx, t, s, noise_bound=0.2)
    assert info["n_edges"] > 0.7 * 200 * 199 / 2 and launches > 2, (info, launches)


def test_exhausted_budget_is_an_error_then_the_context_works(ctx):
    rng = np.random.default_rng(2)
    t, s = rows(rng.uniform(0, 1, (2000, 3))), rows(rng.uniform(0, 1, (2000, 3)))
    t0 = time.time()
    with pytest.raises(RuntimeError, match="-102.*MULLS_TEASER_SEARCH_LAUNCHES"):
        ctx.coarse_reg_teaser(t, s, noise_bound=0.3)
    elapsed = time.time() - t0
    assert elapsed < 40.0, elapsed
    name, t2, s2, kw = CASES[0]
    assert_equal_oracle(ctx, t2, s2, **kw)


def test_refusals_then_the_context_still_works():
    c = Context(0, 1, 1000, 1000)
    try:
        t, s, _ = scene(300, 0.5, 2)
        with pytest.raises(RuntimeError, match="-102"):
            c.coarse_reg_teaser(np.concatenate([t] * 4), np.concatenate([s] * 4))
        assert c.coarse_reg_teaser(t, s[:299])[0] == -1  # the reference's refusal: a status, not an error
        lib = abi.load_library()
        T = np.full(16, 7.0)
        st, info = C.c_int(5), abi.TeaserInfo()
        tv, sv = abi.cloud_view(abi.as_aos48(t)), abi.cloud_view(abi.as_aos48(s))
        dp = C.POINTER(C.c_double)
        assert lib.mulls_coarse_reg_teaser(c.handle, tv, sv, 0.2, 8, None, C.byref(st), C.byref(info)) == abi.E_ARG
        assert lib.mulls_coarse_reg_teaser(c.handle, tv, sv, 0.2, 8, T.ctypes.data_as(dp), None, C.byref(info)) == abi.E_ARG
        assert lib.mulls_coarse_reg_teaser(c.handle, abi.CloudView(None, 300), sv, 0.2, 8, T.ctypes.data_as(dp), C.byref(st),
                                           C.byref(info)) == abi.E_ARG
        assert np.all(T == 7.0) and st.value == 5
        assert_equal_oracle(c, t, s)
    finally:
        c.close()
    big = Context(0, 1, 40000, 40000)
    try:
        t, s, _ = scene(32769, 0.1, 3)
        with pytest.raises(RuntimeError, match="-102"):
            big.coarse_reg_teaser(t, s)
    finally:
        big.close()


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


@pytest.mark.parametrize("case", ["known_50pct", "n3", "no_edges"])
def test_dropin_on_the_device_returns_the_oracle_matrix(case):
    name, t, s, kw = next(c for c in CASES if c[0] == case)
    kw = dict(dict(noise_bound=0.2, min_inlier_num=8), **kw)
    marker = (100.0 + np.arange(16)).reshape(4, 4)
    exp = oracle_teaser(t, s, tran=marker, **kw)
    with tempfile.TemporaryDirectory() as td:
        exe = build_caller(td, "teaser_caller")
        paths = [os.path.join(td, f) for f in ("t.bin", "s.bin", "out.bin")]
        np.ascontiguousarray(t, np.float32).tofile(paths[0])
        np.ascontiguousarray(s, np.float32).tofile(paths[1])
        out = subprocess.run([exe] + paths + [repr(float(kw["noise_bound"])), str(kw["min_inlier_num"])],
                             capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stdout + out.stderr
        got = np.fromfile(paths[2], np.float64)
        base = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert int(got[0]) == exp["status"]
    assert same_bits(got[1:].reshape(4, 4), exp["T"])  # the marker on -1
    assert base.returncode == 0 and "ran on a device: 1" in base.stdout and "failures 0" in base.stdout, base.stdout


def test_python_mirror_keeps_tran_mat_on_failure():
    t, s, _ = scene(300, 0.5, 2)
    reg = CRegistration(0, 1000, 1000)
    guess = np.arange(16.0).reshape(4, 4)
    status, T = reg.coarse_reg_teaser(t[:3], s[:3], guess)
    assert status == -1 and np.array_equal(T, guess)
    status, T = reg.coarse_reg_teaser(t, s, guess)
    exp = oracle_teaser(t, s)
    assert status == exp["status"] == 1 and np.array_equal(T, exp["T"])
