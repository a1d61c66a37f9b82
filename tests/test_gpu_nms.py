"""GPU checks of mulls_non_max_suppress (CFilter::non_max_suppress, the in-place overload, cfilter.hpp:1183-1240): the
kept row indices of the CPU restatement (tests/harness/nms_oracle.cpp), index for index, on every cloud of
tests/test_nms.py, on the vertex clouds of demo scans 000000, 000001 and 000015 and on the 16 demo vertex clouds
together; the global chain of test/mulls_reg.cpp (extract, NMS on both vertex clouds, NCC, RANSAC) on the device against
the same chain on the CPU; refusals; the resident batch it leaves alone; and the C++ drop-in on the device."""
import ctypes as C
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

from mulls_b200 import abi, synth
from mulls_b200.registration import Context
from test_gpu_ransac import vertex_clouds
from test_ncc import ROOT, _chain_mod, oracle_ncc
from test_nms import CASES, box, build_nms_caller, oracle_nms
from test_ransac import oracle_ransac

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, 1, 4096, 130000)
    yield c
    c.close()


def assert_equal_oracle(ctx, rows, radius):
    exp, exp_performed = oracle_nms(rows, radius)
    got, performed = ctx.non_max_suppress(rows, radius)
    assert performed == exp_performed
    assert np.array_equal(got, exp), (len(got), len(exp), np.flatnonzero(got[: len(exp)] != exp[: len(got)])[:10])
    return got


@pytest.mark.parametrize("name,rows,radius", CASES, ids=[c[0] for c in CASES])
def test_cases_equal_oracle(ctx, name, rows, radius):
    assert_equal_oracle(ctx, rows, radius)


@functools.lru_cache(maxsize=None)
def demo_scan(k):
    mod = _chain_mod()
    z = np.load(os.path.join(ROOT, "tests", "golden", "demo_chain.npz"))
    return mod.decode_scan(z[f"scan{k}_dmm"], z[f"scan{k}_i"])


@pytest.mark.parametrize("radius", [0.25, 0.175])
@pytest.mark.parametrize("scan", [0, 1, 15])
def test_demo_vertex_clouds(ctx, scan, radius):
    v = vertex_clouds(0, 1)[scan] if scan < 2 else vertex_clouds(0, 15)[1]
    kept = assert_equal_oracle(ctx, v, radius)
    assert 0 < len(kept) < len(v)


def test_concatenated_16_demo_vertex_clouds(ctx):
    """a submap-like cloud: the 16 scans' vertex clouds in one, heavy suppression across chunks"""
    mod = _chain_mod()
    gp, cp = mod.chain_params()
    v = np.concatenate([ctx.extract_semantic_pts(demo_scan(k), 0.0, gp, cp)["vertex"] for k in range(16)])
    assert len(v) > 4096
    kept = assert_equal_oracle(ctx, v, 0.25)
    assert len(kept) < 0.9 * len(v)


@pytest.mark.parametrize("scans", [(0, 15)], ids=["000000_000015"])
def test_mulls_reg_global_chain(ctx, scans):
    """test/mulls_reg.cpp:134-179: extract_semantic_pts, non_max_suppress(pc_vertex, 0.25 * pca_neigh_r) on both
    blocks, find_feature_correspondence_ncc with the flags' defaults (no fixed number, 3000, not reciprocal), then
    coarse_reg_ransac with noise bound 4 x 0.25 — on the device, and on the CPU from the oracle's features"""
    mod = _chain_mod()
    gp, cp = mod.chain_params()
    nms_r = 0.25 * 1.0
    dev, cpu = [], []
    for k in scans:
        v = ctx.extract_semantic_pts(demo_scan(k), 0.0, gp, cp)["vertex"]
        idx, performed = ctx.non_max_suppress(v, nms_r)
        assert performed
        dev.append(v[idx])
        o = np.ascontiguousarray(mod.oracle_features(demo_scan(k), gp, cp)["vertex"], np.float32)
        oidx, _ = oracle_nms(o, nms_r)
        cpu.append(o[oidx])
    assert all(np.array_equal(d.view(np.uint32), c.view(np.uint32)) for d, c in zip(dev, cpu))
    ti, si = ctx.ncc_correspondences(dev[0], dev[1], False, 3000, False)
    oti, osi = oracle_ncc(cpu[0], cpu[1], False, 3000, False)
    assert np.array_equal(ti, oti) and np.array_equal(si, osi)
    status, T, n_inl, _ = ctx.coarse_reg_ransac(dev[0][ti], dev[1][si], noise_bound=4.0 * nms_r, tran_mat=np.full((4, 4), 7.0))
    exp = oracle_ransac(cpu[0][oti], cpu[1][osi], noise_bound=4.0 * nms_r)
    assert (status, n_inl) == (exp["status"], exp["n_inliers"])
    assert np.array_equal(T.view(np.uint64), exp["T"].view(np.uint64))
    assert status >= 0


def test_short_cloud_is_not_performed(ctx):
    rows, r = box(np.random.default_rng(3), 9, 0.2)
    idx, performed = ctx.non_max_suppress(rows, r)
    assert not performed and len(idx) == 0
    assert ctx.stats()["kernel_launches"] == 0


def test_refusals_then_the_context_still_works():
    c = Context(0, 1, 1000, 1000)
    try:
        rows, r = box(np.random.default_rng(4), 1001, 1.0)
        with pytest.raises(RuntimeError, match="-102"):
            c.non_max_suppress(rows, r)
        lib = abi.load_library()
        v = abi.cloud_view(abi.as_aos48(rows[:500]))
        idx = np.full(500, -7, np.int32)
        n, performed = C.c_size_t(5), C.c_int(5)
        ip = idx.ctypes.data_as(C.POINTER(C.c_int32))
        assert lib.mulls_non_max_suppress(c.handle, v, 0.25, None, C.byref(n), C.byref(performed)) == abi.E_ARG
        assert lib.mulls_non_max_suppress(c.handle, v, 0.25, ip, None, C.byref(performed)) == abi.E_ARG
        assert lib.mulls_non_max_suppress(c.handle, v, 0.25, ip, C.byref(n), None) == abi.E_ARG
        assert lib.mulls_non_max_suppress(None, v, 0.25, ip, C.byref(n), C.byref(performed)) == abi.E_ARG
        assert np.all(idx == -7) and n.value == 5 and performed.value == 5
        assert_equal_oracle(c, rows[:1000], r)
    finally:
        c.close()


def test_resident_batch_is_left_alone():
    pair = synth.make_pair(1000, "small")
    rows, r = box(np.random.default_rng(5), 3000, 2.0)
    c = Context(0, 1, 100000, 100000)
    try:
        c.upload([pair])
        r0, _ = c.run_resident()
        assert_equal_oracle(c, rows, r)
        r1, _ = c.run_resident()  # no re-upload: the batch and its grid are still there
        assert np.array_equal(r0[0]["T"], r1[0]["T"]) and r0[0]["code"] == r1[0]["code"] and r0[0]["iters"] == r1[0]["iters"]
    finally:
        c.close()


@pytest.mark.parametrize("case", ["zero_nan_inf_scores", "chain_3000_chunks", "nonfinite_coords"])
def test_dropin_on_the_device_returns_the_oracle_rows(case):
    name, rows, r = next(c for c in CASES if c[0] == case)
    exp, _ = oracle_nms(rows, r)
    with tempfile.TemporaryDirectory() as td:
        exe = build_nms_caller(td)
        paths = [os.path.join(td, f) for f in ("in.bin", "a.bin", "b.bin")]
        np.ascontiguousarray(rows, np.float32).tofile(paths[0])
        out = subprocess.run([exe] + paths + [repr(float(r))], capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stdout + out.stderr
        a = np.fromfile(paths[1], np.float32).reshape(-1, 12)
        b = np.fromfile(paths[2], np.float32).reshape(-1, 12)
        base = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    want = np.ascontiguousarray(rows[exp], np.float32)
    assert np.array_equal(a.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(b.view(np.uint32), want.view(np.uint32))
    assert base.returncode == 0 and "ran on a device: 1" in base.stdout and "failures 0" in base.stdout, base.stdout
