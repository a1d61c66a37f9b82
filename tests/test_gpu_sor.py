"""GPU checks of mulls_sor_filter (CFilter::sor_filter -> pcl::StatisticalOutlierRemoval): bit for bit the mean
distances, statistics and keep mask of the CPU restatement (tests/harness/sor_oracle.cpp), on the adversarial clouds of
tests/test_sor.py and on a synthetic merged map, through both host layouts; refusals; the resident batch it replaces;
and the C++ drop-in on the device."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from mulls_b200 import abi, synth
from mulls_b200.registration import Context
from test_sor import CLOUDS, assert_same_result, build_sor_caller, cluster_cloud, oracle_sor_filter, rows_of

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, 1, 4096, 1_500_000)
    yield c
    c.close()


@pytest.fixture(scope="module")
def merged_map():
    """every sweep of a short drive moved into the map frame, plus 0.2 % scattered outliers: about 1.1 M points"""
    return synth.make_merged_map(5, 10, n_points=110000)


@pytest.mark.parametrize("name,rows,mean_k,n_std", CLOUDS, ids=[c[0] for c in CLOUDS])
def test_adversarial_clouds_equal_oracle(ctx, name, rows, mean_k, n_std):
    assert_same_result(ctx.sor_filter(rows, mean_k, n_std), oracle_sor_filter(rows, mean_k, n_std))


@pytest.mark.parametrize("mean_k", [1, 20, 50, 63])
def test_adversarial_clouds_at_every_list_capacity(ctx, mean_k):
    rows = dict((c[0], c[1]) for c in CLOUDS)["triple"]
    assert_same_result(ctx.sor_filter(rows, mean_k, 1.5), oracle_sor_filter(rows, mean_k, 1.5))


@pytest.mark.parametrize("mean_k", [1, 20, 50])
def test_merged_map_equals_oracle(ctx, merged_map, mean_k):
    assert len(merged_map) >= 1 << 18  # shipped in the packed host layout (host_pack)
    exp = oracle_sor_filter(merged_map, mean_k, 2.0)
    assert_same_result(ctx.sor_filter(merged_map, mean_k, 2.0), exp)
    if mean_k == 20:  # the same cloud as 48-byte rows
        ctx.set_tunable("host_pack", 0)
        try:
            assert_same_result(ctx.sor_filter(merged_map, mean_k, 2.0), exp)
        finally:
            ctx.set_tunable("host_pack", 2)
        keep = exp[0]
        assert 0 < int((~keep).sum()) < len(keep) // 10


def test_same_cloud_twice_and_around_a_registration():
    pair = synth.make_pair(1000, "small")
    rows = cluster_cloud(np.random.default_rng(5))
    exp = oracle_sor_filter(rows, 20, 2.0)
    c = Context(0, 1, 100000, 100000)
    try:
        r0, _ = c.run_batch([pair])
        assert_same_result(c.sor_filter(rows, 20, 2.0), exp)
        assert_same_result(c.sor_filter(rows, 20, 2.0), exp)
        r1, _ = c.run_batch([pair])
        assert_same_result(c.sor_filter(rows, 20, 2.0), exp)
        assert np.array_equal(r0[0]["T"], r1[0]["T"]) and r0[0]["code"] == r1[0]["code"]
        with pytest.raises(RuntimeError, match="-101"):  # the filter replaced the resident batch
            c.run_resident()
    finally:
        c.close()


def test_refusals():
    c = Context(0, 1, 1000, 1000)
    try:
        rng = np.random.default_rng(2)
        with pytest.raises(RuntimeError, match="-102"):
            c.sor_filter(rows_of(rng.uniform(-1, 1, (1001, 3))), 20, 2.0)
        rows = rows_of(rng.uniform(-1, 1, (200, 3)))
        for k in (0, -3, 64):
            with pytest.raises(RuntimeError, match="-101"):
                c.sor_filter(rows, k, 2.0)
        few = rows_of(rng.uniform(-1, 1, (21, 3)))
        few[5, 2] = np.inf  # 20 finite points for mean_k = 20
        with pytest.raises(RuntimeError, match="-101"):
            c.sor_filter(few, 20, 2.0)
        with pytest.raises(RuntimeError, match="-101"):
            c.sor_filter(rows_of(np.zeros((0, 3))), 20, 2.0)
        assert_same_result(c.sor_filter(few, 19, 2.0), oracle_sor_filter(few, 19, 2.0))  # and the context still works
    finally:
        c.close()


def test_dropin_shim_on_the_device_returns_the_oracle_rows(merged_map):
    rows = np.ascontiguousarray(merged_map[:300000])
    keep, _, _ = oracle_sor_filter(rows, 20, 2.0)
    with tempfile.TemporaryDirectory() as td:
        exe = build_sor_caller(td)
        src, a, b = (os.path.join(td, f) for f in ("in.bin", "out.bin", "inplace.bin"))
        rows.tofile(src)
        out = subprocess.run([exe, src, a, b, "20", "2.0"], capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stdout + out.stderr
        got_a = np.fromfile(a, np.float32).reshape(-1, 12)
        got_b = np.fromfile(b, np.float32).reshape(-1, 12)
        base = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    expect = rows[keep]
    assert np.array_equal(got_a.view(np.uint32), expect.view(np.uint32))
    assert np.array_equal(got_b.view(np.uint32), expect.view(np.uint32))
    assert base.returncode == 0 and "ran on a device: 1" in base.stdout and "failures 0" in base.stdout, base.stdout
