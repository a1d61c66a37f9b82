"""GPU checks of the raw-scan corrections against the CPU restatement (tests/harness/rawscan_oracle.cpp): timestamp ratios,
skip decisions and every untouched column bit for bit; the outputs of asin / cos / sin / atan2 / acos within one float
ulp (CUDA's double functions are not the host's libm; the count of values that differ at all is printed). On the
adversarial clouds of tests/test_rawscan.py, a 120k-point scan, a 1.9 M-point merged map, the six-cloud batch in one call,
the refusals; and the drop-in CFilter on the device."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from mulls_b200 import abi, synth
from mulls_b200.registration import Context
from oracle import oracle
from test_adaptive_pca import orc_classify_adaptive
from test_rawscan import (MOTION_CLOUDS, TRANSFORMS, TS_CLOUDS, VERTICAL_CASES, F32, assert_azimuth_ratio, assert_rows_close,
                          assert_rows_equal, build_rawscan_caller, geometry_cloud, orc_batch_motion, orc_motion, orc_ratio,
                          orc_scanner_filter, orc_vertical, rows_of, scan_like)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, 1, 16, 2_000_000)
    yield c
    c.close()


@pytest.fixture(scope="module")
def merged_map():
    """about 1.9 M points, curvature = a timestamp in a 100 ms sweep"""
    m = synth.make_merged_map(11, 16, n_points=120000)
    m[:, 9] = np.random.default_rng(3).uniform(0.0, 100.0, len(m)).astype(F32)
    return m


def with_xyz(rows, xyz):
    out = np.array(rows, F32, copy=True)
    out[:, :3] = xyz
    return out


def with_curvature(rows, c):
    out = np.array(rows, F32, copy=True)
    out[:, 9] = c
    return out


def check_vertical(ctx, rows, var, inverse_z=False):
    xyz, applied = ctx.vertical_intrinsic_calibration(rows, var, inverse_z)
    exp, ok = orc_vertical(rows, var, inverse_z)
    assert applied == ok
    if var == 0 or var >= 180 or inverse_z:
        assert_rows_equal(with_xyz(rows, xyz), exp, f"vertical {var}")
        return 0
    return assert_rows_close(with_xyz(rows, xyz), exp, f"vertical {var} ({len(rows)} points)")


@pytest.mark.parametrize("var,inverse_z", VERTICAL_CASES)
def test_vertical_calibration_equals_restatement(ctx, var, inverse_z):
    rows = geometry_cloud(np.random.default_rng(3))
    check_vertical(ctx, rows, var, inverse_z)
    for n in (0, 1):
        check_vertical(ctx, rows[:n], var, inverse_z)
    check_vertical(ctx, scan_like(120000, np.random.default_rng(1)), var, inverse_z)


@pytest.mark.parametrize("name,rows,duration", TS_CLOUDS, ids=[c[0] for c in TS_CLOUDS])
def test_timestamp_ratio_equals_restatement(ctx, name, rows, duration):
    got = ctx.timestamp_ratio(rows, True, 180.0, duration)
    assert_rows_equal(with_curvature(rows, got), orc_ratio(rows, True, duration_ms=duration), name)


@pytest.mark.parametrize("begin", [180.0, 90.0, 270.0, 0.0])
def test_azimuth_ratio_equals_restatement(ctx, begin):
    for rows in (geometry_cloud(np.random.default_rng(4)), scan_like(120000, np.random.default_rng(5), False)):
        got = with_curvature(rows, ctx.timestamp_ratio(rows, False, begin))
        assert_azimuth_ratio(got, rows, begin, f"device azimuth {begin} ({len(rows)} points)")
        # and against the restatement: both within one float ulp of the same angle
        exp = orc_ratio(rows, False, begin)
        print(f"  {int((got[:, 9].view(np.uint32) != exp[:, 9].view(np.uint32)).sum())} ratios differ from the host's")


@pytest.mark.parametrize("tname", sorted(TRANSFORMS))
@pytest.mark.parametrize("name,rows,thre", MOTION_CLOUDS, ids=[c[0] for c in MOTION_CLOUDS])
def test_motion_compensation_equals_restatement(ctx, tname, name, rows, thre):
    T = TRANSFORMS[tname]
    got = with_xyz(rows, ctx.motion_compensation(rows, T, thre))
    exp = orc_motion(rows, T, thre)
    if tname in ("identity", "near_identity"):
        assert_rows_equal(got, exp, name)
    else:
        assert_rows_close(got, exp, f"motion {tname} {name}")
    c = rows[:, 9]
    skip = (c < F32(thre)) | (c.astype(np.float64) > 1.0 - float(F32(thre)))
    assert_rows_equal(got[skip], rows[skip], "skipped rows")


def test_merged_map_and_scan(ctx, merged_map):
    scan = scan_like(124668, np.random.default_rng(8))
    for rows in (scan, merged_map):
        check_vertical(ctx, rows, 0.5)
        ts = ctx.timestamp_ratio(rows, True)
        exp = orc_ratio(rows, True)
        assert_rows_equal(with_curvature(rows, ts), exp, f"timestamps ({len(rows)} points)")
        got = with_xyz(exp, ctx.motion_compensation(exp, TRANSFORMS["small"]))
        assert_rows_close(got, orc_motion(exp, TRANSFORMS["small"]), f"motion ({len(rows)} points)")


@pytest.mark.parametrize("keypoints", [False, True])
def test_six_cloud_batch_in_one_call(ctx, keypoints):
    rng = np.random.default_rng(9)
    clouds = [rows_of(rng.uniform(-30, 30, (n, 3)), rng.uniform(0, 1, n)) for n in (30000, 0, 5000, 1, 70000, 2000)]
    T = TRANSFORMS["negative_w"]
    k = 6 if keypoints else 5
    got = ctx.motion_compensation(clouds[:k], T)
    assert ctx.stats()["kernel_launches"] == 1
    exp = orc_batch_motion(clouds, T, keypoints)
    for i in range(k):
        assert_rows_close(with_xyz(clouds[i], got[i]), exp[i], f"batch cloud {i}")


def test_refusals():
    c = Context(0, 1, 16, 1000)
    try:
        rows = rows_of(np.random.default_rng(2).uniform(-9, 9, (1001, 3)))
        with pytest.raises(RuntimeError, match="-102"):
            c.vertical_intrinsic_calibration(rows, 0.5)
        with pytest.raises(RuntimeError, match="-102"):
            c.timestamp_ratio(rows, True)
        with pytest.raises(RuntimeError, match="-102"):
            c.motion_compensation([rows[:600], rows[600:]], np.eye(4))  # 1001 points together
        for clouds in ([], [rows[:10]] * 7):
            with pytest.raises(RuntimeError, match="-101"):
                c.motion_compensation(clouds, np.eye(4))
        lib = abi.load_library()
        view = abi.cloud_view(np.ascontiguousarray(rows[:10]))
        assert lib.mulls_timestamp_ratio(c.handle, view, 1, 180.0, 100.0, None) == abi.E_ARG
        assert lib.mulls_vertical_intrinsic_calibration(c.handle, view, 0.5, 0, None, None) == abi.E_ARG
        assert lib.mulls_motion_compensation(c.handle, None, 1, None, 0.0, None) == abi.E_ARG
        # and the context still works
        xyz = c.motion_compensation(rows[:600], TRANSFORMS["small"])
        assert_rows_close(with_xyz(rows[:600], xyz), orc_motion(rows[:600], TRANSFORMS["small"]), "after refusals")
    finally:
        c.close()


def test_resident_batch_survives_the_calls():
    pair = synth.make_pair(1000, "small")
    c = Context(0, 1, 100000, 100000)
    try:
        c.upload([pair])
        r0, _ = c.run_resident()
        rows = scan_like(5000, np.random.default_rng(4))
        c.vertical_intrinsic_calibration(rows, 0.5)
        c.timestamp_ratio(rows, True)
        c.motion_compensation(rows, TRANSFORMS["small"])
        r1, _ = c.run_resident()
        assert np.array_equal(r0[0]["T"], r1[0]["T"]) and r0[0]["code"] == r1[0]["code"]
    finally:
        c.close()


# ---------------------------------------------------------------------------------------------------------------------
# the drop-in CFilter on the device
# ---------------------------------------------------------------------------------------------------------------------
def shim_params():
    """the parameters the drop-in extract_semantic_pts hands the device for the argument list of
    tests/stubs/rawscan_caller.cpp (include/common/cfilter_b200.hpp, first call of the process: seeds 0)"""
    g = abi.default_ground_params()
    g.min_grid_pt_num, g.grid_resolution, g.max_height_difference, g.neighbor_height_diff = 10, 3.0, 0.3, 1.5
    g.max_ground_height, g.ground_random_down_rate, g.ground_random_down_down_rate = 5.0, 15, 2
    g.nonground_random_down_rate, g.reliable_neighbor_grid_num_thre, g.estimate_ground_normal_method = 3, 0, 3
    g.normal_estimation_radius, g.distance_weight_downsampling_method, g.standard_distance = 2.0, 2, 15.0
    g.fixed_num_downsampling, g.down_ground_fixed_num, g.intensity_thre = 0, 300, np.finfo(F32).max
    g.apply_grid_wise_outlier_filter, g.random_seed = 1, 0  # apply_scanner_filter is passed on there (cfilter.hpp:2361)
    p = abi.default_classify_params()
    p.neighbor_searching_radius, p.neighbor_k, p.neigh_k_min, p.pca_down_rate = 1.0, 50, 8, 1
    p.edge_thre, p.planar_thre, p.edge_thre_down, p.planar_thre_down = 0.65, 0.65, 0.75, 0.75
    p.extract_vertex_points_method, p.curvature_thre, p.vertex_curvature_non_max_radius = 2, 0.12, 1.5 * F32(1.0)
    p.linear_vertical_sin_high_thre, p.linear_vertical_sin_low_thre = 0.94, 0.17
    p.planar_vertical_sin_high_thre, p.planar_vertical_sin_low_thre = 0.98, 0.34
    p.fixed_num_downsampling, p.pillar_down_fixed_num, p.facade_down_fixed_num = 0, 200, 800
    p.beam_down_fixed_num, p.roof_down_fixed_num, p.unground_down_fixed_num = 200, 100, 10000
    p.beam_height_max, p.roof_height_min, p.feature_pts_ratio_guess = np.finfo(F32).max, 0.0, 0.3
    p.sharpen_with_nms, p.use_distance_adaptive_pca, p.pca_unit_distance, p.random_seed = 1, 1, 30.0, 0
    return g, p


@pytest.mark.parametrize("method", [1, 2])
def test_dropin_replays_the_driver_as_the_restatements_do(ctx, method):
    from test_ground import raw_scan

    raw, _ = raw_scan()
    rng = np.random.default_rng(6)
    ego = rng.uniform(-1.2, 1.2, (40, 3)) * [1, 1, 0.5]  # inside the 1.75 m self ring
    ghost = np.stack([rng.uniform(-12, 12, 40), rng.uniform(-12, 12, 40), rng.uniform(-8.9, -6.1, 40)], 1)  # underground
    raw = np.concatenate([raw, rows_of(np.concatenate([ego, ghost]))])
    raw[:, 9] = rng.uniform(0.0, 100.0, len(raw)).astype(F32)  # timestamps (ms)
    T = TRANSFORMS["small"]
    with tempfile.TemporaryDirectory() as td:
        exe = build_rawscan_caller(td)
        path = os.path.join(td, "raw.bin")
        raw.tofile(path)
        out = subprocess.run([exe, path, str(method), td], capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stdout + out.stderr
        got = {k: np.fromfile(os.path.join(td, k + ".bin"), F32).reshape(-1, 12) for k in (
            "raw", "ground", "pillar", "beam", "facade", "roof", "vertex", "ground_down", "pillar_down", "beam_down",
            "facade_down", "roof_down")}
    # :407-412. The trigonometric steps come from the device (checked against the restatement here); every step after
    # them is restated on the CPU, so that a last-bit difference of a coordinate cannot move a discrete decision
    xyz, applied = ctx.vertical_intrinsic_calibration(raw, 0.5)
    assert applied
    r = with_xyz(raw, xyz)
    assert_rows_close(r, orc_vertical(raw, 0.5)[0], "driver vertical")
    if method == 1:
        r2 = orc_ratio(r, True)
        assert_rows_equal(with_curvature(r, ctx.timestamp_ratio(r, True)), r2, "driver timestamps")
    else:
        r2 = with_curvature(r, ctx.timestamp_ratio(r, False, 90.0))
        assert_azimuth_ratio(r2, r, 90.0, "driver azimuth")
    # :2334-2343, then the chain of restatements of :2346-2399
    filtered = orc_scanner_filter(r2, 2.0, -7.0)
    assert len(filtered) <= len(r2) - 80
    g, p = shim_params()
    down = oracle.voxel_downsample(filtered, 0.05)
    og = oracle.fast_ground_filter(down, g)
    oc = orc_classify_adaptive(og["unground"], p)
    assert oc["pillar"].shape[0] + oc["facade"].shape[0] > 0
    # :707-711: pc_raw, the five feature clouds and their down-sampled ones, vertex untouched
    exp = {"raw": orc_motion(filtered, T), "vertex": oc["vertex"]}
    for k in ("ground", "ground_down"):
        exp[k] = orc_motion(og[k], T)
    for k in ("pillar", "beam", "facade", "roof", "pillar_down", "beam_down", "facade_down", "roof_down"):
        exp[k] = orc_motion(oc[k], T)
    for k, e in exp.items():
        if k == "vertex":
            assert_rows_equal(got[k], e, k)
        else:
            assert_rows_close(got[k], e, f"driver {k} (method {method})")
