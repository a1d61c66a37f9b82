"""The call frame the stateless front-end entry points share (PCA, SOR, raw-scan corrections, NCC, RANSAC, voxel and
ground filters, classification, extract_semantic_pts): each call reports its own kernel launches and device time, a
call that launches nothing reports zero launches whatever ran before it, mulls_extract_semantic_pts counts each of its
stages once, and a call that fails leaves the context as good as a fresh one."""
import ctypes as C

import numpy as np
import pytest

from mulls_b200 import abi, synth
from mulls_b200.registration import Context

pytestmark = pytest.mark.gpu

EMPTY = np.zeros((0, 12), np.float32)


@pytest.fixture(scope="module")
def raw():
    """every return of a small synthetic sweep (ground, pillars, facades, ...), normals and curvature wiped"""
    rows = np.concatenate(synth.make_pair(5, "small")["tgt"], axis=0).copy()
    rows[:, 3:8] = 0
    rows[:, 9:] = 0
    return np.ascontiguousarray(rows)


@pytest.fixture(scope="module")
def unground():
    """the non-ground returns of another sweep, normals wiped: what the classification takes"""
    tgt = synth.make_pair(7, "small")["tgt"]
    rows = np.concatenate([tgt[c] for c in (abi.PILLAR, abi.FACADE, abi.BEAM, abi.ROOF)], axis=0).copy()
    rows[:, 4:8] = 0
    return np.ascontiguousarray(rows)


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, 1, 16, 200000)
    yield c
    c.close()


def classify_params():
    p = abi.default_classify_params()
    p.neighbor_searching_radius, p.neighbor_k, p.neigh_k_min, p.pca_down_rate = 1.0, 30, 8, 1
    p.fixed_num_downsampling, p.random_seed = 1, 5
    return p


def run_sor(ctx, raw):
    """a call that launches kernels, so that stale statistics would show"""
    ctx.sor_filter(raw, 10, 1.0)
    st = ctx.stats()
    assert st["kernel_launches"] > 0 and st["ms_total"] > 0


def launches(ctx):
    return ctx.stats()["kernel_launches"]


def assert_same_rows(a, b, tag):
    assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), tag


NOTHING_LAUNCHED = {
    "voxel_downsample_disabled": lambda c, raw: c.voxel_downsample(raw, 0.0),
    "classify_nground_empty": lambda c, raw: c.classify_nground(EMPTY, classify_params()),
    "fast_ground_filter_empty": lambda c, raw: c.fast_ground_filter(EMPTY, abi.default_ground_params()),
    "timestamp_ratio_empty": lambda c, raw: c.timestamp_ratio(EMPTY),
    "motion_compensation_empty": lambda c, raw: c.motion_compensation(EMPTY, np.eye(4)),
    "vertical_calibration_disabled": lambda c, raw: c.vertical_intrinsic_calibration(raw, 0.0),
}


@pytest.mark.parametrize("name", sorted(NOTHING_LAUNCHED))
def test_a_call_that_launches_nothing_reports_no_launches(ctx, raw, name):
    run_sor(ctx, raw)
    NOTHING_LAUNCHED[name](ctx, raw)
    assert launches(ctx) == 0


@pytest.mark.parametrize("resolution", [0.0, 0.1])
def test_extract_semantic_pts_counts_each_stage_once(ctx, raw, resolution):
    gp, cp = abi.default_ground_params(), classify_params()
    down, expect = raw, 0
    if resolution > 0:
        down = ctx.voxel_downsample(raw, resolution)
        expect += launches(ctx)
    g = ctx.fast_ground_filter(down, gp)
    expect += launches(ctx)
    c = ctx.classify_nground(g["unground"], cp)
    expect += launches(ctx)
    run_sor(ctx, raw)
    e = ctx.extract_semantic_pts(raw, resolution, gp, cp)
    st = ctx.stats()
    assert st["kernel_launches"] == expect and st["ms_total"] > 0
    assert_same_rows(e["down"], down, "down")
    for k in ("ground", "ground_down"):
        assert_same_rows(e[k], g[k], k)
    for k in abi.OUT_NAMES:
        assert_same_rows(e[k], c[k], k)
    assert len(g["ground"]) > 0 and len(c["facade"]) > 0


def test_ground_filter_counts_the_kernels_it_launches(ctx, raw):
    g = ctx.fast_ground_filter(raw, abi.default_ground_params())
    assert len(g["ground"]) > 0 and len(g["unground"]) > 0
    # k_gf_bbox and k_gf_setup, then ten kernels over the cells (the library sort and scans are not counted)
    assert launches(ctx) == 12


def test_a_failed_call_leaves_the_context_as_good_as_a_fresh_one(ctx, unground):
    p = classify_params()
    rows = abi.as_aos48(unground)
    n = len(rows)
    assert n < p.unground_down_fixed_num  # the unground output holds every input row
    bufs = [np.zeros((n, 12), np.float32) for _ in range(abi.OUT_COUNT)]
    out = abi.ClassifyOut()
    for k in range(abi.OUT_COUNT):
        out.rows[k] = bufs[k].ctypes.data_as(C.POINTER(C.c_float))
    out.cap = n - 1  # every class fits, the last output (unground) does not: the earlier copies are in flight
    assert ctx.lib.mulls_classify_nground(ctx.handle, abi.cloud_view(rows), C.byref(p), C.byref(out)) == -102
    after = ctx.classify_nground(rows, p)
    fresh = Context(0, 1, 16, 200000)
    try:
        expect = fresh.classify_nground(rows, p)
    finally:
        fresh.close()
    for k in abi.OUT_NAMES:
        assert_same_rows(after[k], expect[k], k)
    assert len(expect["facade"]) > 0 and len(expect["unground"]) == n
