"""The Morton order the ingest builds inside every (pair, segment) on the device (k_make_keys' digit histograms,
k_digit_scan, the four k_sort_pass passes and k_cell_count), point by point against numpy: a stable sort of the 36-bit
Morton codes of the points the intersection filter keeps, equal codes in input order (np.lexsort on the input index and
the code). The clouds are adversarial for the sort: many equal keys, segments of zero, one and two points, a segment of
more than 2^17 points (tens of tiles in one look-back chain), a pair wider than 500 m (the level-0 cell doubles), and
filtered-out points in every segment."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = np.uint64(0xFFFFFFFFFFFFFFFF)


@pytest.fixture(scope="module")
def sort_lib():
    src = os.path.join(ROOT, "tests", "harness", "ingest_sort_device.cu")
    out = os.path.join(ROOT, "tests", "harness", "_build", "libingest_sort_device.so")
    deps = [src] + [os.path.join(ROOT, "mulls_b200", "csrc", f)
                    for f in ("kernels_ingest.cuh", "device_types.cuh", "device_math.cuh", "grid_key.cuh", "search_core.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false",
                               "-I", os.path.join(ROOT, "include"), "-Xcompiler", "-fPIC", "-shared", "-o", out, src])
    lb = C.CDLL(out)
    P = C.c_void_p
    lb.is_run.restype = C.c_int
    lb.is_run.argtypes = [P, P, C.c_int, P, P, P, P, P, P, P, P, P]
    return lb


def spread12(v):
    v = np.asarray(v, np.uint64) & np.uint64(0xFFF)
    r = np.zeros_like(v)
    for b in range(12):
        r |= ((v >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b)
    return r


def morton36(c):
    return spread12(c[:, 0]) | (spread12(c[:, 1]) << np.uint64(1)) | (spread12(c[:, 2]) << np.uint64(2))


def rows(xyz):
    r = np.zeros((len(xyz), 12), np.float32)
    r[:, :3] = xyz
    r[:, 6] = 1.0
    return r


def run(lib, pairs, tbounds):
    """pairs: per pair a list of 12 (n, 3) clouds (targets then sources)"""
    n_pairs = len(pairs)
    clouds = [np.asarray(c, np.float32).reshape(-1, 3) for p in pairs for c in p]
    in_n = np.array([len(c) for c in clouds], np.uint32)
    n_in = int(in_n.sum())
    r = np.ascontiguousarray(np.concatenate([rows(c) for c in clouds]) if n_in else np.zeros((1, 12), np.float32))
    tb = np.ascontiguousarray(np.asarray(tbounds, np.float64).reshape(n_pairs, 6))
    keys = np.zeros(max(n_in, 1), np.uint64)
    tgt_idx = np.zeros(max(n_in, 1), np.int32)
    src_idx = np.zeros(max(n_in, 1), np.int32)
    seg_start = np.zeros(12 * n_pairs, np.uint32)
    seg_count = np.zeros(12 * n_pairs, np.uint32)
    h0o = np.zeros(4 * n_pairs, np.float32)
    ibb = np.zeros(6 * n_pairs, np.float64)
    cells = np.zeros(6 * n_pairs, np.uint32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib.is_run(ptr(r), ptr(in_n), n_pairs, ptr(tb), ptr(keys), ptr(tgt_idx), ptr(src_idx), ptr(seg_start),
                    ptr(seg_count), ptr(h0o), ptr(ibb), ptr(cells))
    assert rc == 0, f"CUDA error {rc - 1}"
    return dict(clouds=clouds, n_in=n_in, keys=keys[:n_in], tgt_idx=tgt_idx, src_idx=src_idx, seg_start=seg_start,
                seg_count=seg_count, h0=h0o.reshape(n_pairs, 4)[:, 0], origin=h0o.reshape(n_pairs, 4)[:, 1:],
                ibb=ibb.reshape(n_pairs, 6), cells=cells.reshape(n_pairs, 6))


def n_levels(h0):
    rmax = np.float32(2.5) * np.float32(1.5) * np.float32(1.0001)
    L = 2
    while L < 12 and np.float32(0.999) * np.float32(0.5) * h0 * np.float32(1 << (L - 1)) < rmax:
        L += 1
    return L


def check(out, n_pairs):
    """every segment: the device order equals the stable numpy order of its kept points; keys, slices, counts, tail"""
    kept_total = 0
    tgt_base = src_base = 0
    for p in range(n_pairs):
        ibb, h0, origin = out["ibb"][p], out["h0"][p], out["origin"][p]
        for s in range(12):
            xyz = out["clouds"][12 * p + s]
            x = xyz.astype(np.float64)
            inside = np.all((x > ibb[:3]) & (x < ibb[3:]), axis=1)
            cell = np.floor((xyz - origin) * (np.float32(1) / h0)).astype(np.int64)
            m = morton36(np.clip(cell, 0, 4095).astype(np.uint64))
            idx = np.nonzero(inside)[0]
            order = idx[np.lexsort((idx, m[idx]))]
            n = len(order)
            assert out["seg_count"][12 * p + s] == n, (p, s)
            start = int(out["seg_start"][12 * p + s])
            assert start == kept_total, (p, s)
            want = (np.uint64(12 * p + s) << np.uint64(36)) | m[order]
            np.testing.assert_array_equal(out["keys"][start:start + n], want, err_msg=f"keys of pair {p} seg {s}")
            if s < 6:
                got = out["tgt_idx"][tgt_base:tgt_base + n]
                tgt_base += len(xyz)
                L = n_levels(h0)
                assert out["cells"][p, s] == sum(len(np.unique(m[idx] >> np.uint64(3 * l))) for l in range(L)), (p, s)
            else:
                got = out["src_idx"][src_base:src_base + n]
                src_base += len(xyz)
            np.testing.assert_array_equal(got, order, err_msg=f"order of pair {p} seg {s}")
            kept_total += n
    assert np.all(out["keys"][kept_total:] == NONE)
    assert kept_total < out["n_in"]  # every batch here filters points out


def with_outliers(rng, xyz, frac=0.1):
    """replace a fraction of the points by points outside the +-50 m target bound (and the 1 m pad)"""
    xyz = np.array(xyz, np.float32)
    k = int(round(frac * len(xyz)))
    if k:
        sel = rng.choice(len(xyz), k, replace=False)
        xyz[sel] = rng.uniform(55, 70, (k, 3)).astype(np.float32) * rng.choice([-1, 1], (k, 3))
    return xyz


def scan_like(rng, n, half=45.0):
    """a ring-ordered ground-ish cloud: neighbours in input order are neighbours in space"""
    t = np.linspace(0, 40 * np.pi, n)
    r = 5 + half * 0.8 * (t / t[-1])
    return np.stack([r * np.cos(t), r * np.sin(t), rng.normal(0, 1.0, n)], 1).astype(np.float32)


BOUND = [-50, -50, -50, 50, 50, 50]


@pytest.mark.gpu
def test_segment_order_on_adversarial_segments(sort_lib):
    rng = np.random.default_rng(7)
    dup = rng.uniform(-40, 40, (60, 3)).astype(np.float32)[rng.integers(0, 60, 20000)]  # many equal keys
    pair0 = [
        with_outliers(rng, dup),
        rng.uniform(-10, 10, (1, 3)),                        # one point
        np.zeros((0, 3)),                                     # empty
        with_outliers(rng, rng.uniform(-45, 45, (3000, 3))),
        with_outliers(rng, scan_like(rng, 150000)),          # > 2^17 points: 37 tiles in one look-back chain
        with_outliers(rng, rng.uniform(-45, 45, (500, 3))),
        with_outliers(rng, scan_like(rng, 7000)),            # source ground: part of the intersection box
        np.zeros((0, 3)),
        np.array([[1.0, 2.0, 3.0], [90.0, 0.0, 0.0]]),       # two points, one filtered out
        with_outliers(rng, rng.uniform(-45, 45, (40000, 3))),
        with_outliers(rng, dup[:4097]),                      # one point past a tile, equal keys across the boundary
        with_outliers(rng, rng.uniform(-45, 45, (9000, 3))),
    ]
    pair1 = [with_outliers(rng, rng.uniform(-45, 45, (n, 3))) for n in (5000, 4096, 4095, 0, 1, 8192)] + \
            [with_outliers(rng, rng.uniform(-45, 45, (n, 3))) for n in (3000, 300, 2, 0, 4097, 100)]
    pairs = [pair0, pair1]
    out = run(sort_lib, pairs, [BOUND, BOUND])
    check(out, len(pairs))


@pytest.mark.gpu
def test_segment_order_when_the_level0_cell_has_doubled(sort_lib):
    rng = np.random.default_rng(8)
    wide = lambda n: np.concatenate([rng.uniform(-400, 400, (n, 1)), rng.uniform(-30, 30, (n, 2))], 1)
    bound = [-1000, -1000, -1000, 1000, 1000, 1000]
    pair = [np.concatenate([wide(n), rng.uniform(1100, 1200, (n // 10 + 1, 3))]) for n in
            (30000, 2000, 700, 1, 5000, 64)]
    pair += [np.concatenate([wide(n), rng.uniform(1100, 1200, (n // 10 + 1, 3))]) for n in
             (20000, 3000, 900, 1, 0, 10)]
    out = run(sort_lib, [pair], [bound])
    assert out["h0"][0] >= 0.25  # 800 m do not fit 4092 cells of 0.125 m
    check(out, 1)
