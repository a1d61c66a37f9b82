"""CPU checks of the raw-scan corrections (CFilter::vertical_intrinsic_calibration cfilter.hpp:250-291,
get_pts_timestamp_ratio_in_frame :412-467, apply_motion_compensation / batch_apply_motion_compensation :470-549, and the
scanner filter of extract_semantic_pts :2334-2343 / :914-929):
- the CPU restatement (tests/harness/rawscan_oracle.cpp) against an independent numpy restatement on adversarial clouds:
  bit for bit where only + - * / sqrt and comparisons are involved, within one float ulp where asin / cos / sin / atan2 /
  acos are (libm and numpy need not round those alike);
- the drop-in CFilter replays test/mulls_slam.cpp:404-428 and :707-711 against the stand-in headers."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

from mulls_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
DBL_MAX = np.finfo(np.float64).max


# ---------------------------------------------------------------------------------------------------------------------
# the CPU restatement
# ---------------------------------------------------------------------------------------------------------------------
_LIBS = {}


def rawscan_oracle_lib(out_dir=None):
    """Build (when a source is newer) and load tests/harness/rawscan_oracle.cpp (default into tests/harness/_build)."""
    out_dir = out_dir or os.path.join(ROOT, "tests", "harness", "_build")
    if out_dir in _LIBS:
        return _LIBS[out_dir]
    src = os.path.join(ROOT, "tests", "harness", "rawscan_oracle.cpp")
    out = os.path.join(out_dir, "librawscan_oracle.so")
    deps = [src, os.path.join(ROOT, "oracle", "mulls_oracle.cpp"), os.path.join(ROOT, "include", "mulls_b200", "abi.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(out_dir, exist_ok=True)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        subprocess.check_call([cxx, "-O3", "-fPIC", "-fopenmp", "-ffp-contract=off", "-std=c++17", "-w", "-shared", "-o", out, src])
    lb = C.CDLL(out)
    fp, dp = C.POINTER(C.c_float), C.POINTER(C.c_double)
    lb.orc_vertical_intrinsic_calibration.restype = C.c_int
    lb.orc_vertical_intrinsic_calibration.argtypes = [fp, C.c_size_t, C.c_double, C.c_int, C.c_int]
    lb.orc_timestamp_ratio.restype = C.c_int
    lb.orc_timestamp_ratio.argtypes = [fp, C.c_size_t, C.c_int, C.c_double, C.c_float, C.c_int]
    lb.orc_motion_compensation.restype = None
    lb.orc_motion_compensation.argtypes = [fp, C.c_size_t, dp, C.c_float, C.c_int]
    lb.orc_batch_motion_compensation.restype = None
    lb.orc_batch_motion_compensation.argtypes = [C.POINTER(fp), C.POINTER(C.c_size_t), dp, C.c_int, C.c_int]
    lb.orc_oracle_motion_compensate.restype = None
    lb.orc_oracle_motion_compensate.argtypes = [fp, C.c_size_t, dp]
    lb.orc_extract_scanner_filter.restype = C.c_size_t
    lb.orc_extract_scanner_filter.argtypes = [fp, C.c_size_t, C.c_float, C.c_float]
    _LIBS[out_dir] = lb
    return lb


def _rows(rows):
    r = np.array(abi.as_aos48(rows), dtype=F32, order="C", copy=True)
    return r, r.ctypes.data_as(C.POINTER(C.c_float))


def orc_vertical(rows, var, inverse_z=False, threads=0, lib_dir=None):
    """(rows after the member, its return value)"""
    r, p = _rows(rows)
    ok = rawscan_oracle_lib(lib_dir).orc_vertical_intrinsic_calibration(p, len(r), float(var), int(inverse_z), int(threads))
    return r, bool(ok)


def orc_ratio(rows, timestamp_available, begin_deg=180.0, duration_ms=100.0, threads=0, lib_dir=None):
    r, p = _rows(rows)
    rawscan_oracle_lib(lib_dir).orc_timestamp_ratio(p, len(r), int(timestamp_available), float(begin_deg), float(duration_ms),
                                                    int(threads))
    return r


def orc_motion(rows, T, thre=0.0, threads=0, lib_dir=None):
    r, p = _rows(rows)
    Td = np.ascontiguousarray(T, np.float64).reshape(16)
    rawscan_oracle_lib(lib_dir).orc_motion_compensation(p, len(r), Td.ctypes.data_as(C.POINTER(C.c_double)), float(thre),
                                                        int(threads))
    return r


def orc_batch_motion(clouds, T, undistort_keypoints=False, threads=0, lib_dir=None):
    rs = [_rows(c) for c in clouds]
    ptrs = (C.POINTER(C.c_float) * 6)(*[p for _, p in rs])
    ns = (C.c_size_t * 6)(*[len(r) for r, _ in rs])
    Td = np.ascontiguousarray(T, np.float64).reshape(16)
    rawscan_oracle_lib(lib_dir).orc_batch_motion_compensation(ptrs, ns, Td.ctypes.data_as(C.POINTER(C.c_double)),
                                                              int(undistort_keypoints), int(threads))
    return [r for r, _ in rs]


def orc_scanner_filter(rows, approx_scanner_height=2.0, underground_thre=-7.0):
    r, p = _rows(rows)
    n = rawscan_oracle_lib().orc_extract_scanner_filter(p, len(r), float(approx_scanner_height), float(underground_thre))
    return np.ascontiguousarray(r[:n])


# ---------------------------------------------------------------------------------------------------------------------
# the independent restatement (numpy, vectorised)
# ---------------------------------------------------------------------------------------------------------------------
def np_vertical(rows, var, inverse_z=False):
    r = np.array(rows, F32, copy=True)
    if var == 0:
        return r, False
    if var >= 180.0 or inverse_z:
        r[:, 2] = -r[:, 2]  # z *= (-1.0): g++ -O3 emits a sign flip, which flips the sign of a NaN as well
        return r, False
    x, y, z = r[:, 0], r[:, 1], r[:, 2]
    with np.errstate(all="ignore"):
        dist = np.sqrt((x * x + y * y) + z * z).astype(np.float64)  # float products and sum, float sqrt
        v = np.arcsin(z.astype(np.float64) / dist)
        vc = v + var / 180.0 * math.pi
        hs = np.cos(vc) / np.cos(v)
        nx, ny, nz = (x.astype(np.float64) * hs).astype(F32), (y.astype(np.float64) * hs).astype(F32), (dist * np.sin(vc)).astype(F32)
    r[:, 0], r[:, 1], r[:, 2] = nx, ny, nz
    return r, True


def np_ratio(rows, timestamp_available, begin_deg=180.0, duration_ms=100.0):
    r = np.array(rows, F32, copy=True)
    if len(r) == 0:
        return r
    with np.errstate(all="ignore"):
        if timestamp_available:
            c = r[:, 9]
            nan = np.flatnonzero(np.isnan(c))
            suffix = c[nan[-1] + 1:] if len(nan) else c
            if len(suffix) == 0:  # the last timestamp is NaN: both running values end on it
                last = first = float(c[-1])
            else:  # the max_ / min_ macros: among equal values (+0 / -0) the later point wins
                rev = suffix[::-1]
                last, first = float(rev[np.argmax(rev)]), float(rev[np.argmin(rev)])
                if not len(nan):
                    last = -DBL_MAX if -DBL_MAX > last else last
                    first = DBL_MAX if DBL_MAX < first else first
            dur = F32(duration_ms)
            actual = last - first
            if actual < float(dur) * 0.75:
                dur = F32(actual)
            s = (last - c.astype(np.float64)) / float(dur)
            lo = np.where(0.0 > s, 0.0, s)
            r[:, 9] = np.where(1.0 < lo, 1.0, lo).astype(F32)
        else:
            r[:, 9] = _ratio_of_angle(float_atan2(r[:, 1], r[:, 0]), begin_deg)
    return r


def float_atan2(y, x):
    """the float overload std::atan2(float, float), to within one float ulp: numpy's double atan2 of the widened
    arguments, rounded to float (numpy's own float32 arctan2 is less accurate than that)"""
    with np.errstate(all="ignore"):
        return np.arctan2(np.asarray(y, F32).astype(np.float64), np.asarray(x, F32).astype(np.float64)).astype(F32)


def _ratio_of_angle(ang32, begin_deg):
    with np.errstate(all="ignore"):
        ang = np.asarray(ang32, F32).astype(np.float64)
        ang = np.where(ang < 0, ang + 2 * math.pi, ang)
        ang = ang + begin_deg / 180.0 * math.pi
        ang = np.where(ang >= 2 * math.pi, ang - 2 * math.pi, ang)
        return ((2 * math.pi - ang) / (2 * math.pi)).astype(F32)


def np_quaternion(T):
    """Eigen::Quaterniond(Matrix3d): (x, y, z, w)"""
    m = np.asarray(T, np.float64)[:3, :3]
    q = [0.0] * 4
    t = m[0, 0] + m[1, 1] + m[2, 2]
    if t > 0.0:
        t = math.sqrt(t + 1.0)
        q[3] = 0.5 * t
        t = 0.5 / t
        q[0], q[1], q[2] = (m[2, 1] - m[1, 2]) * t, (m[0, 2] - m[2, 0]) * t, (m[1, 0] - m[0, 1]) * t
    else:
        i = 0
        if m[1, 1] > m[0, 0]:
            i = 1
        if m[2, 2] > m[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = math.sqrt(m[i, i] - m[j, j] - m[k, k] + 1.0)
        q[i] = 0.5 * t
        t = 0.5 / t
        q[3] = (m[k, j] - m[j, k]) * t
        q[j] = (m[j, i] + m[i, j]) * t
        q[k] = (m[k, i] + m[i, k]) * t
    return q


def np_motion(rows, T, thre=0.0):
    r = np.array(rows, F32, copy=True)
    T = np.asarray(T, np.float64)
    qx0, qy0, qz0, qw0 = np_quaternion(T)
    c = r[:, 9]
    move = ~((c < F32(thre)) | (c.astype(np.float64) > 1.0 - float(F32(thre))))
    s = c[move].astype(np.float64)
    d = qw0
    with np.errstate(all="ignore"):
        if abs(d) >= 1.0 - np.finfo(np.float64).eps:
            s0, s1 = 1.0 - s, s
        else:
            th = math.acos(abs(d))
            s0, s1 = np.sin((1.0 - s) * th) / math.sin(th), np.sin(s * th) / math.sin(th)
        if d < 0:
            s1 = -s1
        qx, qy, qz, qw = s1 * qx0, s1 * qy0, s1 * qz0, s0 + s1 * qw0
        v = r[move, :3].astype(np.float64)
        ux, uy, uz = qy * v[:, 2] - qz * v[:, 1], qz * v[:, 0] - qx * v[:, 2], qx * v[:, 1] - qy * v[:, 0]
        ux, uy, uz = ux + ux, uy + uy, uz + uz
        out = np.stack([v[:, 0] + qw * ux + (qy * uz - qz * uy) + s * T[0, 3],
                        v[:, 1] + qw * uy + (qz * ux - qx * uz) + s * T[1, 3],
                        v[:, 2] + qw * uz + (qx * uy - qy * ux) + s * T[2, 3]], 1)
    r[move, :3] = out.astype(F32)
    return r


def np_scanner_filter(rows, approx_scanner_height=2.0, underground_thre=-7.0):
    r = np.asarray(rows, F32)
    h, u = F32(approx_scanner_height), F32(underground_thre)
    z_min = F32(float(-h) - 4.0)
    z_min_min = -h + u  # float
    x, y, z = r[:, 0], r[:, 1], r[:, 2]
    with np.errstate(all="ignore"):
        ds = x * x + y * y
        keep = (ds > F32(1.75) * F32(1.75)) & (z > z_min_min) & ((ds > F32(20.0) * F32(20.0)) | (z > z_min))
    return np.ascontiguousarray(r[keep])


# ---------------------------------------------------------------------------------------------------------------------
# comparisons
# ---------------------------------------------------------------------------------------------------------------------
def ulp_diff(a, b):
    """per value: 0 for equal bits (or both NaN), else the distance in float32 ulps (huge for NaN against a number)"""
    a, b = np.asarray(a, F32).ravel(), np.asarray(b, F32).ravel()

    def key(v):
        i = v.view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)

    d = np.abs(key(a) - key(b))
    both_nan = np.isnan(a) & np.isnan(b)
    one_nan = np.isnan(a) ^ np.isnan(b)
    d = np.where(both_nan | (a.view(np.uint32) == b.view(np.uint32)), 0, d)
    return np.where(one_nan, 1 << 40, d)


def assert_rows_close(got, exp, what, max_ulp=1, cols=(0, 1, 2)):
    """every column outside `cols` bit-identical; `cols` within max_ulp float ulps. Returns the count of values of `cols`
    that differ at all."""
    got, exp = np.asarray(got, F32), np.asarray(exp, F32)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    other = [c for c in range(12) if c not in cols]
    assert np.array_equal(got[:, other].view(np.uint32), exp[:, other].view(np.uint32)), what
    d = ulp_diff(got[:, list(cols)], exp[:, list(cols)])
    assert d.max(initial=0) <= max_ulp, (what, int(d.max()), np.flatnonzero(d > max_ulp)[:8])
    n = int((d > 0).sum())
    print(f"{what}: {n} of {d.size} values differ by one float ulp")
    return n


def assert_rows_equal(got, exp, what):
    """bit for bit, except that any NaN equals any NaN: which operand's NaN an operation passes on, and with what sign,
    is not specified and differs between compilers and between the host and the device"""
    got, exp = np.asarray(got, F32), np.asarray(exp, F32)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    bad = (got.view(np.uint32) != exp.view(np.uint32)) & ~(np.isnan(got) & np.isnan(exp))
    assert not bad.any(), (what, np.flatnonzero(bad.any(1))[:8])


def assert_azimuth_ratio(got, rows, begin, what):
    """the float atan2 within one float ulp of numpy's, everything after it exact: each ratio is the one computed from
    numpy's angle or from one of its two float neighbours. Returns the count of ratios that differ from numpy's."""
    got = np.asarray(got, F32)
    exp = np_ratio(rows, False, begin)
    assert_rows_equal(np.delete(got, 9, 1), np.delete(exp, 9, 1), what)
    with np.errstate(all="ignore"):
        a = float_atan2(np.asarray(rows, F32)[:, 1], np.asarray(rows, F32)[:, 0])
        ok = np.zeros(len(got), bool)
        for cand in (a, np.nextafter(a, F32(np.inf)), np.nextafter(a, F32(-np.inf))):
            r = _ratio_of_angle(cand, begin)
            ok |= (r.view(np.uint32) == got[:, 9].view(np.uint32)) | (np.isnan(r) & np.isnan(got[:, 9]))
    assert ok.all(), (what, np.flatnonzero(~ok)[:8])
    n = int((got[:, 9].view(np.uint32) != exp[:, 9].view(np.uint32)).sum())
    print(f"{what}: {n} of {len(got)} ratios come from an angle one float ulp off numpy's")
    return n


# ---------------------------------------------------------------------------------------------------------------------
# the clouds (shared with tests/test_gpu_rawscan.py)
# ---------------------------------------------------------------------------------------------------------------------
def rows_of(xyz, curvature=None):
    xyz = np.asarray(xyz, F32).reshape(-1, 3)
    out = np.zeros((len(xyz), 12), F32)
    out[:, :3] = xyz
    out[:, 4:7] = (0.0, 0.0, 1.0)
    out[:, 8] = np.arange(len(xyz)) % 256
    out[:, 9] = 0.5 if curvature is None else np.asarray(curvature, F32)
    return out


def up(v):
    return np.nextafter(F32(v), F32(np.inf))


def down(v):
    return np.nextafter(F32(v), F32(-np.inf))


def scan_like(n, rng, timestamps=True):
    """a spinning-LiDAR-shaped scan: 64 rings out to 80 m, curvature = the point's time in a 100 ms sweep (ms)"""
    az = np.sort(rng.uniform(-np.pi, np.pi, n))
    el = rng.uniform(-0.43, 0.05, n)
    rg = rng.uniform(2.0, 80.0, n)
    xyz = np.stack([rg * np.cos(el) * np.cos(az), rg * np.cos(el) * np.sin(az), rg * np.sin(el)], 1)
    t = (az + np.pi) / (2 * np.pi) * 100.0 if timestamps else np.zeros(n)
    return rows_of(xyz, t)


def geometry_cloud(rng):
    """the adversarial geometry: origin, axes, +-pi azimuths (signed zeros), straight up / down, non-finite rows"""
    special = [[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [-1, -0.0, 0], [-1, 0.0, 0], [-0.0, 0, 0],
               [0, 0, 5], [0, 0, -5], [3, 4, 0], [-3, -4, 12], [1e-30, 1e-30, 1e-30], [1e20, -1e20, 1e19],
               [np.nan, 1, 1], [1, np.inf, 0], [-np.inf, 0, 0], [2, 2, np.nan]]
    return rows_of(np.concatenate([np.array(special, np.float64), rng.uniform(-60, 60, (3000, 3))]))


def scanner_cloud():
    """points exactly on, and one float either side of, 1.75^2 and 20^2 (on the x axis: dis_square = x*x exactly) and
    the two z thresholds of approx_scanner_height 2, underground_thre -7 (z_min -6, z_min_min -9), plus non-finite rows"""
    pts = []
    for r in (F32(1.75), up(1.75), down(1.75), F32(20.0), up(20.0), down(20.0), F32(10.0), F32(30.0)):
        for z in (F32(-6.0), up(-6.0), down(-6.0), F32(-9.0), up(-9.0), down(-9.0), F32(0.0), F32(-20.0)):
            pts += [[r, 0.0, z], [0.0, -r, z]]
    pts += [[0, 0, 0], [np.nan, 30, 0], [30, 0, np.nan], [np.inf, 0, 0], [5, 5, -np.inf]]
    return rows_of(np.array(pts, np.float64))


def timestamp_clouds(rng):
    """(name, rows, duration_ms): curvature = timestamps in ms"""
    base = rng.uniform(0.0, 100.0, 400).astype(F32)
    out = []
    out.append(("span_above", rows_of(rng.uniform(-9, 9, (400, 3)), base), 100.0))  # span ~100 > 75: ratio by 100
    out.append(("span_below", rows_of(rng.uniform(-9, 9, (400, 3)), base * F32(0.5)), 100.0))  # ~50 < 75: the span
    out.append(("span_at_075", rows_of(rng.uniform(-9, 9, (3, 3)), [10.0, 85.0, 40.0]), 100.0))  # exactly 75
    out.append(("all_equal", rows_of(rng.uniform(-9, 9, (50, 3)), np.full(50, 42.0)), 100.0))  # 0 / 0: NaN
    for where in ("first", "middle", "last"):
        c = base.copy()
        c[{"first": 0, "middle": 200, "last": 399}[where]] = np.nan
        out.append((f"nan_{where}", rows_of(rng.uniform(-9, 9, (400, 3)), c), 100.0))
    c = base.copy()
    c[[17, 250]] = np.nan
    out.append(("nan_twice", rows_of(rng.uniform(-9, 9, (400, 3)), c), 100.0))
    out.append(("signed_zeros", rows_of(rng.uniform(-9, 9, (6, 3)), [0.0, -0.0, 0.0, -0.0, 0.0, -0.0]), 100.0))
    out.append(("zero_tie", rows_of(rng.uniform(-9, 9, (3, 3)), [-5.0, 0.0, -0.0]), 100.0))  # last = the later zero
    out.append(("infinite", rows_of(rng.uniform(-9, 9, (5, 3)), [3.0, np.inf, 5.0, -np.inf, 4.0]), 100.0))
    out.append(("all_minus_inf", rows_of(rng.uniform(-9, 9, (3, 3)), [-np.inf] * 3), 100.0))
    out.append(("one_point", rows_of([[1, 2, 3]], [7.0]), 100.0))
    out.append(("empty", rows_of(np.zeros((0, 3))), 100.0))
    out.append(("scan", scan_like(5000, rng), 100.0))
    return out


def motion_clouds(rng):
    """(name, rows, thre): curvature = timestamp ratios, exactly 0, 1, +-thre, 1 - thre and one float off each"""
    thre = F32(0.05)
    special = [0.0, -0.0, 1.0, up(0.0), down(0.0), up(1.0), down(1.0), thre, up(thre), down(thre), -thre,
               F32(1.0 - 0.05), up(F32(1.0 - 0.05)), down(F32(1.0 - 0.05)), 0.5, np.nan, np.inf]
    s = np.concatenate([np.array(special, F32), rng.uniform(0, 1, 2000).astype(F32)])
    rows = rows_of(rng.uniform(-50, 50, (len(s), 3)), s)
    return [("special_thre0", rows, 0.0), ("special_thre", rows, float(thre)), ("negative_thre", rows, -0.05),
            ("one_point", rows_of([[4, -2, 1]], [0.25]), 0.0), ("empty", rows_of(np.zeros((0, 3))), 0.0)]


def rotation(axis, angle, t=(0.0, 0.0, 0.0)):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K
    T[:3, 3] = t
    return T


def transforms():
    """identity; near-identity (|q.w| >= 1 - eps: the linear slerp branch); a small motion; a rotation whose quaternion
    has a negative w (Eigen's trace <= 0 branch)"""
    Ts = {"identity": np.eye(4), "near_identity": rotation((0.3, -1, 0.2), 1e-9, (0.5, 0.0, 0.0)),
          "small": rotation((0.1, 0.2, 1.0), 0.04, (1.2, -0.3, 0.05))}
    for k in range(100):
        T = rotation(np.random.default_rng(k).normal(size=3), 2.6, (0.3, 0.2, -0.1))
        if np_quaternion(T)[3] < 0:
            Ts["negative_w"] = T
            break
    return Ts


TRANSFORMS = transforms()
VERTICAL_CASES = [(0.0, False), (180.0, False), (200.0, False), (0.5, True), (-1.3, False), (0.7, False), (2.0, False)]
TS_CLOUDS = timestamp_clouds(np.random.default_rng(11))
MOTION_CLOUDS = motion_clouds(np.random.default_rng(12))


# ---------------------------------------------------------------------------------------------------------------------
# the CPU restatement against numpy
# ---------------------------------------------------------------------------------------------------------------------
def test_transforms_cover_the_slerp_branches():
    assert abs(np_quaternion(TRANSFORMS["near_identity"])[3]) >= 1 - np.finfo(np.float64).eps
    assert np_quaternion(TRANSFORMS["negative_w"])[3] < 0


@pytest.mark.parametrize("var,inverse_z", VERTICAL_CASES)
def test_vertical_calibration_equals_numpy(var, inverse_z):
    rows = geometry_cloud(np.random.default_rng(3))
    got, ok = orc_vertical(rows, var, inverse_z)
    exp, eok = np_vertical(rows, var, inverse_z)
    assert ok == eok
    if var == 0 or var >= 180 or inverse_z:
        assert_rows_equal(got, exp, "vertical")
    else:
        assert_rows_close(got, exp, f"vertical {var}")
        assert np.isnan(got[0, :3]).all()  # the origin: 0 / 0
    for n in (0, 1):
        g, _ = orc_vertical(rows[:n], var, inverse_z)
        assert_rows_close(g, np_vertical(rows[:n], var, inverse_z)[0], "vertical small")


@pytest.mark.parametrize("name,rows,duration", TS_CLOUDS, ids=[c[0] for c in TS_CLOUDS])
def test_timestamp_ratio_equals_numpy(name, rows, duration):
    got = orc_ratio(rows, True, duration_ms=duration)
    assert_rows_equal(got, np_ratio(rows, True, duration_ms=duration), name)
    assert_rows_equal(orc_ratio(rows, True, duration_ms=duration, threads=1), got, name)


def test_timestamp_semantics():
    d = dict((c[0], c[1]) for c in TS_CLOUDS)
    assert np.isnan(orc_ratio(d["all_equal"], True)[:, 9]).all()
    assert np.isnan(orc_ratio(d["nan_last"], True)[:, 9]).all()  # last = first = NaN
    r = np.delete(orc_ratio(d["nan_middle"], True)[:, 9], 200)  # the NaN point itself stays NaN
    assert np.isfinite(r).all() and r.min() >= 0 and r.max() <= 1  # the suffix sets last / first; the rest clamps
    # signed zeros: the later point wins each tie, and the ratio keeps the sign of last - curvature
    z = orc_ratio(d["signed_zeros"], True)[:, 9]
    assert np.isnan(z).all()
    # [-5, 0, -0]: last = -0 (the later of the tied zeros), so the point at +0 gets (-0 - 0) / 5 = -0
    r = orc_ratio(d["zero_tie"], True)[:, 9]
    assert r.view(np.uint32).tolist() == np.array([1.0, -0.0, 0.0], F32).view(np.uint32).tolist()


@pytest.mark.parametrize("begin", [180.0, 90.0, 270.0, 0.0])
def test_azimuth_ratio_equals_numpy(begin):
    for rows in (geometry_cloud(np.random.default_rng(4)), scan_like(4000, np.random.default_rng(5), False)):
        assert_azimuth_ratio(orc_ratio(rows, False, begin), rows, begin, f"azimuth {begin}")


@pytest.mark.parametrize("tname", sorted(TRANSFORMS))
@pytest.mark.parametrize("name,rows,thre", MOTION_CLOUDS, ids=[c[0] for c in MOTION_CLOUDS])
def test_motion_compensation_equals_numpy(tname, name, rows, thre):
    T = TRANSFORMS[tname]
    got = orc_motion(rows, T, thre)
    exp = np_motion(rows, T, thre)
    if tname in ("identity", "near_identity"):  # no transcendental function runs
        assert_rows_equal(got, exp, name)
    else:
        assert_rows_close(got, exp, f"motion {tname} {name}")
    # the skip decision: rows outside [thre, 1 - thre] are untouched
    c = rows[:, 9]
    skip = (c < F32(thre)) | (c.astype(np.float64) > 1.0 - float(F32(thre)))
    assert_rows_equal(got[skip], rows[skip], "skipped")


@pytest.mark.parametrize("tname", sorted(TRANSFORMS))
def test_motion_compensation_equals_the_oracles_own(tname):
    rows = MOTION_CLOUDS[0][1]
    r, p = _rows(rows)
    Td = np.ascontiguousarray(TRANSFORMS[tname], np.float64).reshape(16)
    rawscan_oracle_lib().orc_oracle_motion_compensate(p, len(r), Td.ctypes.data_as(C.POINTER(C.c_double)))
    assert_rows_equal(orc_motion(rows, TRANSFORMS[tname], 0.0), r, tname)


@pytest.mark.parametrize("keypoints", [False, True])
def test_batch_equals_one_cloud_at_a_time(keypoints):
    rng = np.random.default_rng(9)
    clouds = [rows_of(rng.uniform(-30, 30, (n, 3)), rng.uniform(0, 1, n)) for n in (300, 0, 50, 1, 700, 20)]
    T = TRANSFORMS["small"]
    got = orc_batch_motion(clouds, T, keypoints)
    for k, (g, c) in enumerate(zip(got, clouds)):
        assert_rows_equal(g, orc_motion(c, T, 0.0) if (k < 5 or keypoints) else c, f"cloud {k}")


@pytest.mark.parametrize("h,u", [(2.0, -7.0), (1.7, -5.0), (0.0, 0.0)])
def test_scanner_filter_equals_numpy(h, u):
    for rows in (scanner_cloud(), geometry_cloud(np.random.default_rng(6)), scan_like(3000, np.random.default_rng(7))):
        assert_rows_equal(orc_scanner_filter(rows, h, u), np_scanner_filter(rows, h, u), f"scanner {h} {u}")


def test_scanner_filter_boundaries():
    rows = scanner_cloud()
    kept = orc_scanner_filter(rows, 2.0, -7.0)
    keyed = {tuple(r[:3].view(np.uint32)) for r in kept}

    def has(x, y, z):
        return tuple(np.array([x, y, z], F32).view(np.uint32)) in keyed

    assert not has(1.75, 0.0, 0.0) and has(up(1.75), 0.0, 0.0)  # strictly outside the self ring
    assert not has(30.0, 0.0, -9.0) and has(30.0, 0.0, up(-9.0))  # strictly above z_min_min everywhere
    assert not has(20.0, 0.0, -6.0) and has(up(20.0), 0.0, -6.0) and has(20.0, 0.0, up(-6.0))  # ghosts within 20 m
    assert not np.isnan(kept[:, :3]).any() and len(orc_scanner_filter(rows[:0])) == 0


# ---------------------------------------------------------------------------------------------------------------------
# the drop-in CFilter: test/mulls_slam.cpp:404-428 and :707-711 against the stand-in headers
# ---------------------------------------------------------------------------------------------------------------------
def build_rawscan_caller(td):
    libdir = os.path.join(ROOT, "mulls_b200", "csrc")
    exe = os.path.join(td, "rawscan_caller")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-I", os.path.join(ROOT, "include", "dropin"),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "stubs", "ref"),
                           "-I", os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests", "stubs", "rawscan_caller.cpp"),
                           "-o", exe, "-L", libdir, "-lmulls_b200", f"-Wl,-rpath,{libdir}"])
    return exe


def test_dropin_rawscan_caller_compiles_and_links():
    """Without a GPU every call reports the missing device and leaves its clouds as they were."""
    import torch

    with tempfile.TemporaryDirectory() as td:
        exe = build_rawscan_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "rawscan drop-in compiled and linked" in out.stdout and "failures 0" in out.stdout, out.stdout
    if not torch.cuda.is_available():
        assert "ran on a device: 0" in out.stdout
