"""CPU checks of the keypoint non-maximum suppression (CFilter::non_max_suppress, the in-place overload,
cfilter.hpp:1183-1240, with the readings abi.h states for mulls_non_max_suppress):
- the CPU restatement (tests/harness/nms_oracle.cpp, candidates from the oracle's kd-tree) against an independent numpy
  restatement (brute force, or scipy cKDTree candidates re-checked with the float distance at large sizes), index for
  index, on adversarial clouds;
- the drop-in CFilter replays test/mulls_reg.cpp:145-149 and the in-place overload's two call forms against the
  stand-in headers.
The clouds (CASES) are shared with tests/test_gpu_nms.py."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest
from scipy.spatial import cKDTree

from mulls_b200 import abi
from test_sor import build_sor_caller

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


# ---------------------------------------------------------------------------------------------------------------------
# the independent restatement
# ---------------------------------------------------------------------------------------------------------------------
def flann_d2(p, q):
    """FLANN L2_Simple<float>: ((dx*dx + dy*dy) + dz*dz) in float32, broadcast over the leading axes."""
    with np.errstate(over="ignore", invalid="ignore"):
        d = (np.asarray(q, F32) - np.asarray(p, F32)).astype(F32)
        return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def score_order(rows):
    """descending normal[3]; equal scores (+0 == -0) in input order; NaN after every number, in input order"""
    s = np.asarray(rows, F32)[:, 7].astype(np.float64)
    nan = np.isnan(s)
    neg = np.where(nan, 0.0, -s) + 0.0  # + 0.0 turns -0 into +0
    return np.lexsort((np.arange(len(s)), neg, nan))


def np_nms(rows, radius):
    """(kept input indices in order, performed) of cfilter.hpp:1183-1240"""
    rows = np.asarray(rows, F32)
    n = len(rows)
    if n < 10:
        return np.zeros(0, np.int32), False
    order = score_order(rows)
    P = rows[order, :3]
    with np.errstate(over="ignore"):
        r2 = F32(np.float64(F32(radius)) * np.float64(F32(radius)))
    fin = np.isfinite(P).all(1)
    visited = np.zeros(n, bool)
    kept = []
    big = n > 6000
    if big and r2 > 0 and fin.any():
        fidx = np.flatnonzero(fin)
        tree = cKDTree(P[fin].astype(np.float64))
        rad = float(np.sqrt(np.float64(r2))) * (1 + 1e-4) + 1e-30
        lists = tree.query_ball_point(P[fin].astype(np.float64), rad, workers=-1)
        cand = np.full(n, None, object)
        cand[fidx] = [fidx[np.asarray(c, np.int64)] for c in lists]
    for i in range(n):
        if visited[i]:
            continue
        kept.append(order[i])
        visited[i] = True
        if not (r2 > 0) or not fin[i]:
            continue
        if big:
            c = cand[i]
            visited[c[flann_d2(P[i], P[c]) < r2]] = True
        else:
            visited |= flann_d2(P[i], P) < r2
    return np.asarray(kept, np.int32), True


# ---------------------------------------------------------------------------------------------------------------------
# the CPU restatement on the oracle's kd-tree (tests/harness/nms_oracle.cpp), the checker of the device path
# ---------------------------------------------------------------------------------------------------------------------
_LIBS = {}


def nms_oracle_lib(out_dir=None):
    out_dir = out_dir or os.path.join(ROOT, "tests", "harness", "_build")
    if out_dir in _LIBS:
        return _LIBS[out_dir]
    src = os.path.join(ROOT, "tests", "harness", "nms_oracle.cpp")
    out = os.path.join(out_dir, "libnms_oracle.so")
    deps = [src, os.path.join(ROOT, "oracle", "mulls_oracle.cpp"), os.path.join(ROOT, "include", "mulls_b200", "abi.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(out_dir, exist_ok=True)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        subprocess.check_call([cxx, "-O3", "-fPIC", "-fopenmp", "-ffp-contract=off", "-std=c++17", "-w", "-shared", "-o", out, src])
    lb = C.CDLL(out)
    lb.orc_non_max_suppress.restype = C.c_int
    lb.orc_non_max_suppress.argtypes = [abi.CloudView, C.c_float, C.POINTER(C.c_int32), C.POINTER(C.c_size_t), C.POINTER(C.c_int)]
    _LIBS[out_dir] = lb
    return lb


def oracle_nms(rows, radius, lib_dir=None):
    """CFilter::non_max_suppress on the CPU: (kept input indices in order, performed)"""
    cloud = abi.as_aos48(rows)
    idx = np.zeros(max(len(cloud), 1), np.int32)
    n, performed = C.c_size_t(0), C.c_int(0)
    rc = nms_oracle_lib(lib_dir).orc_non_max_suppress(abi.cloud_view(cloud), float(radius), idx.ctypes.data_as(C.POINTER(C.c_int32)),
                                                      C.byref(n), C.byref(performed))
    assert rc == 0
    return idx[: n.value].copy(), bool(performed.value)


# ---------------------------------------------------------------------------------------------------------------------
# the clouds (shared with tests/test_gpu_nms.py)
# ---------------------------------------------------------------------------------------------------------------------
def rows_of(xyz, score):
    xyz = np.asarray(xyz, F32)
    out = np.zeros((len(xyz), 12), F32)
    out[:, :3] = xyz
    out[:, 4:7] = (0.0, 0.0, 1.0)
    out[:, 7] = score
    out[:, 8] = np.arange(len(xyz)) % 256
    return out


def box(rng, n, edge, radius=0.25):
    return rows_of(rng.uniform(-edge, edge, (n, 3)), rng.uniform(0, 1, n)), radius


def boundary_pairs():
    """pairs whose float distance is exactly r2 (kept apart) and one float inside it (suppressed), at r = 0.3, whose
    square (0.09) is not a float; the pairs sit 10 m apart, each with the higher score first"""
    r = F32(0.3)
    r2 = F32(np.float64(r) * np.float64(r))
    xs, scores = [], []
    at = inside = None
    d = F32(r)
    for _ in range(64):  # walk to the float d whose flann distance is exactly r2
        dd = flann_d2(np.zeros(3, F32), np.array([d, 0, 0], F32))
        if dd == r2:
            at = d
            break
        d = np.nextafter(d, F32(0) if dd > r2 else F32(1), dtype=F32)
    assert at is not None
    inside = np.nextafter(at, F32(0), dtype=F32)
    assert flann_d2(np.zeros(3, F32), np.array([inside, 0, 0], F32)) < r2
    for k in range(12):
        base = np.array([0.0, 10.0 * k, -2.0], F32)  # x = 0: the x difference is the offset itself
        off = at if k % 2 == 0 else inside
        xs += [base, base + np.array([off, 0, 0], F32)]
        scores += [2.0 + k, 1.0 + k]
    return rows_of(np.array(xs, F32), np.array(scores, F32)), float(r)


def chain_line(n, radius, rng, descending=True):
    """points on a line at 0.75 r: with scores falling along it, a suppresses b, so c survives; n > 1024 puts the
    chain across the chunk boundaries"""
    x = np.arange(n, dtype=np.float64) * 0.75 * radius
    xyz = np.stack([x, np.zeros(n), np.zeros(n)], 1)
    score = np.linspace(1, 0, n) if descending else rng.uniform(0, 1, n)
    perm = rng.permutation(n)
    return rows_of(xyz[perm], score[perm].astype(F32)), radius


def lattice(spacing, radius, rng, m=14):
    ax = np.arange(m, dtype=F32) * F32(spacing)
    g = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    return rows_of(g[rng.permutation(len(g))], rng.uniform(0, 1, len(g))), radius


def special_scores(rng, n):
    s = rng.uniform(-1, 1, n).astype(F32)
    pick = rng.integers(0, 6, n)
    s[pick == 0] = 0.0
    s[pick == 1] = -0.0
    s[pick == 2] = np.nan
    s[pick == 3] = np.inf
    s[pick == 4] = -np.inf
    return s


def nonfinite_coords(rng):
    rows, r = box(rng, 3000, 3.0)
    k = rng.choice(3000, 200, replace=False)
    vals = np.array([np.nan, np.inf, -np.inf], F32)
    rows[k, rng.integers(0, 3, 200)] = vals[rng.integers(0, 3, 200)]
    rows[k[:20], :3] = np.nan
    return rows, r


def huge_cluster(rng, centre, n=3000, steps=6):
    """n points on the floats next to `centre` (+-steps ulps per axis) and at -centre: distances 0, one ulp (7.6e22 at
    1e30) or an overflow to inf"""
    c = F32(centre)
    ulps = [c]
    for _ in range(steps):
        ulps.append(np.nextafter(ulps[-1], F32(np.inf), dtype=F32))
    lo = [c]
    for _ in range(steps):
        lo.append(np.nextafter(lo[-1], F32(0), dtype=F32))
    vals = np.array(sorted(set(ulps + lo)), F32)
    xyz = vals[rng.integers(0, len(vals), (n, 3))]
    flip = rng.uniform(0, 1, n) < 0.2
    xyz[flip] = -xyz[flip]
    return rows_of(xyz, rng.uniform(0, 1, n))


def make_cases():
    rng = np.random.default_rng(20261017)
    cases = []
    for n in (9, 10):
        rows, r = box(rng, n, 0.3)
        cases.append((f"n{n}", rows, r))
    rows, _ = box(rng, 2000, 2.0)
    rows[:, 7] = 0.5
    cases.append(("all_equal_scores", rows, 0.25))
    rows, _ = box(rng, 3000, 3.0)
    rows[:, 7] = special_scores(rng, 3000)
    cases.append(("zero_nan_inf_scores", rows, 0.25))
    rows, _ = box(rng, 40, 1.0)
    rows[:, 7] = special_scores(rng, 40)
    cases.append(("zero_nan_inf_scores_small", rows, 0.25))
    cases.append(("boundary_pairs",) + boundary_pairs())
    cases.append(("chain_600",) + chain_line(600, 0.25, rng))
    cases.append(("chain_3000_chunks",) + chain_line(3000, 0.25, rng))
    cases.append(("chain_3000_random_scores",) + chain_line(3000, 0.25, rng, descending=False))
    xyz = rng.normal(0, 0.03, (2500, 3))
    cases.append(("dense_cluster", rows_of(xyz, rng.uniform(0, 1, 2500)), 0.25))
    cases.append(("lattice_at_r",) + lattice(0.25, 0.25, rng))
    cases.append(("lattice_below_r",) + lattice(np.nextafter(F32(0.25), F32(0), dtype=F32), 0.25, rng))
    cases.append(("nonfinite_coords",) + nonfinite_coords(rng))
    cases.append(("cluster_1e30", huge_cluster(rng, 1e30), 0.25))
    cases.append(("cluster_1e30_r1e23", huge_cluster(rng, 1e30), 1e23))
    cases.append(("cluster_3e38", huge_cluster(rng, 3e38), 0.25))
    cases.append(("cluster_3e38_r1e19", huge_cluster(rng, 3e38), 1e19))
    mixed, _ = box(rng, 2000, 2.0)
    mixed = np.concatenate([mixed, huge_cluster(rng, 1e30, 600), huge_cluster(rng, 3e38, 600)])
    cases.append(("mixed_scales", mixed[rng.permutation(len(mixed))], 0.25))
    for r in (-0.3, 0.0, float("nan")):
        rows, _ = box(rng, 3000, 2.0)
        cases.append((f"radius_{r}", rows, r))
    for n in (10, 1023, 1024, 1025, 5000, 120000):
        edge = 0.6 * (n / 1000.0) ** (1 / 3)  # about 8 points per r^3 box
        rows, r = box(rng, n, edge)
        cases.append((f"size_{n}", rows, r))
    return cases


CASES = make_cases()


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,rows,radius", CASES, ids=[c[0] for c in CASES])
def test_restatement_equals_numpy(name, rows, radius):
    got, performed = oracle_nms(rows, radius)
    exp, exp_performed = np_nms(rows, radius)
    assert performed == exp_performed
    assert np.array_equal(got, exp), (len(got), len(exp))


def test_cases_mean_what_they_say():
    by = {c[0]: c for c in CASES}
    kept, performed = oracle_nms(by["n9"][1], 0.25)
    assert not performed and len(kept) == 0
    kept, _ = oracle_nms(*by["boundary_pairs"][1:])
    assert len(kept) == 12 * 2 - 6  # the six pairs at exactly r2 keep both points, the six inside keep one
    kept, _ = oracle_nms(*by["chain_3000_chunks"][1:])
    assert len(kept) == 1500  # every second point of the line
    assert len(oracle_nms(*by["dense_cluster"][1:])[0]) == 1
    for r in ("radius_0.0", "radius_nan"):
        assert len(oracle_nms(*by[r][1:])[0]) == 3000
    a = oracle_nms(by["radius_-0.3"][1], -0.3)[0]
    assert np.array_equal(a, oracle_nms(by["radius_-0.3"][1], 0.3)[0])
    rows = by["nonfinite_coords"][1]
    kept = oracle_nms(rows, 0.25)[0]
    assert set(np.flatnonzero(~np.isfinite(rows[:, :3]).all(1))) <= set(kept.tolist())
    assert len(oracle_nms(*by["size_1025"][1:])[0]) < 1025


def test_sorted_order_ignores_the_sign_of_zero_and_puts_nan_last():
    rows = rows_of(np.arange(12)[:, None] * np.array([[10.0, 0, 0]]), np.array(
        [np.nan, -0.0, 1.0, 0.0, np.nan, -np.inf, np.inf, -0.0, 2.0, 0.0, np.nan, -1.0], F32))
    kept, performed = oracle_nms(rows, 0.5)
    assert performed
    assert kept.tolist() == [6, 8, 2, 1, 3, 7, 9, 11, 5, 0, 4, 10]


# ---------------------------------------------------------------------------------------------------------------------
# the drop-in (include/dropin/cfilter.hpp) against the stand-in headers
# ---------------------------------------------------------------------------------------------------------------------
def build_nms_caller(td):
    libdir = os.path.join(ROOT, "mulls_b200", "csrc")
    exe = os.path.join(td, "nms_caller")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-I", os.path.join(ROOT, "include", "dropin"),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "stubs", "nms_ref"),
                           "-I", os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests", "stubs", "nms_caller.cpp"),
                           "-o", exe, "-L", libdir, "-lmulls_b200", f"-Wl,-rpath,{libdir}"])
    return exe


def test_dropin_nms_compiles_and_links():
    """Without a GPU both calls report the missing device and leave the clouds alone; the prebuilt-tree form and the
    overloads of :1243 and :1314 reach the reference members either way. The unchanged callers of the other stand-in
    (tests/stubs/ref, which declares no non_max_suppress) still compile against the drop-in."""
    import torch

    with tempfile.TemporaryDirectory() as td:
        exe = build_nms_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
        build_sor_caller(td)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "nms drop-in compiled and linked" in out.stdout and "failures 0" in out.stdout
    if not torch.cuda.is_available():
        assert "ran on a device: 0" in out.stdout
