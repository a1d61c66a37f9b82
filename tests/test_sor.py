"""CPU checks of the statistical outlier filter (CFilter::sor_filter, cfilter.hpp:203-247 -> pcl::StatisticalOutlierRemoval,
PCL 1.10 applyFilterIndices as restated in SURVEY Appendix B item 10):
- the CPU restatement (tests/harness/sor_oracle.cpp, on the oracle's kd-tree) against an independent numpy / scipy
  restatement, bit for bit;
- the templated k-nearest search of search_core.cuh (knn_search, KnnList<kCap>), which k_search_shoot and k_sor_dist run
  on the device, instantiated on the host by tests/harness/knn_host.cu, against a brute-force scan;
- the drop-in CFilter replays test/mulls_slam.cpp:1008-1009 and both overloads against the stand-in headers."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest
from scipy.spatial import cKDTree

from mulls_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------------------------------
# the independent restatement
# ---------------------------------------------------------------------------------------------------------------------
def flann_d2(p, q):
    """FLANN L2_Simple<float>: ((dx*dx + dy*dy) + dz*dz) in float32, broadcast over the leading axes."""
    d = (q - p).astype(np.float32)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def np_sor(rows, mean_k, n_std):
    """(keep bool[n], distances float32[n], stats dict) or None when the cloud has at most mean_k finite points."""
    xyz = np.asarray(rows, np.float32)[:, :3]
    fin = np.isfinite(xyz).all(1)
    P = xyz[fin]
    if len(P) <= mean_k:
        return None
    tree = cKDTree(P.astype(np.float64))
    want = mean_k + 1
    margin = 8
    while True:  # extra neighbours until the shell past the (mean_k+1)-th is strictly farther: ties all inside
        kq = min(len(P), want + margin)
        dd, idx = tree.query(P.astype(np.float64), k=kq)
        dd, idx = dd.reshape(len(P), kq), idx.reshape(len(P), kq)
        if kq == len(P) or np.all(dd[:, -1] > dd[:, want - 1] * (1 + 1e-5) + 1e-30):
            break
        margin *= 4
    d2 = np.sort(flann_d2(P[:, None, :], P[idx]), axis=1)[:, :want]
    # sum of sqrt((double) d2) over positions 1..mean_k, sequential along the row
    sums = np.cumsum(np.sqrt(d2[:, 1:].astype(np.float64)), axis=1)[:, -1]
    distances = np.zeros(len(xyz), np.float32)
    distances[fin] = (sums / mean_k).astype(np.float32)
    s = np.cumsum(distances.astype(np.float64))[-1]
    sq = np.cumsum((distances * distances).astype(np.float64))[-1]  # the float product, widened
    valid = float(len(P))
    mean = s / valid
    variance = (sq - s * s / valid) / (valid - 1)
    with np.errstate(invalid="ignore"):
        stddev = np.sqrt(np.float64(variance))
    thr = mean + n_std * stddev
    keep = ~(distances.astype(np.float64) > thr)
    return keep, distances, {"mean": mean, "stddev": float(stddev), "threshold": float(thr), "n_valid": len(P),
                             "n_kept": int(keep.sum())}


def same_double(a, b):
    return np.float64(a).tobytes() == np.float64(b).tobytes()


def assert_same_result(got, exp):
    gk, gd, gs = got
    ek, ed, es = exp
    assert np.array_equal(gd.view(np.uint32), ed.view(np.uint32)), np.flatnonzero(gd.view(np.uint32) != ed.view(np.uint32))[:10]
    for k in ("mean", "stddev", "threshold"):
        assert same_double(gs[k], es[k]), (k, gs[k], es[k])
    assert gs["n_valid"] == es["n_valid"] and gs["n_kept"] == es["n_kept"]
    assert np.array_equal(gk, ek)


# ---------------------------------------------------------------------------------------------------------------------
# the CPU restatement on the oracle's kd-tree (tests/harness/sor_oracle.cpp), the checker of the device path
# ---------------------------------------------------------------------------------------------------------------------
_SOR_LIBS = {}


def sor_oracle_lib(out_dir=None):
    """Build (when a source is newer) and load tests/harness/sor_oracle.cpp; out_dir: where the library goes
    (default tests/harness/_build)."""
    out_dir = out_dir or os.path.join(ROOT, "tests", "harness", "_build")
    if out_dir in _SOR_LIBS:
        return _SOR_LIBS[out_dir]
    src = os.path.join(ROOT, "tests", "harness", "sor_oracle.cpp")
    out = os.path.join(out_dir, "libsor_oracle.so")
    deps = [src, os.path.join(ROOT, "oracle", "mulls_oracle.cpp"), os.path.join(ROOT, "include", "mulls_b200", "abi.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(out_dir, exist_ok=True)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        subprocess.check_call([cxx, "-O3", "-fPIC", "-fopenmp", "-ffp-contract=off", "-std=c++17", "-w", "-shared", "-o", out, src])
    lb = C.CDLL(out)
    lb.orc_sor_filter.restype = C.c_int
    lb.orc_sor_filter.argtypes = [abi.CloudView, C.c_int, C.c_double, C.POINTER(C.c_uint8), C.POINTER(C.c_float),
                                  C.POINTER(abi.SorStats), C.c_int]
    lb.orc_num_threads.restype = C.c_int
    _SOR_LIBS[out_dir] = lb
    return lb


def oracle_sor_filter(rows, mean_k, n_std, threads=0, lib_dir=None):
    """CFilter::sor_filter on the CPU: (keep bool[n], distances float32[n], stats dict), or the MULLS_E_* code when the
    call is refused. threads: 0 = every core, 1 = reference-shaped."""
    cloud = abi.as_aos48(rows)
    n = len(cloud)
    bits = np.zeros(max((n + 7) // 8, 1), np.uint8)
    dist = np.zeros(max(n, 1), np.float32)
    st = abi.SorStats()
    rc = sor_oracle_lib(lib_dir).orc_sor_filter(abi.cloud_view(cloud), int(mean_k), float(n_std),
                                                bits.ctypes.data_as(C.POINTER(C.c_uint8)),
                                                dist.ctypes.data_as(C.POINTER(C.c_float)), C.byref(st), int(threads))
    if rc != 0:
        return rc
    keep = np.unpackbits(bits, bitorder="little")[:n].astype(bool)
    return keep, dist[:n], {k: getattr(st, k) for k, _ in abi.SorStats._fields_}


# ---------------------------------------------------------------------------------------------------------------------
# the clouds (shared with tests/test_gpu_sor.py)
# ---------------------------------------------------------------------------------------------------------------------
def rows_of(xyz):
    xyz = np.asarray(xyz, np.float32)
    out = np.zeros((len(xyz), 12), np.float32)
    out[:, :3] = xyz
    out[:, 4:7] = (0.0, 0.0, 1.0)
    out[:, 8] = np.arange(len(xyz)) % 256  # intensity: any payload, carried along with the row
    return out


def lattice_cloud(rng):
    """shuffled lattice of spacing 0.375 (exact in float, and so are the differences and distances): for mean_k = 1
    every mean distance is the same, the variance is exactly 0 and the threshold is the mean"""
    ax = np.arange(14, dtype=np.float32) * np.float32(0.375)
    g = np.stack(np.meshgrid(ax, ax, ax[:5], indexing="ij"), -1).reshape(-1, 3)
    return rows_of(g[rng.permutation(len(g))])


def triple_cloud(rng):
    base = rng.uniform(-10, 10, (700, 3)).astype(np.float32)
    return rows_of(np.tile(base, (3, 1))[rng.permutation(2100)])


def cluster_cloud(rng):
    dense = rng.normal(0, 0.4, (3000, 3)) + [2.0, -1.0, 0.5]
    sparse = rng.uniform(-30, 30, (120, 3))
    xyz = np.concatenate([dense, sparse])
    return rows_of(xyz[rng.permutation(len(xyz))])


def far_cloud(rng):
    near = rng.uniform(-20, 20, (2500, 3))
    far = np.array([[4000.0, 10.0, 0.0], [-2500.0, 3000.0, 5.0], [0.0, 0.0, -6000.0], [4000.5, 10.0, 0.0]])
    xyz = np.concatenate([near, far])
    return rows_of(xyz[rng.permutation(len(xyz))])


def nonfinite_cloud(rng):
    xyz = rng.uniform(-5, 5, (1500, 3)).astype(np.float32)
    bad = rng.choice(len(xyz), 60, replace=False)
    vals = np.array([np.nan, np.inf, -np.inf], np.float32)
    for k, i in enumerate(bad):
        xyz[i, k % 3] = vals[(k // 3) % 3]
    return rows_of(xyz)


def minimal_cloud(rng, mean_k):
    """exactly mean_k + 1 finite points, plus a NaN row"""
    xyz = rng.uniform(-1, 1, (mean_k + 2, 3)).astype(np.float32)
    xyz[3, 1] = np.nan
    return rows_of(xyz)


def threshold_cloud(rng):
    """isolated pairs (mean_k = 1: a point's distance is its pair's separation), and an n_std chosen so that the
    threshold is EXACTLY one of the distances d_a while another pair sits exactly one float above it: the point at the
    threshold is kept, the one a float above is removed. Returns (rows, n_std, d_a, d_b)."""
    gx, gy = np.meshgrid(np.arange(55) * 10.0, np.arange(55) * 10.0, indexing="ij")
    n_pairs = gx.size
    # along z. Most separations spread over 0.5 .. 3 m (a variance well above the rounding of PCL's float squares);
    # a third packed into 0.3 mm at 2.5 m, where consecutive floats (2.4e-7 apart) are all taken
    sep = np.where(np.arange(n_pairs) % 3 == 0, rng.uniform(2.5, 2.5003, n_pairs), rng.uniform(0.5, 3.0, n_pairs))
    sep = sep.astype(np.float32)
    a = np.stack([gx.ravel(), gy.ravel(), np.zeros(n_pairs)], 1).astype(np.float32)
    b = np.stack([gx.ravel(), gy.ravel(), sep], 1).astype(np.float32)
    rows = rows_of(np.concatenate([a, b]))
    _, dist, st = np_sor(rows, 1, 0.0)
    u = np.unique(dist)
    up = np.nextafter(u, np.float32(np.inf))
    cand = u[np.isin(up, u)]
    cand = cand[np.argsort(np.abs(cand.astype(np.float64) - st["mean"]))]
    mean, sd = st["mean"], st["stddev"]
    for d_a in cand[:50]:
        target = np.float64(d_a)
        lo, hi = (target - mean) / sd - 1.0, (target - mean) / sd + 1.0
        for _ in range(200):  # bisection over n_std for mean + n_std * sd == d_a exactly
            mid = lo + (hi - lo) / 2
            v = mean + mid * sd
            if v == target:
                return rows, float(mid), d_a, np.nextafter(d_a, np.float32(np.inf))
            if v < target:
                lo = mid
            else:
                hi = mid
            if mid in (lo, hi) and hi - lo <= np.spacing(abs(mid)):
                break
    raise AssertionError("no n_std puts the threshold on a distance")


def cpu_clouds():
    """(name, rows, mean_k, n_std) of the adversarial clouds"""
    out = []
    rng = np.random.default_rng(7)
    out.append(("lattice_k1", lattice_cloud(rng), 1, 2.0))
    out.append(("lattice_k20", lattice_cloud(rng), 20, 1.0))
    out.append(("triple", triple_cloud(rng), 20, 2.0))
    out.append(("triple_k2", triple_cloud(rng), 2, 2.0))
    out.append(("cluster", cluster_cloud(rng), 20, 2.0))
    out.append(("far", far_cloud(rng), 20, 2.0))
    out.append(("nonfinite", nonfinite_cloud(rng), 20, 2.0))
    out.append(("minimal", minimal_cloud(rng, 20), 20, 2.0))
    out.append(("cluster_k50", cluster_cloud(rng), 50, 1.0))
    rows, n_std, _, _ = threshold_cloud(np.random.default_rng(8))
    out.append(("threshold", rows, 1, n_std))
    return out


CLOUDS = cpu_clouds()


@pytest.mark.parametrize("name,rows,mean_k,n_std", CLOUDS, ids=[c[0] for c in CLOUDS])
def test_oracle_equals_numpy_restatement(name, rows, mean_k, n_std):
    exp = np_sor(rows, mean_k, n_std)
    got = oracle_sor_filter(rows, mean_k, n_std)
    assert_same_result(got, exp)
    assert_same_result(oracle_sor_filter(rows, mean_k, n_std, threads=1), exp)  # the sums do not depend on the threads


def test_degenerate_clouds_as_pcl_leaves_them():
    rows = CLOUDS[0][1]
    keep, dist, st = oracle_sor_filter(rows, 1, 2.0)
    assert np.all(dist == dist[0])
    # equal distances: no positive variance (PCL's formula gives 0 here, NaN for a negative rounding); a point at the
    # threshold is kept, and so is every point under a NaN threshold
    assert not (st["stddev"] > 0) and st["threshold"] == st["mean"]
    assert keep.all()
    keep, dist, st = oracle_sor_filter(dict((c[0], c[1]) for c in CLOUDS)["nonfinite"], 20, 2.0)
    xyz = dict((c[0], c[1]) for c in CLOUDS)["nonfinite"][:, :3]
    bad = ~np.isfinite(xyz).all(1)
    assert np.all(dist[bad] == 0) and np.all(keep[bad]) and st["n_valid"] == int((~bad).sum())


def test_point_on_the_threshold_is_kept_and_one_float_above_is_removed():
    rows, n_std, d_a, d_b = threshold_cloud(np.random.default_rng(8))
    keep, dist, st = oracle_sor_filter(rows, 1, n_std)
    assert st["threshold"] == np.float64(d_a)
    assert np.any(dist == d_a) and np.any(dist == d_b)
    assert np.all(keep[dist == d_a]) and not np.any(keep[dist == d_b])


def test_refusals():
    rng = np.random.default_rng(3)
    rows = rows_of(rng.uniform(-1, 1, (21, 3)))
    rows[0, 0] = np.nan  # 20 finite points: not more than mean_k = 20
    assert oracle_sor_filter(rows, 20, 2.0) == abi.E_ARG
    assert oracle_sor_filter(rows, 0, 2.0) == abi.E_ARG
    assert isinstance(oracle_sor_filter(rows, 19, 2.0), tuple)


# ---------------------------------------------------------------------------------------------------------------------
# the templated k-nearest search of search_core.cuh on the host
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def klib():
    src = os.path.join(ROOT, "tests", "harness", "knn_host.cu")
    out = os.path.join(ROOT, "tests", "harness", "_build", "libknn_host.so")
    deps = [src, os.path.join(ROOT, "tests", "harness", "search_host.cu")] + [
        os.path.join(ROOT, "mulls_b200", "csrc", f) for f in ("search_core.cuh", "grid_key.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "-diag-suppress", "20014,20011",
                               "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-o", out, src])
    lb = C.CDLL(out)
    lb.sh_build.restype = C.c_void_p
    lb.sh_build.argtypes = [C.c_void_p, C.c_uint32, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int]
    lb.sh_free.argtypes = [C.c_void_p]
    lb.kh_knn.restype = C.c_int
    lb.kh_knn.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return lb


def cell_size_for(xyz):
    """k_pair_setup: the level-0 cell doubles from 0.125 m until 4092 cells span the extent of the targets"""
    ext = float((xyz.max(0).astype(np.float64) - xyz.min(0).astype(np.float64)).max())
    h0 = 0.125
    while (ext + 8 * h0) * 1.001 > h0 * 4092:
        h0 *= 2
    return h0


def knn_run(lib, tgt, q, cap, k, leaf=32, start_level=5):
    tgt = np.ascontiguousarray(tgt, np.float32)
    q = np.ascontiguousarray(q, np.float32)
    h0 = cell_size_for(tgt)
    origin = (tgt.min(0) - np.float32(2 * h0)).astype(np.float32)
    pts4 = np.ascontiguousarray(np.concatenate([tgt, np.zeros((len(tgt), 1), np.float32)], axis=1))
    G = lib.sh_build(pts4.ctypes.data, len(tgt), float(origin[0]), float(origin[1]), float(origin[2]), h0, 12, leaf)
    idx = np.empty((len(q), k), np.int32)
    d2 = np.empty((len(q), k), np.float32)
    n = np.empty(len(q), np.int32)
    rc = lib.kh_knn(G, q.ctypes.data, len(q), cap, k, start_level, idx.ctypes.data, d2.ctypes.data, n.ctypes.data)
    lib.sh_free(G)
    assert rc == 0
    return idx, d2, n


def knn_brute(tgt, q, k):
    tgt = np.asarray(tgt, np.float32)
    idx = np.empty((len(q), k), np.int64)
    d2 = np.empty((len(q), k), np.float32)
    order_idx = np.arange(len(tgt))
    for i, p in enumerate(np.asarray(q, np.float32)):
        d = flann_d2(p, tgt)
        o = np.lexsort((order_idx, d))[:k]
        idx[i], d2[i] = o, d[o]
    return idx, d2


def knn_clouds():
    rng = np.random.default_rng(41)
    ax = np.arange(20, dtype=np.float32) * np.float32(0.0625)
    lat = np.stack(np.meshgrid(ax, ax, ax[:6], indexing="ij"), -1).reshape(-1, 3)
    lat = lat[rng.permutation(len(lat))]
    lat_q = np.concatenate([lat[:150], lat[150:300] + np.float32(0.03125)])
    dense = np.concatenate([rng.uniform(0, 0.1, (3000, 3)) + 1.0, rng.uniform(-3, 5, (1500, 3)),
                            [[900.0, 0.0, 0.0], [-700.0, 50.0, 3.0]]]).astype(np.float32)
    dense_q = np.concatenate([dense[::40], dense[-2:], rng.uniform(-4, 6, (80, 3))]).astype(np.float32)
    ext = 20000.0
    corners = np.array([[x, y, z] for x in (0, ext) for y in (0, ext) for z in (0, ext)], np.float32)
    wide = np.concatenate([rng.uniform(0, ext, (3000, 3)), corners, corners + 3.0 * (corners < 1) - 3.0 * (corners > 1)]).astype(np.float32)
    wide_q = np.concatenate([wide[::25], corners]).astype(np.float32)
    off = np.array([6000.0, -3000.0, 40.0])
    return [("lattice", lat, lat_q), ("far_outliers", dense, dense_q), ("extent_20km", wide, wide_q),
            ("lattice_6km", (lat + off).astype(np.float32), (lat_q + off).astype(np.float32)),
            ("far_outliers_6km", (dense + off).astype(np.float32), (dense_q + off).astype(np.float32))]


KNN_CLOUDS = knn_clouds()


@pytest.mark.parametrize("name,tgt,q", KNN_CLOUDS, ids=[c[0] for c in KNN_CLOUDS])
@pytest.mark.parametrize("cap,k", [(10, 10), (16, 1), (16, 16), (32, 21), (64, 51), (64, 64)])
def test_knn_core_equals_brute_force(klib, name, tgt, q, cap, k):
    bi, bd = knn_brute(tgt, q, k)
    for leaf, start in ((32, 5), (32, 1), (4, 1)):
        idx, d2, n = knn_run(klib, tgt, q, cap, k, leaf=leaf, start_level=start)
        assert np.all(n == k)
        assert np.array_equal(d2, bd), (leaf, start)
        assert np.array_equal(idx, bi), (leaf, start)


def test_knn_core_with_fewer_targets_than_k(klib):
    tgt = np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0]], np.float32)
    q = np.array([[0.1, 0, 0], [50, 50, 50]], np.float32)
    idx, d2, n = knn_run(klib, tgt, q, 16, 5)
    assert np.all(n == 3)
    assert idx[0, :3].tolist() == [0, 1, 2] and idx[1, :3].tolist() == [2, 1, 0]
    assert np.all(idx[:, 3:] == -1) and np.all(np.isinf(d2[:, 3:]))


# ---------------------------------------------------------------------------------------------------------------------
# the drop-in CFilter: test/mulls_slam.cpp:1008-1009 and both overloads, against the stand-in headers
# ---------------------------------------------------------------------------------------------------------------------
def build_sor_caller(td):
    libdir = os.path.join(ROOT, "mulls_b200", "csrc")
    exe = os.path.join(td, "sor_caller")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-I", os.path.join(ROOT, "include", "dropin"),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "stubs", "ref"),
                           "-I", os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests", "stubs", "sor_caller.cpp"),
                           "-o", exe, "-L", libdir, "-lmulls_b200", f"-Wl,-rpath,{libdir}"])
    return exe


def test_dropin_sor_filter_compiles_and_links():
    """Without a GPU both calls report the missing device, return false and leave the map as it was."""
    import torch

    with tempfile.TemporaryDirectory() as td:
        exe = build_sor_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "sor drop-in compiled and linked" in out.stdout and "failures 0" in out.stdout
    if not torch.cuda.is_available():
        assert "ran on a device: 0" in out.stdout
