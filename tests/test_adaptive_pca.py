"""Distance-adaptive PCA neighbourhoods: get_pc_pca_feature with distance_adaptive_on (include/common/pca.hpp:310-326),
as classify_nground_pts calls it for the SLAM driver (cfilter.hpp:2093, unit_distance 30; test/mulls_slam.cpp:363-377
and :418-428 pass use_distance_adaptive_pca = true).

A query at range dist = sqrt(x*x + y*y + z*z) (float norm, widened) > unit_dist searches the radius
(float)(sqrt(dist / unit_dist) * radius); nearer queries search `radius`. The close / far split of the neighbour lists
and the NMS keep the base radius.

CPU part: the restatement (tests/harness/adaptive_pca_oracle.cpp, which includes the oracle unchanged) against an
independent numpy restatement, neighbour lists exactly; its classification with the flag off against the oracle, bit
for bit. GPU part: mulls_pca_features_adaptive, mulls_classify_nground and mulls_extract_semantic_pts with the flag on
against the restatement, and the drop-in CFilter replaying test/mulls_slam.cpp:418-428."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from mulls_b200 import abi
from oracle import oracle
from test_classify import kitti_params, unground_cloud
from test_ground import params as ground_params
from test_ground import raw_scan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


# ---------------------------------------------------------------------------------------------------------------------
# the independent restatement
# ---------------------------------------------------------------------------------------------------------------------
def np_radius(xyz, radius, unit_dist):
    """pca.hpp:313-320 per point: float32 norm (products and sum in float, the float sqrt), widened; strict `>`;
    (float)(sqrt(dist / unit) * radius) in float64."""
    x = np.asarray(xyz, F32)[:, :3]
    s = (x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2]
    dist = np.sqrt(s).astype(np.float64)
    r = np.full(len(x), F32(radius), F32)
    far = dist > np.float64(F32(unit_dist))
    r[far] = (np.sqrt(dist[far] / np.float64(F32(unit_dist))) * np.float64(F32(radius))).astype(F32)
    return r


def flann_d2(p, q):
    """FLANN L2_Simple<float>: ((dx*dx + dy*dy) + dz*dz) in float32."""
    d = (np.asarray(q, F32) - np.asarray(p, F32)).astype(F32)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def np_neighbours(rows, radius, k, stride, unit_dist):
    """radiusSearch(i, r_i, ..., k) for every stride-th point, brute force: d2 < (float)((double)r*r), sorted by
    (d2, index), at most k. Returns (pt_num int32[n], lists: dict i -> int array)."""
    xyz = np.asarray(rows, F32)[:, :3]
    r = np_radius(xyz, radius, unit_dist) if unit_dist > 0 else np.full(len(xyz), F32(radius), F32)
    r2 = (r.astype(np.float64) * r.astype(np.float64)).astype(F32)
    pt_num = np.zeros(len(xyz), np.int32)
    lists = {}
    for i in range(0, len(xyz), stride):
        d2 = flann_d2(xyz[i], xyz)
        idx = np.flatnonzero(d2 < r2[i])
        order = np.lexsort((idx, d2[idx]))
        sel = idx[order][:k] if k > 0 else idx[order]
        pt_num[i] = len(sel)
        lists[i] = sel
    return pt_num, lists


# ---------------------------------------------------------------------------------------------------------------------
# the CPU restatement (tests/harness/adaptive_pca_oracle.cpp), the checker of the device path
# ---------------------------------------------------------------------------------------------------------------------
_LIB = []


def adaptive_lib():
    """Build (when a source is newer) and load tests/harness/adaptive_pca_oracle.cpp into tests/harness/_build."""
    if _LIB:
        return _LIB[0]
    out_dir = os.path.join(ROOT, "tests", "harness", "_build")
    src = os.path.join(ROOT, "tests", "harness", "adaptive_pca_oracle.cpp")
    out = os.path.join(out_dir, "libadaptive_pca_oracle.so")
    deps = [src, os.path.join(ROOT, "oracle", "mulls_oracle.cpp"), os.path.join(ROOT, "include", "mulls_b200", "abi.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(out_dir, exist_ok=True)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        tmp = out + f".{os.getpid()}.tmp"
        subprocess.check_call([cxx, "-O3", "-fPIC", "-fopenmp", "-ffp-contract=off", "-std=c++17", "-w", "-shared", "-o", tmp, src])
        os.replace(tmp, out)
    lb = C.CDLL(out)
    lb.orc_pca_features_adaptive.restype = C.c_int
    lb.orc_pca_features_adaptive.argtypes = [abi.CloudView, C.c_float, C.c_int, C.c_int, C.c_float, C.POINTER(abi.PcaOut),
                                             C.POINTER(C.c_int32)]
    lb.orc_classify_nground_adaptive.restype = C.c_int
    lb.orc_classify_nground_adaptive.argtypes = [abi.CloudView, C.POINTER(abi.ClassifyParams), C.POINTER(abi.ClassifyOut)]
    _LIB.append(lb)
    return lb


def orc_pca_features_adaptive(cloud, radius, k, stride, unit_dist, want_lists=False):
    """get_pc_pca_feature(..., distance_adaptive_on = unit_dist > 0, unit_dist) on the CPU: as oracle.pca_features,
    plus "nbr" ([n][k] neighbour indices, -1 past pt_num) when want_lists."""
    cloud = abi.as_aos48(cloud)
    n = cloud.shape[0]
    ev, pr, nr = (np.zeros((n, 3), F32) for _ in range(3))
    cnt = np.zeros(n, np.int32)
    nbr = np.full((n, max(k, 1)), -1, np.int32) if want_lists else None
    out = abi.PcaOut(ev.ctypes.data_as(C.POINTER(C.c_float)), pr.ctypes.data_as(C.POINTER(C.c_float)),
                     nr.ctypes.data_as(C.POINTER(C.c_float)), cnt.ctypes.data_as(C.POINTER(C.c_int32)))
    rc = adaptive_lib().orc_pca_features_adaptive(abi.cloud_view(cloud), float(radius), int(k), int(stride), float(unit_dist),
                                                  C.byref(out), nbr.ctypes.data_as(C.POINTER(C.c_int32)) if want_lists else None)
    assert rc == 0, rc
    res = {"eigenvalues": ev, "principal": pr, "normal": nr, "pt_num": cnt}
    if want_lists:
        res["nbr"] = nbr
    return res


def orc_classify_adaptive(cloud, params):
    """classify_nground_pts on the CPU with use_distance_adaptive_pca honoured ({"rc": code} when refused)."""
    return abi.classify_call(adaptive_lib().orc_classify_nground_adaptive, None, cloud, params)


# ---------------------------------------------------------------------------------------------------------------------
# adversarial clouds
# ---------------------------------------------------------------------------------------------------------------------
def _rows(xyz):
    r = np.zeros((len(xyz), 12), F32)
    r[:, :3] = np.asarray(xyz, F32)
    return r


def _shells(center, rng, n, r_lo, r_hi):
    """n points around `center` at distances spread over [r_lo, r_hi]"""
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.asarray(center, np.float64) + d * rng.uniform(r_lo, r_hi, (n, 1))


def cloud_at_unit_range(radius=1.0):
    """queries at range exactly 30 and one float beyond, and at 30.5 / 45 / 90, with neighbours spread over 0.5..2 r"""
    rng = np.random.default_rng(1)
    x30 = F32(30.0)
    centers = [(x30, 0, 0), (np.nextafter(x30, F32(np.inf)), 0.0, 0.0), (0, 0, x30), (0, np.nextafter(x30, F32(np.inf)), 0),
               (30.5, 0, 0), (0, 45, 0), (-90, 0, 0), (10, 10, 0)]
    pts = [np.asarray(centers, np.float64)]
    for c in centers:
        pts.append(_shells(c, rng, 60, 0.3 * radius, 2.2 * radius))
    return _rows(np.concatenate(pts))


def _float_at_squared(r2):
    """a float32 dz with fl(dz*dz) == r2, and the next float below it (fl < r2), or None"""
    z = F32(np.sqrt(np.float64(r2)))
    for _ in range(8):
        z = np.nextafter(z, F32(0))
    for _ in range(16):
        if F32(z * z) == r2:
            below = np.nextafter(z, F32(0))
            assert F32(below * below) < r2
            return z, below
        z = np.nextafter(z, F32(np.inf))
    return None


def cloud_at_adaptive_radius(radius=1.0, unit=30.0):
    """a neighbour exactly at the query's adaptive squared radius (excluded: strict <) and one float inside (kept)"""
    pts = []
    for q in ((60.0, 0.0, 0.0), (0.0, -75.0, 0.0), (50.0, 40.0, 0.0), (120.0, 0.0, 0.0), (0.0, 33.0, 0.0)):
        for shift in range(64):
            qq = np.asarray(q, F32) + np.asarray([shift, shift, 0], F32) * F32(0.0625)
            r = np_radius(qq[None], radius, unit)[0]
            r2 = F32(np.float64(r) * np.float64(r))
            hit = _float_at_squared(r2)
            if hit is not None:
                break
        assert hit is not None
        at, inside = hit
        # the neighbours sit on the z axis through the query: dx = dy = 0 exactly, d2 = fl(dz*dz)
        pts += [qq, qq + np.asarray([0, 0, at], F32), qq - np.asarray([0, 0, inside], F32),
                qq + np.asarray([0, 0, F32(0.5) * at], F32), qq - np.asarray([0, 0, F32(0.25) * at], F32)]
        assert flann_d2(qq, pts[-4]) == r2 and flann_d2(qq, pts[-3]) < r2
    return _rows(np.asarray(pts, F32))


def cloud_far_clusters(radius=0.5):
    """dense clusters at 200 m and 1 km (radius there > 2.5 x the base radius) plus near clutter"""
    rng = np.random.default_rng(3)
    parts = [rng.uniform(-8, 8, (600, 3)),
             _shells((200.0, 0, 0), rng, 500, 0.0, 3.0),
             _shells((0, 1000.0, 5.0), rng, 500, 0.0, 4.0),
             _shells((-700.0, -700.0, 0), rng, 300, 0.0, 6.0)]
    return _rows(np.concatenate(parts))


def cloud_asymmetric_pairs(radius=1.0):
    """radial pairs A, B with r_A < |AB| < r_B: B lists A, A does not list B. A at range 29.9 keeps the base radius; A at
    range 40 has an adapted radius too, just below B's."""
    pts = []
    for u in ((1, 0, 0), (0, 1, 0), (0, 0, -1), (0.6, 0.8, 0), (1 / 3, -2 / 3, 2 / 3)):
        u = np.asarray(u, np.float64)
        for a, b in ((29.9, 30.904), (40.0, 41.17)):
            A, B = (a * radius * u).astype(F32), (b * radius * u).astype(F32)
            rA, rB = np_radius(np.stack([A, B]), radius, 30.0 * radius)
            d = np.sqrt(np.float64(flann_d2(A, B)))
            assert rA < d < rB, (a, b, rA, d, rB)
            pts += [A, B]
    return _rows(np.asarray(pts, F32))


CLOUDS = {
    "unit_range": (cloud_at_unit_range, 1.0),
    "adaptive_radius": (cloud_at_adaptive_radius, 1.0),
    "far_clusters": (cloud_far_clusters, 0.5),
    "asymmetric": (cloud_asymmetric_pairs, 1.0),
}


def far_unground_cloud():
    """the kitti-shaped unground cloud plus a wall at 200 m and a pole and a wall at ~1 km, sparse as a scan sees them"""
    rng = np.random.default_rng(11)
    ung = unground_cloud()
    wall = np.stack([np.full(900, 200.0), rng.uniform(-15, 15, 900), rng.uniform(-1, 8, 900)], 1)
    pole = np.stack([rng.normal(20, 0.05, 300), rng.normal(990, 0.05, 300), rng.uniform(-1, 9, 300)], 1)
    wall2 = np.stack([rng.uniform(-40, 40, 600), np.full(600, 1000.0), rng.uniform(-1, 12, 600)], 1)
    extra = np.zeros((1800, 12), F32)
    extra[:, :3] = np.concatenate([wall, pole, wall2])
    extra[:, 8] = rng.uniform(0, 100, 1800)
    out = np.concatenate([ung[:18000], extra])
    np.random.default_rng(12).shuffle(out)
    return np.ascontiguousarray(out)


def classify_variant(variant):
    """the five configurations of test_gpu_classify_matches_oracle, plus the far-cluster cloud"""
    ung = unground_cloud()
    if variant == "kitti":
        p = kitti_params()
    elif variant == "no_nms":
        p = kitti_params(sharpen_with_nms=0)
    elif variant == "no_vertex":
        p = kitti_params(curvature_thre=0.0, fixed_num_downsampling=0)
    elif variant == "dense_stride1":
        p = kitti_params(pca_down_rate=1, neighbor_searching_radius=1.0, neighbor_k=50, neigh_k_min=8,
                         unground_down_fixed_num=12000)
    elif variant == "small":
        ung = unground_cloud(seed=9, config="small")
        p = kitti_params(fixed_num_downsampling=0, pca_down_rate=1)
    else:
        ung = far_unground_cloud()
        p = kitti_params(fixed_num_downsampling=0)
    return ung, p


CLASSIFY_VARIANTS = ["kitti", "no_nms", "no_vertex", "dense_stride1", "small", "far_clusters"]


def _assert_same(g, o, tag):
    for k in abi.OUT_NAMES:
        assert g[k].shape == o[k].shape, f"{tag}: {k} {g[k].shape} vs {o[k].shape}"
        assert np.array_equal(g[k].view(np.uint32), o[k].view(np.uint32)), f"{tag}: {k} differs"


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_radius_formula_at_the_unit_boundary():
    x30 = F32(30.0)
    up = np.nextafter(x30, F32(np.inf))
    r = np_radius(np.array([[x30, 0, 0], [up, 0, 0], [0, 0, -x30], [60, 0, 0], [1000, 0, 0]], F32), 1.0, 30.0)
    assert r[0] == F32(1.0) and r[2] == F32(1.0)  # dist == unit: strict `>` keeps the base radius
    assert r[3] == F32(np.sqrt(2.0)) and abs(r[4] - np.sqrt(1000 / 30)) < 1e-6
    # one float beyond: adapted; sqrt(1 + 2^-22) is within half an ulp of 1, so the radius rounds back to 1
    assert np.sqrt(np.float64(up) / 30.0) > 1.0 and r[1] == F32(1.0)
    r2 = np_radius(np.array([[up, 0, 0]], F32), 1.5, 30.0)
    assert r2[0] == F32(np.sqrt(np.float64(up) / 30.0) * 1.5)


@pytest.mark.parametrize("name", sorted(CLOUDS))
@pytest.mark.parametrize("k,stride", [(30, 1), (5, 1), (30, 2)])
def test_restatement_neighbourhoods_match_numpy(name, k, stride):
    make, radius = CLOUDS[name]
    rows = make(radius)
    got = orc_pca_features_adaptive(rows, radius, k, stride, 30.0, want_lists=True)
    pt_num, lists = np_neighbours(rows, radius, k, stride, 30.0)
    assert np.array_equal(got["pt_num"], pt_num)
    for i, sel in lists.items():
        assert np.array_equal(got["nbr"][i, : len(sel)], sel), i
        assert (got["nbr"][i, len(sel):] == -1).all()
    assert (got["pt_num"][np.setdiff1d(np.arange(len(rows)), np.arange(0, len(rows), stride))] == 0).all()


def test_the_clouds_exercise_what_they_name():
    # exactly at the adaptive squared radius: out; one float inside: in
    rows = cloud_at_adaptive_radius()
    got = orc_pca_features_adaptive(rows, 1.0, 30, 1, 30.0, want_lists=True)
    for q in range(0, len(rows), 5):
        assert q + 1 not in got["nbr"][q] and q + 2 in got["nbr"][q]
    # asymmetric pairs: B lists A, A does not list B
    rows = cloud_asymmetric_pairs()
    got = orc_pca_features_adaptive(rows, 1.0, 30, 1, 30.0, want_lists=True)
    for a in range(0, len(rows), 2):
        assert a in got["nbr"][a + 1] and a + 1 not in got["nbr"][a]
    # far clusters: neighbourhoods grow with the range; the fixed radius sees far fewer
    rows = cloud_far_clusters()
    ada = orc_pca_features_adaptive(rows, 0.5, 0, 1, 30.0)["pt_num"]
    fix = oracle.pca_features(rows, 0.5, 0, 1)["pt_num"]
    far = np.linalg.norm(rows[:, :3], axis=1) > 500
    assert np.sqrt(np.linalg.norm(rows[far, :3], axis=1).min() / 30) * 0.5 > 2.5 * 0.5
    assert ada[far].mean() > 5 * fix[far].mean()
    near = np.linalg.norm(rows[:, :3], axis=1) <= 30
    assert np.array_equal(ada[near], fix[near])


@pytest.mark.parametrize("name", sorted(CLOUDS))
def test_restatement_without_adaptation_is_the_oracle(name):
    make, radius = CLOUDS[name]
    rows = make(radius)
    for k, stride in ((30, 1), (0, 2)):
        got = orc_pca_features_adaptive(rows, radius, k, stride, 0.0)
        ref = oracle.pca_features(rows, radius, k, stride)
        for key in ("pt_num", "eigenvalues", "principal", "normal"):
            assert np.array_equal(got[key].view(np.uint32), ref[key].view(np.uint32)), (key, k, stride)


@pytest.mark.parametrize("variant", CLASSIFY_VARIANTS)
def test_restatement_classification(variant):
    """off: the oracle's output bit for bit; on (unit 30 and 35): deterministic and different from off"""
    ung, p = classify_variant(variant)
    off = orc_classify_adaptive(ung, p)
    _assert_same(off, oracle.classify_nground(ung, p), variant + " off")
    p.use_distance_adaptive_pca = 1
    results = {}
    for unit in (30.0, 35.0):
        p.pca_unit_distance = unit
        a, b = orc_classify_adaptive(ung, p), orc_classify_adaptive(ung, p)
        _assert_same(a, b, f"{variant} unit {unit} repeated")
        results[unit] = a
    changed = lambda x, y: any(x[k].shape != y[k].shape or not np.array_equal(x[k], y[k]) for k in abi.OUT_NAMES)
    assert changed(results[30.0], off)
    assert changed(results[30.0], results[35.0])
    p.pca_unit_distance = 0.0
    assert orc_classify_adaptive(ung, p) == {"rc": -103}


def test_struct_and_defaults():
    assert abi.ClassifyParams.pca_unit_distance.offset == abi.ClassifyParams.random_seed.offset + 4
    assert abi.default_classify_params().pca_unit_distance == 0.0
    assert "mulls_pca_features_adaptive" in abi.EXPORTED_SYMBOLS


def build_slam_frontend_caller(td):
    libdir = os.path.join(ROOT, "mulls_b200", "csrc")
    exe = os.path.join(td, "slam_frontend_caller")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-I", os.path.join(ROOT, "include", "dropin"),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "stubs", "ref"),
                           "-I", os.path.join(ROOT, "tests", "stubs"),
                           os.path.join(ROOT, "tests", "stubs", "slam_frontend_caller.cpp"),
                           "-o", exe, "-L", libdir, "-lmulls_b200", f"-Wl,-rpath,{libdir}"])
    return exe


def _parse_frontend(stdout):
    line = next(s for s in stdout.splitlines() if s.startswith("slam front end:"))
    toks = line.replace(";", "").split()
    return {toks[i]: int(toks[i + 1]) for i in range(3, len(toks) - 1, 2)}


def test_slam_frontend_caller_compiles_and_links():
    """test/mulls_slam.cpp:418-428 against the drop-in headers; without a GPU the call reports the missing device"""
    import torch

    with tempfile.TemporaryDirectory() as td:
        exe = build_slam_frontend_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    d = _parse_frontend(out.stdout)
    assert d["failures"] == 0
    if not torch.cuda.is_available():
        assert d["returned"] == 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CLOUDS) + ["scan"])
@pytest.mark.parametrize("k,stride,unit", [(30, 1, 30.0), (5, 2, 30.0), (50, 1, 35.0), (0, 1, 30.0)])
def test_gpu_pca_features_adaptive_matches_restatement(name, k, stride, unit):
    from mulls_b200.registration import Context

    if name == "scan":
        rows, radius = far_unground_cloud(), 0.7
    else:
        make, radius = CLOUDS[name]
        rows = make(radius)
    ctx = Context(0, 1, 16, 100000)
    g = ctx.pca_features(rows, radius, k, stride, unit_dist=unit)
    kk = k if k > 0 else 1024  # the device treats k <= 0 as 1024 (abi.h), the restatements as unlimited
    o = orc_pca_features_adaptive(rows, radius, kk, stride, unit)
    np.testing.assert_array_equal(g["pt_num"], o["pt_num"])
    sel = o["pt_num"] > 3
    lam_o, lam_g = o["eigenvalues"][sel].astype(np.float64), g["eigenvalues"][sel].astype(np.float64)
    scale = lam_o[:, :1] + 1e-12
    assert (np.abs(lam_g - lam_o) / scale).max(initial=0) < 1e-4
    gap01 = (lam_o[:, 0] - lam_o[:, 1]) / scale[:, 0] > 0.05
    gap12 = (lam_o[:, 1] - lam_o[:, 2]) / scale[:, 0] > 0.05
    dp = np.abs((g["principal"][sel] * o["principal"][sel]).sum(1))
    dn = np.abs((g["normal"][sel] * o["normal"][sel]).sum(1))
    assert dp[gap01].min(initial=1) > np.cos(1e-3)
    assert dn[gap01 & gap12].min(initial=1) > np.cos(1e-3)
    if 1 <= k <= 64:  # list mode: the float mean / covariance in radiusSearch order on both sides -> identical bits
        # where the eigenvectors are defined: a collinear neighbourhood (the adaptive-radius cloud lines its neighbours
        # up on the z axis) has a double eigenvalue, and any basis of its plane is an answer
        assert np.array_equal(g["eigenvalues"].view(np.uint32), o["eigenvalues"].view(np.uint32))
        for key, ok in (("principal", gap01), ("normal", gap01 & gap12)):
            assert np.array_equal(g[key][sel][ok].view(np.uint32), o[key][sel][ok].view(np.uint32)), key
        assert not np.any(g["pt_num"][~sel] > 3)
    # the fixed-radius entry point is untouched by an adaptive call before it
    f = ctx.pca_features(rows, radius, k, stride)
    np.testing.assert_array_equal(f["pt_num"], oracle.pca_features(rows, radius, kk, stride)["pt_num"])
    with pytest.raises(RuntimeError, match="-101"):
        ctx.pca_features(rows, radius, k, stride, unit_dist=0.0)
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", CLASSIFY_VARIANTS)
def test_gpu_classify_adaptive_matches_restatement(variant):
    from mulls_b200.registration import Context

    ung, p = classify_variant(variant)
    p.use_distance_adaptive_pca, p.pca_unit_distance = 1, 30.0
    ctx = Context(0, 1, 16, 200000)
    g = ctx.classify_nground(ung, p)
    o = orc_classify_adaptive(ung, p)
    _assert_same(g, o, variant)
    assert g["pillar"].shape[0] + g["beam"].shape[0] + g["facade"].shape[0] > 100
    if variant != "no_vertex":
        assert g["vertex"].shape[0] > 0
    # the flag off on the same context: the oracle's fixed-radius answer
    p.use_distance_adaptive_pca = 0
    _assert_same(ctx.classify_nground(ung, p), oracle.classify_nground(ung, p), variant + " off")
    ctx.close()


@pytest.mark.gpu
def test_gpu_extract_semantic_pts_adaptive_equals_the_chain_of_restatements():
    from mulls_b200.registration import Context

    raw, _ = raw_scan()
    gp = ground_params()
    cp = abi.default_classify_params()
    cp.neighbor_searching_radius, cp.neighbor_k, cp.neigh_k_min, cp.pca_down_rate = 1.0, 30, 8, 1
    cp.fixed_num_downsampling, cp.random_seed = 1, 5
    cp.use_distance_adaptive_pca, cp.pca_unit_distance = 1, 30.0
    ctx = Context(0, 1, 16, 200000)
    g = ctx.extract_semantic_pts(raw, 0.05, gp, cp)
    down = oracle.voxel_downsample(raw, 0.05)
    og = oracle.fast_ground_filter(down, gp)
    oc = orc_classify_adaptive(og["unground"], cp)
    assert np.array_equal(g["down"].view(np.uint32), down.view(np.uint32))
    for k in ("ground", "ground_down"):
        assert g[k].shape == og[k].shape and np.array_equal(g[k].view(np.uint32), og[k].view(np.uint32)), k
    _assert_same(g, oc, "extract")
    assert g["ground"].shape[0] > 100 and g["facade"].shape[0] > 50 and g["pillar"].shape[0] > 5
    ctx.close()


@pytest.mark.gpu
def test_gpu_adaptive_without_a_unit_is_refused():
    from mulls_b200.registration import Context

    ctx = Context(0, 1, 16, 200000)
    p = kitti_params(use_distance_adaptive_pca=1)  # pca_unit_distance stays 0, as a struct filled the old way
    with pytest.raises(RuntimeError, match="-103"):
        ctx.classify_nground(unground_cloud(n_keep=500), p)
    p.pca_unit_distance = -30.0
    with pytest.raises(RuntimeError, match="-103"):
        ctx.classify_nground(unground_cloud(n_keep=500), p)
    raw, _ = raw_scan()
    cp = abi.default_classify_params()
    cp.use_distance_adaptive_pca = 1
    with pytest.raises(RuntimeError, match="-103"):
        ctx.extract_semantic_pts(raw, 0.05, ground_params(), cp)
    ctx.close()


@pytest.mark.gpu
def test_gpu_slam_frontend_call_yields_feature_clouds():
    """test/mulls_slam.cpp:418-428 through the drop-in CFilter, use_distance_adaptive_pca = true: the call returns true
    and fills the pillar, facade and ground clouds on the device"""
    raw, _ = raw_scan()
    with tempfile.TemporaryDirectory() as td:
        exe = build_slam_frontend_caller(td)
        path = os.path.join(td, "raw.bin")
        raw.astype(F32).tofile(path)
        out = subprocess.run([exe, path], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    d = _parse_frontend(out.stdout)
    assert d["raw"] == len(raw) and d["returned"] == 1 and d["failures"] == 0, out.stdout
    assert d["pillar"] > 0 and d["facade"] > 0 and d["ground"] > 0, out.stdout
