"""CPU checks of NDT with the KDTREE neighbourhood (omp_ndt with use_direct_search = false, K1-K5 of
mulls_b200/csrc/ndt_core.cuh), the mode mulls_omp_ndt_kdtree runs:
- the CPU restatement (tests/harness/ndt_kdtree_oracle.cpp) against an independent numpy restatement with brute-force radius
  search: the float centroid bits, every query's neighbour list (members and order), score, gradient and Hessian at
  fixed poses to float tolerance, and the walk (iteration count, reversals, step lengths, final pose);
- K2 pinned by a third party: cv2.flann's KDTREE_SINGLE radius search over the float centroids returns the same members
  with bit-identical distances;
- adversarial scenes (shared with tests/test_gpu_ndt_kdtree.py) and what each is there for;
- b200::omp_ndt_kdtree compiles against the drop-in headers and replays the mulls_slam call sites
  (tests/stubs/ndt_kdtree_caller.cpp)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from test_ndt import (F32, ROOT, bbox, cases, moved, ndt_oracle_lib, np_angles, np_gauss, np_leaves, np_solve, oracle_ndt,
                      rot, rows, structured_scene, walk_scene)

IP, FP, DP = C.POINTER(C.c_int), C.POINTER(C.c_float), C.POINTER(C.c_double)


_KD_LIBS = {}


def kd_lib(out_dir=None):
    """tests/harness/ndt_kdtree_oracle.cpp, built as tests/test_ndt.py builds the DIRECT7 restatement"""
    out_dir = out_dir or os.path.join(ROOT, "tests", "harness", "_build")
    if out_dir in _KD_LIBS:
        return _KD_LIBS[out_dir]
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available: the host instantiation of ndt_core.cuh cannot be built")
    src = os.path.join(ROOT, "tests", "harness", "ndt_kdtree_oracle.cpp")
    deps = [src] + [os.path.join(ROOT, "mulls_b200", "csrc", f) for f in ("ndt_core.cuh", "ransac_core.cuh", "ground_core.cuh")]
    deps.append(os.path.join(ROOT, "include", "mulls_b200", "abi.h"))
    out = os.path.join(out_dir, "libndt_kdtree_oracle.so")
    if not os.path.exists(out) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(out):
        os.makedirs(out_dir, exist_ok=True)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        tmp = out + f".{os.getpid()}.tmp"
        subprocess.check_call([nvcc, "-x", "cu", "-O2", "-std=c++17", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a",
                               "-ccbin", cxx, "-Xcompiler", "-fPIC,-ffp-contract=off,-fopenmp", "-shared", "-w", "-o", tmp, src,
                               "-lgomp"])
        os.replace(tmp, out)
    from mulls_b200 import abi
    lb = C.CDLL(out)
    lb.orc_ndt_kdtree.restype = C.c_int
    lb.orc_ndt_kdtree.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_float, DP, C.c_int, C.c_float, DP, DP,
                                  C.POINTER(abi.NdtResult), C.POINTER(abi.NdtIter), C.c_int]
    lb.orc_ndt_centroids.restype = C.c_long
    lb.orc_ndt_centroids.argtypes = [C.c_void_p, C.c_long, C.c_float, C.c_long, FP, IP, IP]
    lb.orc_ndt_kdtree_neighbours.restype = None
    lb.orc_ndt_kdtree_neighbours.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_float, DP, C.c_int, IP, IP, FP]
    lb.orc_ndt_kdtree_eval.restype = None
    lb.orc_ndt_kdtree_eval.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_float, DP, DP]
    _KD_LIBS[out_dir] = lb
    return lb


def oracle_kd(case, trace_cap=64):
    from mulls_b200 import abi
    t, s = rows(case["tgt"]), rows(case["src"])
    g = np.ascontiguousarray(case.get("guess", np.eye(4)), np.float64).ravel().copy()
    tb = np.ascontiguousarray(case.get("tb", bbox(case["tgt"])), np.float64)
    sb = np.ascontiguousarray(case.get("sb", bbox(case["src"])), np.float64)
    res = abi.NdtResult()
    tr = (abi.NdtIter * trace_cap)()
    kd_lib().orc_ndt_kdtree(t.ctypes.data, len(t), s.ctypes.data, len(s), case.get("res", 1.0), g.ctypes.data_as(DP),
                            int(case.get("filter", True)), case.get("thre", 10.0), tb.ctypes.data_as(DP), sb.ctypes.data_as(DP),
                            C.byref(res), tr, trace_cap)
    k = min(res.iterations, trace_cap)
    return dict(code=res.code, trans=np.array(res.trans[:]).reshape(4, 4), iterations=res.iterations,
                converged=bool(res.converged), fitness=res.fitness, n_target=res.n_target, n_source=res.n_source,
                trace=dict(p=np.array([tr[i].p[:] for i in range(k)]).reshape(k, 6), step=np.array([tr[i].step for i in range(k)]),
                           score=np.array([tr[i].score for i in range(k)]), reversed=np.array([tr[i].reversed for i in range(k)])))


def oracle_centroids(tgt, res):
    tr = rows(tgt)
    cap = max(len(tgt), 1)
    cent, cnt, rank = np.zeros((cap, 3), F32), np.zeros(cap, np.int32), np.zeros(cap, np.int32)
    m = kd_lib().orc_ndt_centroids(tr.ctypes.data, len(tgt), res, cap, cent.ctypes.data_as(FP), cnt.ctypes.data_as(IP),
                                   rank.ctypes.data_as(IP))
    return cent[:m], cnt[:m], rank[:m]


def oracle_lists(tgt, src, res, p, cap=64):
    tr, sr = rows(tgt), rows(src)
    n = len(src)
    cnt, leaf, d2 = np.zeros(n, np.int32), np.zeros((max(n, 1), cap), np.int32), np.zeros((max(n, 1), cap), F32)
    p = np.ascontiguousarray(p, np.float64)
    kd_lib().orc_ndt_kdtree_neighbours(tr.ctypes.data, len(tgt), sr.ctypes.data, n, res, p.ctypes.data_as(DP), cap,
                                       cnt.ctypes.data_as(IP), leaf.ctypes.data_as(IP), d2.ctypes.data_as(FP))
    assert cnt.max(initial=0) <= cap
    return [(leaf[i, :cnt[i]], d2[i, :cnt[i]]) for i in range(n)]


def oracle_kd_eval(tgt, src, res, p):
    out = np.zeros(43)
    tr, sr = rows(tgt), rows(src)
    p = np.ascontiguousarray(p, np.float64)
    kd_lib().orc_ndt_kdtree_eval(tr.ctypes.data, len(tgt), sr.ctypes.data, len(src), res, p.ctypes.data_as(DP),
                                 out.ctypes.data_as(DP))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the independent restatement: leaves as tests/test_ndt.py, float centroids by a sequential float32 sum, brute force
# ---------------------------------------------------------------------------------------------------------------------
def np_kd_leaves(xyz, res):
    """the leaves in ascending leaf index (np_leaves), each with its float centroid (the float32 running sum in input
    order, cumsum being sequential, over (float)n) and its index in the searchable cloud (-1: under 6 points)"""
    xyz = np.asarray(xyz, F32)
    xyz = xyz[np.isfinite(xyz).all(1)]
    if len(xyz) == 0:
        return [], {}, np.zeros((0, 3), F32), np.zeros(0, np.int64)
    leaves, min_b, max_b, div, inv = np_leaves(xyz, res)
    ijk = (np.floor(xyz * inv) - min_b.astype(F32)).astype(np.int64)
    key = ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1]
    keys = sorted(leaves)
    cent = np.zeros((len(keys), 3), F32)
    rank = np.full(len(keys), -1)
    r = 0
    for i, k in enumerate(keys):
        pts = xyz[key == k]
        cent[i] = np.cumsum(pts, axis=0, dtype=F32)[-1] / F32(len(pts))
        if len(pts) >= 6:
            rank[i], r = r, r + 1
    return keys, leaves, cent, rank


def np_kd_r2(res):
    return F32(np.float64(F32(res)) * np.float64(F32(res)))


def np_kd_d2(q, cent):
    d = (np.asarray(q, F32)[None, :] - cent).astype(F32)
    return ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(F32)


def np_kd_lists(tgt, src, res, shift=(0.0, 0.0, 0.0)):
    """brute force: every searchable centroid with float d2 < r2 from the float query src + shift, in (d2, index) order;
    as leaf positions in ascending leaf index"""
    keys, leaves, cent, rank = np_kd_leaves(tgt, res)
    sr = np.flatnonzero(rank >= 0)
    r2 = np_kd_r2(res)
    out = []
    q = (np.asarray(src, F32) + np.asarray(shift, F32)).astype(F32)
    for x in q:
        if not np.isfinite(x).all() or len(sr) == 0:
            out.append((np.zeros(0, np.int64), np.zeros(0, F32)))
            continue
        d2 = np_kd_d2(x, cent[sr])
        m = d2 < r2
        o = np.lexsort((rank[sr][m], d2[m]))
        out.append((sr[m][o], d2[m][o]))
    return out


def np_kd_eval(tgt, src, res, p):
    """score, gradient and Hessian in double (np_eval's terms) over the brute-force KDTREE neighbours; the query is the
    float moved point, a rejected leaf contributes with a zero inverse covariance"""
    keys, leaves, cent, rank = np_kd_leaves(tgt, res)
    sr = np.flatnonzero(rank >= 0)
    r2 = np_kd_r2(res)
    d1, d2c = np_gauss(res)
    R = rot(p[3], p[4], p[5])
    jt, ht = np_angles(p)
    score, grad, hess = 0.0, np.zeros(6), np.zeros((6, 6))
    for x in np.asarray(src, np.float64):
        y = R @ x + p[:3]
        d2 = np_kd_d2(y.astype(F32), cent[sr])
        m = d2 < r2
        xj, xh = jt @ x, ht @ x
        J = np.zeros((3, 6))
        J[:, :3] = np.eye(3)
        J[:, 3], J[:, 4], J[:, 5] = [0, xj[0], xj[1]], [xj[2], xj[3], xj[4]], [xj[5], xj[6], xj[7]]
        a, b, cc = np.array([0, xh[0], xh[1]]), np.array([0, xh[2], xh[3]]), np.array([0, xh[4], xh[5]])
        d, e, f = xh[6:9], xh[9:12], xh[12:15]
        H = {(3, 3): a, (4, 3): b, (5, 3): cc, (3, 4): b, (4, 4): d, (5, 4): e, (3, 5): cc, (4, 5): e, (5, 5): f}
        for li in sr[m]:
            lf = leaves[keys[li]]
            Ci = lf["icov"] if lf["ok"] else np.zeros((3, 3))
            xt = y - lf["mean"]
            ex = np.exp(-d2c * xt @ Ci @ xt / 2)
            if not (0 <= d2c * ex <= 1):
                continue
            score += -d1 * ex
            g6 = xt @ Ci @ J
            grad += d1 * d2c * ex * g6
            for i in range(6):
                for jj in range(6):
                    hij = H.get((i, jj), np.zeros(3))
                    hess[i, jj] += d1 * d2c * ex * (-d2c * g6[i] * g6[jj] + xt @ Ci @ hij + J[:, jj] @ Ci @ J[:, i])
    return score, grad, hess


def np_kd_walk(tgt, src, res):
    """tests/test_ndt.py's np_walk on np_kd_eval's derivatives"""
    p = np.zeros(6)
    s, g, H = np_kd_eval(tgt, src, res, p)
    steps, rev, nr = [], [], 0
    while True:
        d = np_solve(H, -g)
        n = np.linalg.norm(d)
        if n == 0 or n != n:
            return dict(iterations=nr, step=np.array(steps), reversed=np.array(rev), p=p)
        d = d / n
        d_phi_0 = -(g @ d)
        a, r = 0.0, 0
        if d_phi_0 >= 0 and d_phi_0 != 0:
            d, r = -d, 1
        if d_phi_0 != 0:
            a = min(max(n, 0.05), 0.1)
            p = p + a * d
            s, g, H = np_kd_eval(tgt, src, res, p)
        steps.append(a)
        rev.append(r)
        stop = nr > 35 or (nr and a < 0.1)
        nr += 1
        if stop:
            return dict(iterations=nr, step=np.array(steps), reversed=np.array(rev), p=p)


# ---------------------------------------------------------------------------------------------------------------------
# scenes (shared with tests/test_gpu_ndt_kdtree.py)
# ---------------------------------------------------------------------------------------------------------------------
def _grid(n, step, z=0.0, origin=(0.0, 0.0)):
    u = np.arange(n, dtype=np.float64) * step
    x, y = np.meshgrid(u + origin[0], u + origin[1], indexing="ij")
    return np.c_[x.ravel(), y.ravel(), np.full(x.size, z)].astype(F32)


def kd_cases():
    out = {k: v for k, v in cases().items() if k not in ("limit", "far")}
    base = structured_scene(3000, 31, extent=8.0)
    rng = np.random.default_rng(32)
    # 6 identical points alone in a leaf: searchable, rejected (all eigenvalues 0), so only KDTREE sees it
    ident = np.vstack([base, np.tile(np.array([[2.5, 2.5, 3.5]], F32), (6, 1))])
    out["identical6"] = dict(tgt=ident, src=np.vstack([base[::4], np.array([[2.6, 2.4, 3.3], [2.2, 2.9, 3.6]], F32)]))
    # an exactly planar target (z = x on a 0.1 grid): in many leaves the smallest eigenvalue rounds below zero
    plane = _grid(60, 0.1, origin=(-3.0, -3.0))
    plane[:, 2] = plane[:, 0]
    out["planar"] = dict(tgt=plane, src=(plane[::3] + np.array([0.05, -0.03, 0.2], F32)).astype(F32))
    # leaves of exactly 5 and exactly 6 points (a 5-point leaf is not searchable)
    lv = []
    for i in range(40):
        c = np.array([i % 8, (i // 8) % 5, 0], np.float64) + 0.5
        m = 5 if i % 2 else 6
        lv.append(c + rng.uniform(-0.3, 0.3, (m, 3)))
    five_six = np.vstack(lv).astype(F32)
    out["five_six"] = dict(tgt=five_six, src=(five_six + F32(0.05)).astype(F32))
    # a query exactly at d2 == r2 (excluded) and one float step inside (included): a leaf of 6 points symmetric about
    # (0.5, 0.5, 0.5), whose float centroid is exactly that point
    sym = np.array([[0.25, 0.5, 0.5], [0.75, 0.5, 0.5], [0.5, 0.25, 0.5], [0.5, 0.75, 0.5], [0.5, 0.5, 0.25], [0.5, 0.5, 0.75]], F32)
    inside = np.float32(np.nextafter(F32(1.5), F32(0.0)))
    out["radius_edge"] = dict(tgt=sym, src=np.array([[1.5, 0.5, 0.5], [inside, 0.5, 0.5], [0.5, -0.5, 0.5], [0.5, 0.5, 0.5]], F32),
                              filter=False)
    # a lattice target: centroids on a regular lattice, queries equidistant from several (exact distance ties)
    lat = []
    for i in range(6):
        for j in range(6):
            for k in range(3):
                c = np.array([i, j, k], np.float64) + 0.5
                lat.append(c + np.array([[0.25, 0, 0], [-0.25, 0, 0], [0, 0.25, 0], [0, -0.25, 0], [0, 0, 0.25], [0, 0, -0.25],
                                          [0.125, 0.125, 0.125], [-0.125, -0.125, -0.125]]))
    lattice = np.vstack(lat).astype(F32)
    ties = np.array([[i + 1.0, j + 1.0, 1.0] for i in range(4) for j in range(4)] + [[i + 1.0, j + 0.5, 1.5] for i in range(4)
                                                                                     for j in range(4)], F32)
    out["lattice"] = dict(tgt=lattice, src=np.vstack([ties, lattice[::3]]), filter=False)
    # centroids on cell faces: leaves whose points all lie on x = 1, 2, 3 (the lower face of their cell)
    fx = np.repeat(np.array([1.0, 2.0, 3.0]), 60)
    faces = np.c_[fx, rng.uniform(0, 3, 180), rng.uniform(0, 2, 180)].astype(F32)
    out["faces"] = dict(tgt=faces, src=(faces[::2] + np.array([0.4, 0.0, 0.0], F32)).astype(F32), filter=False)
    # coordinates offset by 1e4
    m = cases()["motion"]
    out["offset_1e4"] = dict(tgt=(m["tgt"] + F32(1e4)).astype(F32), src=(m["src"] + F32(1e4)).astype(F32))
    small = structured_scene(6000, 41, extent=4.0)
    small_src = moved(small[::2] + rng.normal(0, 0.01, (3000, 3)).astype(F32), rot(0.0, 0.0, 0.01).T, np.array([-0.04, 0.03, 0.0]))
    out["offset_1e4_res03"] = dict(tgt=(small + F32(1e4)).astype(F32), src=(small_src + F32(1e4)).astype(F32), res=0.3)
    # 27 neighbours: around the centre of a cell, a cluster in each of the 27 cells of its 3 x 3 x 3 block, placed at
    # the point of that cell nearest the centre (0.53 off it per axis); blocks repeated 4 apart. More than the 8 list
    # entries a device call starts with
    blk = []
    for b in range(6):
        centre = np.array([4.0 * (b % 3), 4.0 * (b // 3), 0.0]) + 0.5
        for o in np.array(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1], indexing="ij")).reshape(3, -1).T:
            blk.append(centre + 0.53 * o + rng.uniform(-0.01, 0.01, (8, 3)))
    dense = np.vstack(blk).astype(F32)
    centres = np.array([[4.0 * (b % 3) + 0.5, 4.0 * (b // 3) + 0.5, 0.5] for b in range(6)], F32)
    out["dense_cube"] = dict(tgt=dense, src=np.vstack([centres, dense[::5] + F32(0.02)]).astype(F32), filter=False)
    out["filter_off_guess"] = dict(tgt=m["tgt"], src=m["src"], guess=cases()["guess"]["guess"], filter=False)
    return out


_CASES = None


def kd_case(name):
    global _CASES
    if _CASES is None:
        _CASES = kd_cases()
    return _CASES[name]


def _leaf_ranks(case):
    res = case.get("res", 1.0)
    _, _, rank = oracle_centroids(case["tgt"], res)
    return rank


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,res", [("motion", 1.0), ("motion", 0.3), ("motion", 0.7), ("offset_1e4", 1.0),
                                      ("offset_1e4", 0.3), ("identical6", 1.0), ("faces", 1.0), ("five_six", 1.0)])
def test_centroids_equal_numpy(name, res):
    """K1: every leaf's float centroid bit for bit, the searchable set (6 or more points, rejected leaves included) and
    its index order"""
    c = kd_case(name)
    cent, cnt, rank = oracle_centroids(c["tgt"], res)
    keys, leaves, ncent, nrank = np_kd_leaves(c["tgt"], res)
    assert len(cent) == len(keys)
    assert np.array_equal(cent.view(np.uint32), ncent.view(np.uint32))
    assert np.array_equal(rank, nrank)
    assert np.array_equal(cnt, [leaves[k]["n"] for k in keys])
    if name == "identical6":  # the rejected leaf is searchable
        rej = [i for i, k in enumerate(keys) if leaves[k]["n"] >= 6 and not leaves[k]["ok"]]
        assert rej and all(rank[i] >= 0 for i in rej)


LIST_SCENES = ["dense_cube", "motion", "motion_res03", "motion_res07", "identical6", "planar", "five_six", "radius_edge", "lattice", "faces",
               "offset_1e4", "offset_1e4_res03", "non_finite", "small_leaves", "empty_target"]


@pytest.mark.parametrize("name", LIST_SCENES)
@pytest.mark.parametrize("shift", [(0.0, 0.0, 0.0), (0.11, -0.07, 0.05)])
def test_neighbour_lists_equal_brute_force(name, shift):
    """K2: every query's neighbours, members and order, against a brute-force search over all centroids (a pure
    translation keeps the float query exactly x + t)"""
    c = kd_case(name)
    res = c.get("res", 1.0)
    tgt, src = c["tgt"], c["src"]
    src = src[np.isfinite(src).all(1)] if name != "non_finite" else src
    o = oracle_lists(tgt, src, res, [shift[0], shift[1], shift[2], 0.0, 0.0, 0.0])
    n = np_kd_lists(tgt, src, res, shift)
    total = 0
    for i, ((ol, od), (nl, nd)) in enumerate(zip(o, n)):
        assert np.array_equal(ol, nl), (i, ol, nl)
        assert np.array_equal(od.view(np.uint32), nd.view(np.uint32)), i
        total += len(ol)
    if name in ("empty_target", "small_leaves"):
        assert total == 0  # K4
    else:
        assert total > 0
    if name == "radius_edge" and shift == (0.0, 0.0, 0.0):
        # d2 == r2 exactly: excluded; one float step inside: included; the ball's other edge point: excluded
        assert [len(x[0]) for x in o] == [0, 1, 0, 1]
        assert o[1][1][0] < np_kd_r2(res) and np.float32(1.0) == np_kd_r2(res)
    if name == "lattice" and shift == (0.0, 0.0, 0.0):
        ties = sum(int(np.any(np.diff(d) == 0)) for _, d in o)
        assert ties >= 16  # exact ties, ordered by index


@pytest.mark.parametrize("name", ["motion", "lattice", "offset_1e4"])
def test_k2_pinned_by_flann(name):
    """cv2.flann's KDTREE_SINGLE index (leaf_max_size 15) over the float centroids, radiusSearch with r2: the same
    members with bit-identical distances; the order differs at most across exact ties"""
    cv2 = pytest.importorskip("cv2")
    c = kd_case(name)
    res = c.get("res", 1.0)
    cent, cnt, rank = oracle_centroids(c["tgt"], res)
    sr = np.flatnonzero(rank >= 0)
    pts = np.ascontiguousarray(cent[sr], F32)
    index = cv2.flann_Index(pts, dict(algorithm=4, leaf_max_size=15))
    r2 = float(np_kd_r2(res))
    src = np.ascontiguousarray(c["src"][np.isfinite(c["src"]).all(1)], F32)
    o = oracle_lists(c["tgt"], src, res, np.zeros(6))
    pos = np.full(len(cent), -1)
    pos[sr] = np.arange(len(sr))
    checked = 0
    for i in range(len(src)):
        n, ind, dist = index.radiusSearch(src[i:i + 1], r2, 64, params=dict(checks=-1, eps=0.0, sorted=True))
        n = int(n)
        ol, od = o[i]
        assert n == len(ol), i
        fi, fd = ind[0, :n], dist[0, :n].astype(F32)
        assert sorted(fi.tolist()) == sorted(pos[ol].tolist()), i
        want = dict(zip(pos[ol].tolist(), od.view(np.uint32).tolist()))
        assert all(want[j] == d for j, d in zip(fi.tolist(), fd.view(np.uint32).tolist())), i
        assert np.array_equal(np.sort(fd).view(np.uint32), od.view(np.uint32)), i  # the same distances in the same order
        checked += n
    assert checked > 50


@pytest.mark.parametrize("res,p", [(1.0, [0, 0, 0, 0, 0, 0]), (1.0, [0.1, -0.05, 0.02, 0.01, -0.02, 0.03]),
                                   (0.7, [0.02, 0.01, 0.0, 0.0, 0.005, -0.01])])
def test_derivatives_equal_numpy(res, p):
    tgt = structured_scene(3000, 11)
    src = structured_scene(500, 12)
    p = np.array(p, np.float64)
    out = oracle_kd_eval(tgt, src, res, p)
    s, g, H = np_kd_eval(tgt, src, res, p)
    assert abs(out[0] - s) <= 1e-4 * abs(s)
    np.testing.assert_allclose(out[1:7], g, rtol=0, atol=2e-4 * np.abs(g).max() + 1e-6)
    np.testing.assert_allclose(out[7:].reshape(6, 6), H, rtol=0, atol=2e-4 * np.abs(H).max())


def test_walk_equals_numpy():
    """the restatement's KDTREE walk against the numpy walk: the same iteration count and reversals, the step lengths
    to 1e-5, the final pose to 1e-4"""
    c = walk_scene()
    o = oracle_kd(c)
    n = np_kd_walk(c["tgt"], c["src"], c["res"])
    assert o["iterations"] == n["iterations"] >= 3
    assert o["trace"]["reversed"].tolist() == n["reversed"].tolist()
    np.testing.assert_allclose(o["trace"]["step"], n["step"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(o["trace"]["p"][-1], n["p"], rtol=0, atol=1e-4)


def test_dense_cube_has_long_lists():
    """the dense_cube scene has points with more than 8 neighbours (the device's starting list capacity), so the GPU
    comparison on it covers the lists' growth"""
    c = kd_case("dense_cube")
    counts = [len(l) for l, _ in oracle_lists(c["tgt"], c["src"], 1.0, np.zeros(6))]
    assert counts[:6] == [27] * 6


def test_rejected_leaves_enter_only_the_kdtree_score():
    """K3: the 6 identical points form a searchable, rejected leaf. At p = 0 the two queries near it have it as a
    neighbour, each adding -d1 to the score and nothing to the gradient or Hessian; DIRECT7 never sees it"""
    c = kd_case("identical6")
    base = dict(tgt=c["tgt"][:-6], src=c["src"])
    z = np.zeros(6)
    with_leaf, without = oracle_kd_eval(c["tgt"], c["src"], 1.0, z), oracle_kd_eval(base["tgt"], base["src"], 1.0, z)
    d1, d2 = np_gauss(1.0)
    assert d2 <= 1.0
    keys, leaves, cent, rank = np_kd_leaves(c["tgt"], 1.0)
    lists = np_kd_lists(c["tgt"], c["src"], 1.0)
    rej = {i for i, k in enumerate(keys) if leaves[k]["n"] >= 6 and not leaves[k]["ok"]}
    hits = sum(sum(int(l in rej) for l in ls) for ls, _ in lists)
    assert hits >= 2
    # score_inc is a float (N4): each visit adds (float)(-d1 * 1)
    np.testing.assert_allclose(with_leaf[0] - without[0], hits * np.float64(F32(-d1)), rtol=1e-9)
    # the identical leaf is alone in its cell, so the other terms of these sums are unchanged
    np.testing.assert_allclose(with_leaf[1:], without[1:], rtol=0, atol=1e-9 * np.abs(without[1:]).max())


def test_planar_target_differs_from_direct7():
    """on an exactly planar target some leaves are rejected (their smallest eigenvalue rounds below zero) and stay
    searchable: the KDTREE score counts them, DIRECT7 does not see them"""
    c = kd_case("planar")
    keys, leaves, cent, rank = np_kd_leaves(c["tgt"], 1.0)
    o_cent, o_cnt, o_rank = oracle_centroids(c["tgt"], 1.0)
    from test_ndt import ndt_oracle_lib as lib
    cap = len(keys)
    k, n, ok = np.zeros(cap, np.int64), np.zeros(cap, np.int32), np.zeros(cap, np.int32)
    mean, icov = np.zeros((cap, 3)), np.zeros((cap, 9), F32)
    tr = rows(c["tgt"])
    lib().orc_ndt_leaves(tr.ctypes.data, len(tr), 1.0, cap, k.ctypes.data_as(C.POINTER(C.c_int64)), n.ctypes.data_as(IP),
                         mean.ctypes.data_as(DP), icov.ctypes.data_as(FP), ok.ctypes.data_as(IP))
    rejected = (n == -1) & (o_rank >= 0)
    assert rejected.any() and np.all(icov[rejected] == 0)
    kd, d7 = oracle_kd(c), oracle_ndt(c)
    assert kd["trace"]["score"][0] != d7["trace"]["score"][0]


@pytest.mark.parametrize("name", sorted(kd_cases()))
def test_walk_outcomes(name):
    c = kd_case(name)
    o = oracle_kd(c)
    tr = o["trace"]
    assert o["iterations"] <= 37
    assert np.all((tr["step"] == 0) | ((tr["step"] >= 0.05) & (tr["step"] <= 0.1)))
    if name in ("empty_source", "empty_target", "small_leaves", "filter_empties"):  # K4 and empty clouds
        assert o["iterations"] == 0 and o["converged"]
        np.testing.assert_array_equal(o["trans"], np.eye(4))
    if name == "non_finite":
        assert o["n_source"] == len(c["src"]) and np.isfinite(o["fitness"])
    if name.startswith("motion") or name in ("guess", "offset_1e4", "filter_off_guess"):
        assert o["code"] == 1 and o["converged"]
    if name == "five_six":  # only the 6-point leaves are searchable
        _, cnt, rank = oracle_centroids(c["tgt"], 1.0)
        assert np.all((rank >= 0) == (cnt >= 6)) and (cnt == 5).sum() == 20 and (cnt == 6).sum() == 20


def test_known_motion_recovered():
    c = cases()["motion"]
    o = oracle_kd(c)
    R, t = rot(0.01, -0.015, 0.03), np.array([0.15, -0.1, 0.05])
    T = o["trans"]
    assert np.linalg.norm(T[:3, 3] - t) < 0.06
    assert np.arccos(np.clip((np.trace(T[:3, :3].T @ R) - 1) / 2, -1, 1)) < 0.06


def build_kdtree_caller(td):
    libdir = os.path.join(ROOT, "mulls_b200", "csrc")
    exe = os.path.join(td, "ndt_kdtree_caller")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-I", os.path.join(ROOT, "include", "dropin"),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "stubs", "ndt_ref"),
                           "-I", os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests", "stubs", "ndt_kdtree_caller.cpp"),
                           "-o", exe, "-L", libdir, "-lmulls_b200", f"-Wl,-rpath,{libdir}"])
    return exe


def test_kdtree_helper_compiles_and_links():
    """tests/stubs/ndt_kdtree_caller.cpp replays mulls_slam.cpp:634-636 and :671-673 with --ndt_searching_method=false
    through b200::omp_ndt_kdtree (without a GPU: -3, Trans1_2 untouched); the drop-in member still calls the reference"""
    import tempfile

    import torch

    with tempfile.TemporaryDirectory() as td:
        exe = build_kdtree_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "ndt kdtree helper compiled and linked" in out.stdout and "failures 0" in out.stdout
    if not torch.cuda.is_available():
        assert "ran on a device: 0" in out.stdout
