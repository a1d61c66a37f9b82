"""mulls_classify_nground on adversarial clouds: promotion cascades, fixed-number sampling at its edges, normals on the
sector boundaries of xy_normal_balanced_downsample, and degenerate neighbourhoods.

The reference (lo::CFilter::classify_nground_pts, cfilter.hpp:2058-2290) runs three stages sequentially that the device
runs in parallel: the vertex promotion (:2169-2210, k_cls_promote_pre / k_cls_promote / k_cls_promote_apply), the
fixed-number sampling (block_sample_append's radix select) and the sector split (k_cls_fixed). Whether the parallel
scheme is right depends on the input, so every scene here is built to exercise one of them, and the test proves it does.

np_classify is an independent numpy restatement of everything after the PCA: the PCA results come from the oracle
(oracle.pca_features, or the adaptive restatement of test_adaptive_pca.py) and the neighbour lists from brute force
(np_neighbours: d2 < float32(r*r) in FLANN's float order, sorted by (d2, index), at most k; the close / far split at
0.64 * r * r). CPU part: np_classify equals oracle.classify_nground bit for bit on every scene, and the scenes have the
properties they are named after. GPU part: Context.classify_nground equals the oracle bit for bit on every scene, twice
on one context."""
import ctypes as C
import ctypes.util
import hashlib
import math
import os

import numpy as np
import pytest

from mulls_b200 import abi
from oracle import oracle
from test_adaptive_pca import flann_d2, np_neighbours, orc_classify_adaptive, orc_pca_features_adaptive
from test_classify import kitti_params

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
X86_NAN = np.uint64(0xFFF8000000000000).view(np.float64)  # what x86 SSE writes for 0/0: the default NaN, sign set


# ---------------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------------
def sample_keys(seed, cloud_id, n):
    """splitmix64(seed << 40 ^ cloud_id << 32 ^ index) for index 0..n-1 (mulls_oracle.cpp sample_key)"""
    z = ((np.uint64(seed) << np.uint64(40)) ^ (np.uint64(cloud_id) << np.uint64(32)) ^ np.arange(n, dtype=np.uint64))
    z = z + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def random_downsample(rows, keep, seed, cloud_id):
    """random_downsample_pcl: the `keep` rows with the smallest keys, order kept; untouched when keep < 0 or n <= keep"""
    if keep < 0 or len(rows) <= keep:
        return rows
    if keep == 0:
        return rows[:0]
    k = sample_keys(seed, cloud_id, len(rows))
    return rows[k <= np.sort(k)[keep - 1]]


_LIBM = C.CDLL(ctypes.util.find_library("m"))
_LIBM.atan2f.restype = C.c_float
_LIBM.atan2f.argtypes = [C.c_float, C.c_float]


def sector_ids(rows, sector_num=4, float_angle=True):
    """cfilter.hpp:572-585: std::atan2(normal_y, normal_x) is the float overload (atan2f); the wrap and the degrees are
    double. An angle of exactly 360 is clamped into the last sector. float_angle=False: the angle in double instead."""
    out = np.empty(len(rows), np.int64)
    for i, (nx, ny) in enumerate(np.asarray(rows, F32)[:, 4:6]):
        ang = float(_LIBM.atan2f(ny, nx)) if float_angle else math.atan2(float(ny), float(nx))
        if ang < 0:
            ang += 2 * math.pi
        ang *= 180.0 / math.pi
        out[i] = min(int(ang / (360.0 / sector_num)), sector_num - 1)
    return out


def xy_normal_balanced_downsample(rows, keep, seed, cloud_id0, sector_num=4):
    if len(rows) <= keep:
        return rows
    sid = sector_ids(rows, sector_num)
    return np.concatenate([random_downsample(rows[sid == j], keep, seed, cloud_id0 + j) for j in range(sector_num)])


def c_div(a, b):
    """C's int division (truncates toward zero)"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def to_f32(x):
    """double -> float as x86 converts: a NaN keeps its sign and the top of its payload"""
    x = np.asarray(x, np.float64)
    f = x.astype(F32)
    nan = np.isnan(x)
    if nan.any():
        b = x[nan].view(np.uint64)
        f.view(np.uint32)[nan] = (((b >> np.uint64(32)) & np.uint64(0x80000000)) | np.uint64(0x7FC00000)
                                  | ((b >> np.uint64(29)) & np.uint64(0x3FFFFF))).astype(np.uint32)
    return f


def ratio(num, den):
    """the double quotient of pca.hpp:425-426; 0/0 of finite operands is the x86 default NaN"""
    with np.errstate(divide="ignore", invalid="ignore"):
        q = num / den
    q[(num == 0) & (den == 0)] = X86_NAN
    return q


_NBR_CACHE = {}


def neighbour_lists(rows, radius, k, stride, unit):
    key = (hashlib.sha1(np.ascontiguousarray(rows[:, :3]).tobytes()).hexdigest(), float(radius), k, stride, float(unit))
    if key not in _NBR_CACHE:
        _NBR_CACHE[key] = np_neighbours(rows, radius, k, stride, unit)
    return _NBR_CACHE[key]


def nms(cloud, r2):
    """non_max_suppress (:1243-1312): sort by score descending, ties in push order; the greedy selection"""
    o = np.argsort(-cloud[:, 7], kind="stable")
    pts = cloud[o]
    alive = np.ones(len(pts), bool)
    kept = []
    for i in range(len(pts)):
        if alive[i]:
            kept.append(i)
            d = pts[:, :3] - pts[i, :3]
            alive &= ~(((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]) < r2)
    return pts, pts[kept]


def np_classify(cloud, P, trace=None):
    """classify_nground_pts after the PCA, restated. trace (a dict) receives the promotion bookkeeping:
    state (0 no candidate, 2 not promoted, 3 promoted neither pillar nor beam, 4 pillar, 5 beam), depth (1 + the depth of
    the deepest earlier counting neighbour for a promotion the threshold labels alone did not decide), parent,
    thr_only (the decision from the threshold labels alone), at_ratio (candidates whose ratio equalled the threshold),
    tipped_by_3 (candidates a state-3 neighbour would have promoted had it counted)."""
    rows = abi.as_aos48(cloud).copy()
    if P.fixed_num_downsampling:
        rows = random_downsample(rows, P.unground_down_fixed_num, P.random_seed, 18).copy()
    n = len(rows)
    stride = P.pca_down_rate if P.pca_down_rate > 0 else 1
    radius, k = F32(P.neighbor_searching_radius), P.neighbor_k
    unit = P.pca_unit_distance if P.use_distance_adaptive_pca else 0.0
    pca = (orc_pca_features_adaptive(rows, radius, k, stride, unit) if unit > 0 else oracle.pca_features(rows, radius, k, stride))
    pt, lists = neighbour_lists(rows, radius, k, stride, unit)
    assert np.array_equal(pt, pca["pt_num"])
    has = pt > 3
    ev = pca["eigenvalues"].astype(np.float64)
    l1, l2, l3 = ev[:, 0], ev[:, 1], ev[:, 2]
    s = l1 + l2 + l3
    curv = np.where(has & (s != 0), ratio(l3, np.where(s == 0, 1.0, s)), 0.0)
    lin = np.where(has, ratio(l1 - l2, l1), 0.0)
    pla = np.where(has, ratio(l2 - l3, l1), 0.0)
    pdir = np.where(has[:, None], pca["principal"], F32(0))
    ndir = np.where(has[:, None], pca["normal"], F32(0))
    # the PCA's own assign_normal(pt, feature, true) (pca.hpp:346-347, min_k = 1)
    an = pt > 1
    rows[an, 4:7] = ndir[an]
    rows[an, 7] = to_f32(pla[an])
    # the threshold loop (:2103-2166)
    big = pt > P.neigh_k_min
    z, pz, nz = rows[:, 2], np.abs(pdir[:, 2]), np.abs(ndir[:, 2])
    edge = big & (lin > P.edge_thre)
    pil = edge & (pz > F32(P.linear_vertical_sin_high_thre))
    bea = edge & ~pil & (pz < F32(P.linear_vertical_sin_low_thre)) & (z < F32(P.beam_height_max))
    plan = big & ~edge & (pla > P.planar_thre)
    roo = plan & (nz > F32(P.planar_vertical_sin_high_thre)) & (z > F32(P.roof_height_min))
    fac = plan & ~roo & (nz < F32(P.planar_vertical_sin_low_thre))
    rows[pil | bea, 4:7] = pdir[pil | bea]
    rows[pil | bea, 7] = to_f32(lin[pil | bea])
    label0 = np.zeros(n, np.int64)
    label0[pil], label0[bea], label0[fac], label0[roo] = 1, 2, 3, 4
    cls = {c: rows[label0 == v].copy() for v, c in enumerate(("pillar", "beam", "facade", "roof"), 1)}
    down = {c: rows[:0].copy() for c in ("pillar", "beam", "facade", "roof")}
    if not P.sharpen_with_nms:
        down["pillar"] = rows[pil & (lin > P.edge_thre_down)].copy()
        down["beam"] = rows[bea & (lin > P.edge_thre_down)].copy()
        down["facade"] = rows[fac & (pla > P.planar_thre_down)].copy()
        down["roof"] = rows[roo & (pla > P.planar_thre_down)].copy()
    # the promotion loop (:2169-2210), in index order
    label = label0.copy()
    state = np.zeros(n, np.int64)
    depth = np.zeros(n, np.int64)
    parent = np.full(n, -1, np.int64)
    thr_only = np.zeros(n, bool)
    at_ratio, tipped_by_3 = [], []
    method = 0 if P.curvature_thre < 1e-8 else P.extract_vertex_points_method
    thre = float(F32(P.feature_pts_ratio_guess) / F32(stride))
    promoted = {"pillar": [], "beam": []}
    if method == 2:
        for i in np.flatnonzero((label0 == 0) & big & (curv > P.curvature_thre)):
            nb = lists[i]
            cnt = int(np.count_nonzero(label[nb]))
            thr_only[i] = 1.0 * int(np.count_nonzero(label0[nb])) / pt[i] > thre
            if 1.0 * cnt / pt[i] == thre:
                at_ratio.append(i)
            if not 1.0 * cnt / pt[i] > thre:
                state[i] = 2
                if 1.0 * (cnt + int(np.count_nonzero(state[nb] == 3))) / pt[i] > thre:
                    tipped_by_3.append(i)
                continue
            rows[i, 4:7] = pdir[i]
            rows[i, 7] = F32(5.0 * curv[i])
            if pz[i] > F32(P.linear_vertical_sin_high_thre):
                label[i], state[i] = 1, 4
                promoted["pillar"].append(rows[i].copy())
            elif pz[i] < F32(P.linear_vertical_sin_low_thre) and z[i] < F32(P.beam_height_max):
                label[i], state[i] = 2, 5
                promoted["beam"].append(rows[i].copy())
            else:
                state[i] = 3
            if not thr_only[i]:
                prev = nb[(nb < i) & (state[nb] >= 4)]
                if len(prev):
                    j = prev[np.argmax(depth[prev])]
                    depth[i], parent[i] = depth[j] + 1, j
            else:
                depth[i] = 1
    for c in ("pillar", "beam"):
        if promoted[c]:
            cls[c] = np.concatenate([cls[c], np.asarray(promoted[c], F32)])
    if trace is not None:
        trace.update(state=state, depth=depth, parent=parent, thr_only=thr_only, at_ratio=at_ratio, tipped_by_3=tipped_by_3,
                     label0=label0, pt_num=pt, curvature=curv)
    # encode_stable_points (:1071-1181)
    min_feature_pts = int(F32(F32(P.feature_pts_ratio_guess) / F32(stride)) * F32(P.neighbor_k)) - 1
    min_curvature = F32(0.3 * P.curvature_thre)
    close_r2 = 0.64 * float(radius) * float(radius)
    vertex = []
    for i in np.flatnonzero(big & has & (curv > min_curvature)):
        nb = lists[i]
        lab = label[nb]
        close = flann_d2(rows[i, :3], rows[nb, :3]).astype(np.float64) < close_r2
        total = len(nb)
        if np.count_nonzero(lab) < min_feature_pts:
            continue
        d = [0, 0, 0]
        for lv in range(1, 5):
            for m, sel in enumerate((lab == lv, (lab == lv) & close, (lab == lv) & ~close)):
                d[m] = d[m] * 100 + 100 * int(np.count_nonzero(sel)) // total
        p = rows[i].copy()
        p[7] = F32(curv[i])
        p[9], p[4], p[5] = F32(d[0]), F32(d[1]), F32(d[2])
        p[8] = np.cumsum(rows[nb, 8], dtype=F32)[-1] / F32(total)
        vertex.append(p)
    # non_max_suppress (:2229-2253)
    if P.sharpen_with_nms:
        nms_radius = F32(0.25 * float(radius))
        r2 = F32(np.float64(nms_radius) * np.float64(nms_radius))
        for c, fixed in (("pillar", P.pillar_down_fixed_num), ("facade", P.facade_down_fixed_num),
                         ("beam", P.beam_down_fixed_num), ("roof", P.roof_down_fixed_num)):
            if fixed > 0 and len(cls[c]) >= 10:
                cls[c], kept = nms(cls[c], r2)
                down[c] = np.concatenate([down[c], kept])
    # the fixed numbers (:2257-2267)
    if P.fixed_num_downsampling:
        down["pillar"] = random_downsample(down["pillar"], P.pillar_down_fixed_num, P.random_seed, 19)
        down["facade"] = xy_normal_balanced_downsample(down["facade"], c_div(P.facade_down_fixed_num, 4), P.random_seed, 20)
        down["beam"] = xy_normal_balanced_downsample(down["beam"], c_div(P.beam_down_fixed_num, 4), P.random_seed, 24)
        down["roof"] = random_downsample(down["roof"], P.roof_down_fixed_num, P.random_seed, 28)
    out = {c: np.ascontiguousarray(cls[c], F32) for c in cls}
    out.update({c + "_down": np.ascontiguousarray(down[c], F32) for c in down})
    out["vertex"] = np.asarray(vertex, F32).reshape(-1, 12)
    out["unground"] = rows
    return out


# ---------------------------------------------------------------------------------------------------------------------
# scenes (finite coordinates only)
# ---------------------------------------------------------------------------------------------------------------------
def _rows(xyz, rng):
    r = np.zeros((len(xyz), 12), F32)
    r[:, :3] = np.asarray(xyz, F32)
    r[:, 8] = rng.uniform(0, 50, len(xyz))
    return r


def _pole(rng, x, y, z0, z1, n):
    return np.stack([rng.normal(x, 0.004, n), rng.normal(y, 0.004, n), np.linspace(z0, z1, n)], 1)


def _column(rng, x, y, n, rad, z0, z1):
    """a thick vertical column, uniform in a disc of radius rad, ordered upward: its neighbourhoods are volumetric, and
    its points are ordered outward from the pole it stands on"""
    r = rad * np.sqrt(rng.uniform(0, 1, n))
    t = rng.uniform(0, 2 * np.pi, n)
    p = np.stack([x + r * np.cos(t), y + r * np.sin(t), rng.uniform(z0, z1, n)], 1)
    return p[np.argsort(p[:, 2], kind="stable")]


def _wall_y(rng, y, x0, x1, z0, z1, n):
    """a wall on the plane y = const exactly"""
    return np.stack([rng.uniform(x0, x1, n), np.full(n, y), rng.uniform(z0, z1, n)], 1)


def scene_cascade(seed=1):
    """Thick columns on thin poles, next to a wall, indices ordered upward from the pole: a column point reaches the
    promotion ratio only through the points below it that were promoted before it. Column A (3000 points, radius 6 cm)
    cascades under the default parameters, column B (2000 points, 5 cm) under the kitti ones. Column C, at 40 m (where
    the adaptive radius grows), is cut into five pieces with blocks of 1026 wall points between them, so its promotion
    chain has links more than 1024 indices apart."""
    rng = np.random.default_rng(seed)
    a = [_pole(rng, 0, 0, -4, 0.2, 200), _column(rng, 0, 0, 3000, 0.06, 0.0, 8.0)]
    b = [_pole(rng, 3, 0, -4, 0.2, 200), _column(rng, 3, 0, 3000, 0.05, 0.0, 12.0)]
    wall = _wall_y(rng, -1.5, -2.0, 5.0, -4.0, 8.0, 5130)
    c_pole, c_col = _pole(rng, 40, 0, -4, 0.2, 200), _column(rng, 40, 0, 1500, 0.06, 0.0, 4.0)
    parts = a + b + [c_pole]
    for s in range(5):
        parts.append(c_col[300 * s: 300 * (s + 1)])
        parts.append(wall[1026 * s: 1026 * (s + 1)])
    return _rows(np.concatenate(parts), rng)


def _wall(rng, centre, normal, n, w=6.0, h=4.0):
    """n points on the plane through centre with the given horizontal normal, spanned by exact multiples"""
    nx, ny = normal
    u, v = rng.uniform(-w / 2, w / 2, n), rng.uniform(0, h, n)
    return np.stack([centre[0] - ny * u, centre[1] + nx * u, centre[2] + v], 1)


def _beam(centre, direction, n, length=6.0):
    t = np.linspace(-length / 2, length / 2, n)
    return np.stack([centre[0] + direction[0] * t, centre[1] + direction[1] * t, np.full(n, centre[2])], 1)


def scene_sectors(seed=2):
    """Walls whose normals lie on the sector boundaries (normal x or y equal to +-0 and +-1, and exact diagonals), and
    exactly straight beams along the axes and the diagonals (principal x or y +-0, +-1): atan2f of these sits on a
    boundary, where the float angle and the double angle fall into different sectors"""
    rng = np.random.default_rng(seed)
    parts = []
    for k, nrm in enumerate(((1, 0), (0, 1), (-1, 0), (0, -1), (1, 1), (1, -1))):
        parts.append(_wall(rng, (20.0 * k, 30.0, 0.0), nrm, 700))
    for k, d in enumerate(((1, 0), (0, 1), (1, 1), (1, -1))):
        parts.append(_beam((20.0 * k, -30.0, 2.0), d, 160))
    parts.append(_pole(rng, 0, 0, 0, 6, 160))
    parts.append(np.stack([rng.uniform(-3, 3, 500), rng.uniform(50, 56, 500), np.full(500, 9.0)], 1))  # a roof
    return _rows(np.concatenate(parts), rng)


def scene_one_wall(seed=3):
    """one long wall (more than 1024 facade points, every normal in one or two sectors: the others empty) and one beam"""
    rng = np.random.default_rng(seed)
    return _rows(np.concatenate([_wall(rng, (0, 10.0, 0), (0, 1), 6000, w=30.0), _beam((0, -10.0, 2.0), (1, 0), 300, 20.0)]), rng)


def scene_degenerate(seed=4, k_min=8, k=50):
    """Clusters of 4, k_min + 1 and k + 5 identical points at representable and at non-representable coordinates (zero
    float covariance: l1 == 0, so linear_2 and planar_2 are 0/0), exactly collinear points (l2 == l3 == 0: every
    point has linear_2 == 1, equal NMS scores in the beam class), all apart from each other, plus some clutter. (An
    exactly vertical line is in test_gpu_vertical_collinear_pole.)"""
    rng = np.random.default_rng(seed)
    parts = []
    for m, size in enumerate((4, k_min + 1, k + 5)):
        parts.append(np.tile([[10.0 * m + 1.0, 2.0, 0.5]], (size, 1)))
        parts.append(np.tile([[10.0 * m + 0.1, 20.2, 0.3]], (size, 1)))
    parts.append(np.stack([np.arange(120) * 0.0625 - 20.0, np.full(120, -4.0), np.full(120, 1.5)], 1))  # collinear
    parts.append(rng.uniform(-45, -35, (800, 3)))
    rows = _rows(np.concatenate(parts), rng)
    return rows[np.random.default_rng(seed).permutation(len(rows))]


def default_params(**kw):
    p = abi.default_classify_params()
    p.random_seed = 7
    for key, v in kw.items():
        setattr(p, key, v)
    return p


PARAMS = {"default": default_params, "kitti": lambda **kw: kitti_params(**{"fixed_num_downsampling": 0, **kw})}


def scene(name, pname):
    P = PARAMS[pname]()
    if name == "cascade":
        return scene_cascade(), P
    if name == "sectors":
        return scene_sectors(), PARAMS[pname](sharpen_with_nms=0, fixed_num_downsampling=1)
    if name == "one_wall":
        return scene_one_wall(), PARAMS[pname](sharpen_with_nms=0, fixed_num_downsampling=1, facade_down_fixed_num=4000)
    if name == "degenerate":
        return scene_degenerate(k_min=P.neigh_k_min, k=P.neighbor_k), P
    if name == "ratio_edge":  # a threshold that a neighbour count can equal: 0.25 / pca_down_rate of 24 neighbours
        return scene_cascade(), PARAMS[pname](neighbor_k=24, feature_pts_ratio_guess=0.25)
    raise KeyError(name)


SCENES = ["cascade", "sectors", "one_wall", "degenerate", "ratio_edge"]


def sampling_variants(pname):
    """Fixed numbers chosen from the counts the *_down clouds reach before the sampling: for every class, and for every
    non-empty sector of the facade / beam clouds, keep = count - 1, count and count + 1 (facade and beam fixed numbers
    4 * keep + 1..3, not divisible by 4); keep 1 and 0; the unground cloud at n - 1, n and n + 1 points (n > 1024); a
    sector of more than 1024 points with keep = its count - 1."""
    out = []
    for name in ("sectors", "one_wall"):
        rows, P = scene(name, pname)
        P.fixed_num_downsampling = 0
        base = oracle.classify_nground(rows, P)
        for c, field in (("pillar", "pillar_down_fixed_num"), ("roof", "roof_down_fixed_num")):
            m = len(base[c + "_down"])
            for keep in sorted({max(m - 1, 0), m, m + 1, 1, 0}):
                out.append((name, {field: keep}))
        for c, field in (("facade", "facade_down_fixed_num"), ("beam", "beam_down_fixed_num")):
            counts = np.bincount(sector_ids(base[c + "_down"]), minlength=4)
            keeps = {1, 0} | {int(m) + d for m in counts if m > 1 for d in (-1, 0, 1)}
            for j, keep in enumerate(sorted(keeps)):
                out.append((name, {field: 4 * keep + 1 + j % 3}))
        if name == "sectors":
            n = len(rows)
            for keep in (n - 1, n, n + 1):
                out.append((name, {"unground_down_fixed_num": keep}))
    return out


def run_variant(name, pname, over):
    rows, P = scene(name, pname)
    for key, v in over.items():
        setattr(P, key, v)
    return rows, P


def assert_bits(a, b, tag):
    for key in abi.OUT_NAMES:
        assert a[key].shape == b[key].shape, f"{tag}: {key} {a[key].shape} vs {b[key].shape}"
        assert np.array_equal(a[key].view(np.uint32), b[key].view(np.uint32)), f"{tag}: {key} differs"


def chain_gaps(trace, lo, hi):
    """the longest run of promotion links (i, parent[i]) more than 1024 indices apart among the points lo..hi"""
    best = 0
    for i in range(lo, hi):
        run, j = 0, i
        while trace["parent"][j] >= 0:
            if j - trace["parent"][j] > 1024:
                run += 1
            j = trace["parent"][j]
        best = max(best, run)
    return best


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("name", SCENES)
def test_restatement_is_the_oracle(name, pname):
    rows, P = scene(name, pname)
    tr = {}
    assert_bits(np_classify(rows, P, tr), oracle.classify_nground(rows, P), f"{name} {pname}")
    st = tr["state"]
    if name in ("cascade", "ratio_edge"):
        # promotions propagate: decisions the threshold labels alone get wrong, chains of dependent promotions,
        # promotions that do not count (state 3) and would have tipped a later candidate
        assert np.count_nonzero(((st >= 3) != tr["thr_only"])[st > 0]) >= 50
        assert np.count_nonzero(st == 3) > 0 and len(tr["tipped_by_3"]) > 0
    if name == "cascade":
        assert tr["depth"].max() >= 20, tr["depth"].max()
        # column C: promotions whose deepest counting neighbour lies across a wall block, more than 1024 indices back
        i = np.arange(len(rows))
        assert np.count_nonzero((tr["parent"] >= 0) & (i - tr["parent"] > 1024)) >= 3
        assert chain_gaps(tr, 6600, len(rows)) >= 1
    if name == "ratio_edge":  # some candidates sit exactly at the threshold and stay unpromoted (strict >)
        assert len(tr["at_ratio"]) > 0 and (st[tr["at_ratio"]] == 2).all()


def test_scenes_exercise_the_sector_split_and_degenerate_neighbourhoods():
    # sector boundaries: normal components exactly +-0 / +-1 and diagonals; there the float angle (the reference's)
    # and the double angle disagree on the sector
    for pname in PARAMS:
        rows, P = scene("sectors", pname)
        P.fixed_num_downsampling = 0
        o = oracle.classify_nground(rows, P)
        f = o["facade_down"]
        for v in (0.0, 1.0):
            assert (f[:, 4] == v).any() and (f[:, 5] == v).any()
            assert (f[:, 4] == -v).any() and (f[:, 5] == -v).any()
        assert (np.signbit(f[:, 5]) & (f[:, 5] == 0)).any()  # a -0.0
        diag = np.abs(np.abs(f[:, 4]) - np.abs(f[:, 5])) < 1e-6
        assert (diag & (f[:, 4] * f[:, 5] > 0)).any() and (diag & (f[:, 4] * f[:, 5] < 0)).any()
        assert (sector_ids(f) != sector_ids(f, float_angle=False)).sum() > 50
        b = o["beam_down"]
        assert ((np.abs(b[:, 4]) == 1) & (b[:, 5] == 0)).any() and ((b[:, 4] == 0) & (np.abs(b[:, 5]) == 1)).any()
        # one wall: a sector of more than 1024 points, empty sectors, every beam in one sector
        rows, P = scene("one_wall", pname)
        P.fixed_num_downsampling = 0
        o = oracle.classify_nground(rows, P)
        fc, bc = np.bincount(sector_ids(o["facade_down"]), minlength=4), np.bincount(sector_ids(o["beam_down"]), minlength=4)
        assert (fc == 0).any() and (np.count_nonzero(bc) == 1)
        if pname == "default":
            assert fc.max() > 1024
    # degenerate: l1 == 0 gives the x86 default NaN in normal[3]; collinear points give equal NMS scores
    for pname in PARAMS:
        rows, P = scene("degenerate", pname)
        o = oracle.classify_nground(rows, P)
        bits = o["unground"][:, 7].view(np.uint32)
        assert np.count_nonzero(bits == 0xFFC00000) >= (P.neighbor_k + 5) // P.pca_down_rate
        assert not (bits == 0x7FFFFFFF).any() and not (bits == 0x7FC00000).any()
        beam = o["beam"][:, 7]
        assert len(beam) >= 10 and np.count_nonzero(beam == F32(1.0)) >= 10


def test_restatement_fixed_numbers_are_the_oracle():
    seen = 0
    for pname in PARAMS:
        for name, over in sampling_variants(pname):
            rows, P = run_variant(name, pname, over)
            assert_bits(np_classify(rows, P), oracle.classify_nground(rows, P), f"{name} {pname} {over}")
            seen += 1
    assert seen > 40


@pytest.mark.parametrize("name", ["cascade", "degenerate"])
def test_restatement_adaptive_is_the_adaptive_oracle(name):
    rows, P = scene(name, "kitti")
    P.use_distance_adaptive_pca, P.pca_unit_distance = 1, 30.0
    assert_bits(np_classify(rows, P), orc_classify_adaptive(rows, P), name)


def test_sample_keys_and_the_fixed_number_edges():
    # the k-th smallest key is unique (splitmix64 is a bijection): exactly `keep` rows survive
    rows = np.zeros((3000, 12), F32)
    rows[:, 0] = np.arange(3000)
    for keep in (0, 1, 2, 1023, 1024, 1025, 2999, 3000, 3001, -1):
        got = random_downsample(rows, keep, 7, 20)
        assert len(got) == (3000 if keep < 0 else min(keep, 3000))
        assert (np.diff(got[:, 0]) > 0).all()
    assert c_div(7, 4) == 1 and c_div(-7, 4) == -1


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _device_twice(ctx, rows, P, ref, tag):
    for rep in range(2):
        assert_bits(ctx.classify_nground(rows, P), ref, f"{tag} call {rep}")


@pytest.mark.gpu
@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("name", SCENES)
def test_gpu_classify_matches_oracle_on_adversarial_scenes(name, pname):
    from mulls_b200.registration import Context

    rows, P = scene(name, pname)
    ctx = Context(0, 1, 16, 200000)
    _device_twice(ctx, rows, P, oracle.classify_nground(rows, P), f"{name} {pname}")
    if name in ("cascade", "degenerate"):
        P.use_distance_adaptive_pca, P.pca_unit_distance = 1, 30.0
        _device_twice(ctx, rows, P, orc_classify_adaptive(rows, P), f"{name} {pname} adaptive")
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pname", sorted(PARAMS))
def test_gpu_fixed_numbers_match_oracle(pname):
    from mulls_b200.registration import Context

    ctx = Context(0, 1, 16, 200000)
    for name, over in sampling_variants(pname):
        rows, P = run_variant(name, pname, over)
        _device_twice(ctx, rows, P, oracle.classify_nground(rows, P), f"{name} {pname} {over}")
    ctx.close()


@pytest.mark.gpu
def test_gpu_duplicate_clusters_carry_the_x86_nan():
    """the issue's cloud: 12 identical rows at (1, 2, 0.5) behind 3000 unground points; normal[3] of every one is
    0xffc00000, the x86 default NaN, as the oracle writes it"""
    from mulls_b200.registration import Context
    from test_classify import unground_cloud

    dup = np.zeros((12, 12), F32)
    dup[:, :3] = (1.0, 2.0, 0.5)
    rows = np.concatenate([unground_cloud(n_keep=3000), dup])
    P = kitti_params(fixed_num_downsampling=0, pca_down_rate=1)
    ctx = Context(0, 1, 16, 200000)
    g, o = ctx.classify_nground(rows, P), oracle.classify_nground(rows, P)
    assert [hex(v) for v in o["unground"][-12:, 7].view(np.uint32)] == ["0xffc00000"] * 12
    assert [hex(v) for v in g["unground"][-12:, 7].view(np.uint32)] == ["0xffc00000"] * 12
    assert_bits(g, o, "duplicates")
    ctx.close()


@pytest.mark.gpu
@pytest.mark.xfail(strict=True, reason="the PCA's normal of a neighbourhood with a double zero eigenvalue is any unit "
                   "vector of a plane; near the ends of an exactly vertical line the device picks (-1, 0, 0) where the "
                   "oracle picks (0, 1, 0), and the unground rows carry it")
def test_gpu_vertical_collinear_pole():
    from mulls_b200.registration import Context

    rng = np.random.default_rng(5)
    rows = _rows(np.concatenate([np.stack([np.full(60, -30.0), np.full(60, 3.0), np.arange(60) * 0.125], 1),
                                 rng.uniform(-45, -35, (400, 3))]), rng)
    P = default_params()
    ctx = Context(0, 1, 16, 200000)
    try:
        assert_bits(ctx.classify_nground(rows, P), oracle.classify_nground(rows, P), "vertical line")
    finally:
        ctx.close()


@pytest.mark.gpu
def test_gpu_extract_semantic_pts_on_the_degenerate_scene():
    """the degenerate scene through mulls_extract_semantic_pts (voxel filter off), against the chain of the oracle's
    stages; the NaN of the duplicate clusters reaches the unground cloud"""
    from mulls_b200.registration import Context
    from test_ground import params as ground_params

    rows, P = scene("degenerate", "default")
    gp = ground_params()
    ctx = Context(0, 1, 16, 200000)
    g = ctx.extract_semantic_pts(rows, 0.0, gp, P)
    down = oracle.voxel_downsample(rows, 0.0)
    og = oracle.fast_ground_filter(down, gp)
    oc = oracle.classify_nground(og["unground"], P)
    assert np.array_equal(g["down"].view(np.uint32), down.view(np.uint32))
    for key in ("ground", "ground_down"):
        assert np.array_equal(g[key].view(np.uint32), og[key].view(np.uint32)), key
    assert_bits(g, oc, "extract")
    assert (g["unground"][:, 7].view(np.uint32) == 0xFFC00000).any()
    ctx.close()


@pytest.mark.gpu
def test_gpu_deepest_cascade_device_time():
    """the monotone promotion rounds are serial in the chain depth: the device time of the deepest cascade, reported"""
    from mulls_b200.registration import Context

    rows, P = scene("cascade", "default")
    ctx = Context(0, 1, 16, 200000)
    ctx.classify_nground(rows, P)
    ms = []
    for _ in range(5):
        ctx.classify_nground(rows, P)
        ms.append(ctx.stats()["ms_total"])  # CUDA events around the call's stream work
    print(f"deepest cascade ({len(rows)} points): device time per call median {np.median(ms):.3f} ms")
    ctx.close()
