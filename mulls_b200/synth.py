"""Seeded synthetic "KITTI-shape" LiDAR scan pairs (SURVEY.md §8 d).

A spinning multi-beam scanner (HDL-64E geometry by default: 64 beams linearly in [-24.8, +2.0] deg,
2083 azimuth steps, sensor 1.73 m above the ground) is ray-cast against an analytic street scene:
ground plane, two rows of box buildings (facades; low boxes expose their tops = "roof"), vertical
cylinders (pillars) and horizontal rails (beams). Every return carries the feature class of the
primitive it hit, the analytic normal (planar classes) or axis direction (linear classes, as MULLS
stores the principal direction in normal_* for pillars/beams, pca.hpp:437-454) perturbed by 2 deg,
and a uniform random intensity. The generator replaces MULLS's CFilter feature extraction for the
benchmark inputs only; it is deterministic in `seed` (numpy PCG64).

Class order everywhere: ground, pillar, facade, beam, roof, vertex (cregistration.hpp:1196-1232).
"""
from __future__ import annotations

import math

import numpy as np

from . import abi

GT_TRANSLATION = (1.00, 0.05, 0.01)
GT_RPY_DEG = (0.2, 0.1, 1.0)
SENSOR_HEIGHT = 1.73


def rpy_matrix(roll: float, pitch: float, yaw: float) -> np.ndarray:
    """x-y'-z'' rotation, the convention of construct_trans_a (cregistration.hpp:2740-2764)."""
    ca, sa = math.cos(roll), math.sin(roll)
    cb, sb = math.cos(pitch), math.sin(pitch)
    cg, sg = math.cos(yaw), math.sin(yaw)
    return np.array(
        [
            [cg * cb, -sg * ca + cg * sb * sa, sg * sa + cg * sb * ca],
            [sg * cb, cg * ca + sg * sb * sa, -cg * sa + sg * sb * ca],
            [-sb, cb * sa, cb * ca],
        ]
    )


def gt_motion() -> np.ndarray:
    T = np.eye(4)
    T[:3, :3] = rpy_matrix(*[math.radians(a) for a in GT_RPY_DEG])
    T[:3, 3] = GT_TRANSLATION
    return T


def make_scene(seed: int) -> dict:
    """Street scene in world coordinates (ground z = 0, street along +x)."""
    rng = np.random.default_rng(seed)
    boxes = []  # (xmin, ymin, zmin, xmax, ymax, zmax)
    for side in (-1.0, 1.0):
        x = -95.0
        while x < 95.0:
            length = rng.uniform(8.0, 22.0)
            depth = rng.uniform(8.0, 14.0)
            off = rng.uniform(8.0, 25.0)
            height = rng.uniform(4.0, 14.0)
            y0, y1 = (off, off + depth) if side > 0 else (-off - depth, -off)
            boxes.append((x, y0, 0.0, x + length, y1, height))
            x += length + rng.uniform(1.0, 7.0)
    for _ in range(26):  # low boxes: tops visible from the sensor -> "roof"
        cx, cy = rng.uniform(-70, 70), rng.uniform(3.0, 7.5) * rng.choice((-1.0, 1.0))
        lx, ly, h = rng.uniform(2.5, 6.0), rng.uniform(1.5, 2.5), rng.uniform(0.5, 1.1)
        boxes.append((cx - lx / 2, cy - ly / 2, 0.0, cx + lx / 2, cy + ly / 2, h))
    pillars = []  # (cx, cy, radius, height)
    for _ in range(60):
        pillars.append((rng.uniform(-60, 60), rng.uniform(3.0, 7.8) * rng.choice((-1.0, 1.0)), 0.15,
                        rng.uniform(4.0, 9.0)))
    rails = []  # (axis, a0, a1, c_other, cz, radius): axis 0 -> along x at (y=c_other, z=cz)
    for _ in range(30):
        axis = int(rng.integers(0, 2))
        length = rng.uniform(6.0, 18.0)
        if axis == 0:
            a0 = rng.uniform(-60, 45)
            other = rng.uniform(2.5, 7.9) * rng.choice((-1.0, 1.0))
        else:
            a0 = rng.uniform(-8.0, 8.0 - 6.0)
            length = min(length, 12.0)
            other = rng.uniform(-55, 55)
        rails.append((axis, a0, a0 + length, other, rng.uniform(0.4, 3.2), 0.10))
    return {"boxes": np.array(boxes), "pillars": np.array(pillars), "rails": np.array(rails)}


def _perturb(v: np.ndarray, rng: np.random.Generator, sigma_deg: float) -> np.ndarray:
    out = v + rng.normal(0.0, math.radians(sigma_deg), v.shape)
    out /= np.linalg.norm(out, axis=1, keepdims=True)
    return out


def scan(scene: dict, pose: np.ndarray, seed: int, n_points: int = 120000, beams: int = 64,
         elev_deg=(-24.8, 2.0), az_steps: int = 2083, range_noise: float = 0.02):
    """Ray-cast one sweep from sensor pose `pose` (4x4, sensor frame -> world with ground at z=0;
    the sensor sits SENSOR_HEIGHT above pose's origin... the pose translation is the sensor position).
    Returns a list of six (n_c, 7) float32 arrays [x y z nx ny nz intensity] in the SENSOR frame."""
    rng = np.random.default_rng(seed)
    el = np.radians(np.linspace(elev_deg[0], elev_deg[1], beams))
    az = np.arange(az_steps) * (2.0 * math.pi / az_steps)
    EL, AZ = np.meshgrid(el, az, indexing="ij")
    d_local = np.stack([np.cos(EL) * np.cos(AZ), np.cos(EL) * np.sin(AZ), np.sin(EL)], axis=-1).reshape(-1, 3)
    R, o = pose[:3, :3], pose[:3, 3]
    d = d_local @ R.T
    n_rays = d.shape[0]
    best_t = np.full(n_rays, np.inf)
    best_cls = np.full(n_rays, -1, dtype=np.int8)
    best_vec = np.zeros((n_rays, 3))

    # ground plane z = 0
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(d[:, 2] < -1e-9, -o[2] / d[:, 2], np.inf)
    m = t < best_t
    best_t[m], best_cls[m] = t[m], abi.GROUND
    best_vec[m] = (0.0, 0.0, 1.0)

    # boxes (slab method, vectorised rays x boxes in chunks)
    B = scene["boxes"]
    inv = 1.0 / np.where(np.abs(d) < 1e-12, 1e-12, d)
    for b0 in range(0, len(B), 16):
        bb = B[b0:b0 + 16]
        t1 = (bb[None, :, 0:3] - o[None, None, :]) * inv[:, None, :]
        t2 = (bb[None, :, 3:6] - o[None, None, :]) * inv[:, None, :]
        tn = np.minimum(t1, t2)
        tf = np.maximum(t1, t2)
        tnear = tn.max(axis=2)
        tfar = tf.min(axis=2)
        axis = tn.argmax(axis=2)
        hit = (tnear <= tfar) & (tnear > 1e-6)
        tt = np.where(hit, tnear, np.inf)
        k = tt.argmin(axis=1)
        tmin = tt[np.arange(n_rays), k]
        ax = axis[np.arange(n_rays), k]
        m = tmin < best_t
        best_t[m] = tmin[m]
        best_cls[m] = np.where(ax[m] == 2, abi.ROOF, abi.FACADE)
        nv = np.zeros((int(m.sum()), 3))
        nv[np.arange(nv.shape[0]), ax[m]] = -np.sign(d[m, ax[m]])
        best_vec[m] = nv

    # vertical cylinders
    for cx, cy, r, h in scene["pillars"]:
        ox, oy = o[0] - cx, o[1] - cy
        a = d[:, 0] ** 2 + d[:, 1] ** 2
        b = 2.0 * (ox * d[:, 0] + oy * d[:, 1])
        c = ox * ox + oy * oy - r * r
        disc = b * b - 4 * a * c
        ok = (disc > 0) & (a > 1e-12)
        sq = np.sqrt(np.where(ok, disc, 0.0))
        t = np.where(ok, (-b - sq) / (2 * np.where(ok, a, 1.0)), np.inf)
        with np.errstate(invalid="ignore"):
            z = o[2] + t * d[:, 2]
            t = np.where((t > 1e-6) & (z >= 0.0) & (z <= h), t, np.inf)
        m = t < best_t
        best_t[m], best_cls[m] = t[m], abi.PILLAR
        best_vec[m] = (0.0, 0.0, 1.0)

    # horizontal rails
    for axis, a0, a1, other, cz, r in scene["rails"]:
        axis = int(axis)
        u = 1 - axis  # the horizontal coordinate perpendicular to the rail
        ou, oz = o[u] - other, o[2] - cz
        a = d[:, u] ** 2 + d[:, 2] ** 2
        b = 2.0 * (ou * d[:, u] + oz * d[:, 2])
        c = ou * ou + oz * oz - r * r
        disc = b * b - 4 * a * c
        ok = (disc > 0) & (a > 1e-12)
        sq = np.sqrt(np.where(ok, disc, 0.0))
        t = np.where(ok, (-b - sq) / (2 * np.where(ok, a, 1.0)), np.inf)
        with np.errstate(invalid="ignore"):
            al = o[axis] + t * d[:, axis]
            t = np.where((t > 1e-6) & (al >= a0) & (al <= a1), t, np.inf)
        m = t < best_t
        best_t[m], best_cls[m] = t[m], abi.BEAM
        vec = np.zeros(3)
        vec[axis] = 1.0
        best_vec[m] = vec

    rough = np.where(best_cls == abi.GROUND, rng.uniform(-0.03, 0.03, n_rays), 0.0)
    rng_m = best_t + rng.normal(0.0, range_noise, n_rays) + rough
    valid = np.isfinite(best_t) & (rng_m > 1.5) & (rng_m < 80.0)
    idx = np.flatnonzero(valid)
    if idx.size > n_points:
        idx = np.sort(rng.choice(idx, size=n_points, replace=False))
    pts = d_local[idx] * rng_m[idx, None]
    vec_local = best_vec[idx] @ R  # world -> sensor frame (R^T v)
    vec_local = _perturb(vec_local, rng, 2.0)
    inten = rng.uniform(0.0, 255.0, idx.size)
    cls = best_cls[idx]
    out = []
    for c in range(abi.NUM_CLASSES):
        m = cls == c
        arr = np.concatenate([pts[m], vec_local[m], inten[m, None]], axis=1).astype(np.float32)
        out.append(arr)
    return out


def cloud_bound(clouds) -> list:
    """block1->local_bound as DataIo::read_pc_cloud_block would set it: bbox of all points."""
    allp = np.concatenate([c[:, :3] for c in clouds if len(c)], axis=0).astype(np.float64)
    mn, mx = allp.min(0), allp.max(0)
    return [mn[0], mn[1], mn[2], mx[0], mx[1], mx[2]]


def kitti_urban_params(max_iter: int = 20) -> abi.IcpParams:
    """SURVEY §8(d) parameter set (script/config/lo_gflag_list_kitti_urban.txt values, roof enabled)."""
    p = abi.default_params()
    p.max_iter_num = max_iter
    p.dis_thre_unit = 1.4
    p.dis_thre_min = 0.5
    p.dis_thre_update_rate = 1.1
    p.used_feature_type = b"111110"
    p.weight_strategy = b"1111"
    p.pt2pt_residual_window = 0.05
    p.pt2pl_residual_window = 0.05
    p.pt2li_residual_window = 0.05
    p.normal_bearing = 20.0
    p.converge_translation = 0.0005
    p.converge_rotation_d = 0.001
    p.apply_intersection_filter = 1
    return p


def _sensor_pose(T: np.ndarray) -> np.ndarray:
    P = T.copy()
    P[2, 3] += SENSOR_HEIGHT
    return P


def make_pair(seed: int, config: str = "c2", n_points: int | None = None, max_iter: int = 20):
    """One benchmark scan pair.

    config: "c2" scan-to-scan 64-beam 120k; "c3" 120k source vs 5-scan 600k map; "c5" 128-beam 300k;
            "small" a 64-beam scan decimated in azimuth (fast CPU tests).
    Returns dict(tgt=[6 arrays (n,12)], src=[6 arrays (n,12)], params, init_guess (4x4), T_gt (4x4)).
    """
    scene = make_scene(seed)
    M = gt_motion()
    kw = dict(n_points=120000, beams=64, elev_deg=(-24.8, 2.0), az_steps=2083)
    if config == "c5":
        kw = dict(n_points=300000, beams=128, elev_deg=(-25.0, 15.0), az_steps=2344)
    elif config == "small":
        kw = dict(n_points=20000, beams=32, elev_deg=(-24.8, 2.0), az_steps=700)
    if n_points is not None:
        kw["n_points"] = n_points
    I4 = np.eye(4)
    if config == "c3":
        # local map = scans at poses M^0..M^4 expressed in frame 0; source = scan at M^5;
        # initial guess = M^4 (the previous pose), so the remaining error is one motion step.
        poses = [I4]
        for _ in range(5):
            poses.append(poses[-1] @ M)
        tgt = [[] for _ in range(abi.NUM_CLASSES)]
        for k in range(5):
            sc = scan(scene, _sensor_pose(poses[k]), seed * 7919 + k, **kw)
            Rk, tk = poses[k][:3, :3], poses[k][:3, 3]
            for c in range(abi.NUM_CLASSES):
                a = sc[c].astype(np.float64)
                a[:, 0:3] = a[:, 0:3] @ Rk.T + tk
                a[:, 3:6] = a[:, 3:6] @ Rk.T
                tgt[c].append(a.astype(np.float32))
        tgt = [np.concatenate(t, axis=0) for t in tgt]
        src = scan(scene, _sensor_pose(poses[5]), seed * 7919 + 5, **kw)
        init, T_gt = poses[4], poses[5]
    else:
        tgt = scan(scene, _sensor_pose(I4), seed * 7919, **kw)
        src = scan(scene, _sensor_pose(M), seed * 7919 + 1, **kw)
        init, T_gt = I4, M
    params = kitti_urban_params(max_iter)
    params.target_bound[:] = cloud_bound(tgt)
    return {
        "tgt": [abi.as_aos48(t) for t in tgt],
        "src": [abi.as_aos48(s) for s in src],
        "params": params,
        "init_guess": np.ascontiguousarray(init, dtype=np.float64),
        "T_gt": T_gt,
    }


def make_sequence(seed: int, n_frames: int, config: str = "small", n_points: int | None = None, max_iter: int = 20):
    """A drive through one scene: `n_frames` sweeps at poses M^0 .. M^(n-1) (the odometry workload of
    test/mulls_slam.cpp: every frame is registered to a local map built from the previous ones).
    Returns dict(scans=[per frame six (n,12) arrays in the SENSOR frame], poses=[4x4 ground truth], params).
    The vertex class — empty in `scan` — is filled with every 37th pillar/facade point so that the local map's
    sixth cloud is exercised too."""
    scene = make_scene(seed)
    M = gt_motion()
    kw = dict(n_points=120000, beams=64, elev_deg=(-24.8, 2.0), az_steps=2083)
    if config == "small":
        kw = dict(n_points=20000, beams=32, elev_deg=(-24.8, 2.0), az_steps=700)
    if n_points is not None:
        kw["n_points"] = n_points
    poses = [np.eye(4)]
    for _ in range(n_frames - 1):
        poses.append(poses[-1] @ M)
    scans = []
    for k in range(n_frames):
        sc = [abi.as_aos48(a) for a in scan(scene, _sensor_pose(poses[k]), seed * 7919 + k, **kw)]
        sc[abi.VERTEX] = np.ascontiguousarray(np.concatenate([sc[abi.PILLAR], sc[abi.FACADE]], axis=0)[::37])
        scans.append(sc)
    return {"scans": scans, "poses": poses, "params": kitti_urban_params(max_iter)}


def make_merged_map(seed: int, n_sweeps: int, n_points: int = 120000, n_copies: int = 1,
                    outlier_ratio: float = 0.002) -> np.ndarray:
    """The cloud test/mulls_slam.cpp:1008-1009 hands to CFilter::sor_filter (pc_map_merged): every sweep of a drive,
    moved by its pose into the map frame, plus `outlier_ratio` of isolated points scattered over the map's box (what the
    filter is there to remove). n_copies > 1 repeats the drive's map shifted 200 m along x each time: a longer street
    from the same sweeps, cheap to make. Returns (n, 12) float32 rows."""
    scene = make_scene(seed)
    M = gt_motion()
    rng = np.random.default_rng(seed)
    pose = np.eye(4)
    parts = []
    for k in range(n_sweeps):
        sc = np.concatenate(scan(scene, _sensor_pose(pose), seed * 7919 + k, n_points=n_points), axis=0).astype(np.float64)
        sc[:, 0:3] = sc[:, 0:3] @ pose[:3, :3].T + pose[:3, 3]
        sc[:, 3:6] = sc[:, 3:6] @ pose[:3, :3].T
        parts.append(sc)
        pose = pose @ M
    drive = np.concatenate(parts, axis=0)
    drive = np.concatenate([drive + np.array([200.0 * c, 0, 0, 0, 0, 0, 0]) for c in range(n_copies)], axis=0)
    lo, hi = drive[:, :3].min(0), drive[:, :3].max(0)
    n_out = int(len(drive) * outlier_ratio)
    out = np.zeros((n_out, 7))
    out[:, :3] = rng.uniform(lo, hi, (n_out, 3))
    out[:, 5] = 1.0
    cloud = np.concatenate([drive, out], axis=0)
    return abi.as_aos48(cloud[rng.permutation(len(cloud))].astype(np.float32))


def pose_error(T_a: np.ndarray, T_b: np.ndarray):
    """Translation (m) and rotation (rad) difference, the formulas of nav/odom_error_compute.h:65-82."""
    dt = float(np.linalg.norm(T_a[:3, 3] - T_b[:3, 3]))
    Rd = T_b[:3, :3].T @ T_a[:3, :3]
    c = max(-1.0, min(1.0, (np.trace(Rd) - 1.0) / 2.0))
    return dt, float(math.acos(c))
