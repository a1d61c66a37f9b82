"""Adversarial registration scenes for the ICP iteration, shared by the CPU proof that each scene reaches its edge
(test_icp_scenes.py) and the device parity tests (test_gpu_icp_batch.py).

Every scene is the synthetic "small" pair (`synth.make_pair(1000, "small")`) plus placed points, with fixed seeds, returned
as `dict(tgt, src, params, init_guess)`. Each one aims at one rule of determine_corres (cregistration.hpp:1701-1835) or of
the iteration; DESIGN.md §2 and §4 give the rules. Placed structures sit in spots where their class has no other point
within `ISOLATION` metres, so that nothing but the construction decides their matches.

`probe(oracle_mod, pair)` runs the independent numpy restatement of the loop (test_oracle_fullloop_crosscheck.run_loop),
checks it against the oracle in every iteration, and records what determine_corres saw and returned per iteration and
class, so that a test can show that an edge really occurs in the oracle's run."""
import functools
import sys

import numpy as np
from scipy.spatial import cKDTree

import test_oracle_fullloop_crosscheck as fl
from mulls_b200 import abi, synth

F32, F64 = np.float32, np.float64
G, PL, F, B, R, V = abi.GROUND, abi.PILLAR, abi.FACADE, abi.BEAM, abi.ROOF, abi.VERTEX
ISOLATION = 5.0
DEDUP_MIN_SRC = 500  # K_filter_distant_point (cregistration.hpp:1704)


@functools.lru_cache(maxsize=None)
def _base():
    return synth.make_pair(1000, "small")


def base_pair():
    b = _base()
    return dict(tgt=[t.copy() for t in b["tgt"]], src=[s.copy() for s in b["src"]],
                params=abi.IcpParams.from_buffer_copy(b["params"]), init_guess=b["init_guess"].copy())


def rows(xyz, nrm, intensity=100.0):
    """(n, 12) float32 rows: x y z 1, nx ny nz 0, intensity, curvature 0 ..."""
    xyz = np.atleast_2d(np.asarray(xyz, F32))
    nrm = np.broadcast_to(np.asarray(nrm, F32), xyz.shape)
    out = np.zeros((len(xyz), 12), F32)
    out[:, 0:3], out[:, 3], out[:, 4:7], out[:, 8] = xyz, 1.0, nrm, intensity
    return out


def free_spots(pair, c, n, seed, margin=8.0, spacing=2 * ISOLATION):
    """n spots (x, y) inside the pair's extent where class c has no source or target within ISOLATION metres (in xy),
    at least `spacing` apart, on a 1/64 m lattice (exact in float and under small dyadic translations)."""
    tb = np.array(pair["params"].target_bound[:])
    pts = np.concatenate([pair["tgt"][c][:, :2], pair["src"][c][:, :2]]).astype(F64)
    tree = cKDTree(pts) if len(pts) else None
    rng = np.random.default_rng(seed)
    got = []
    for _ in range(200000):
        xy = np.round(rng.uniform(tb[:2] + margin, tb[3:5] - margin) * 64) / 64
        if tree is not None and tree.query(xy)[0] < ISOLATION:
            continue
        if any(np.hypot(*(xy - g)) < spacing for g in got):
            continue
        got.append(xy)
        if len(got) == n:
            return np.array(got)
    raise AssertionError(f"only {len(got)} free spots for class {c}")


def interleave(base, extra, seed):
    """`extra` rows inserted at random positions of `base` (both orders preserved): their indices spread over the class."""
    rng = np.random.default_rng(seed)
    pos = np.sort(rng.choice(len(base) + len(extra), len(extra), replace=False))
    out = np.empty((len(base) + len(extra), 12), F32)
    mask = np.zeros(len(out), bool)
    mask[pos] = True
    out[mask], out[~mask] = extra, base
    return out, pos


def subsample(a, n):
    return a[np.linspace(0, len(a) - 1, n).round().astype(int)] if n else a[:0]


# ---------------------------------------------------------------------------------------------------------------------
# 1. duplicate-check contention
def contention():
    """600 beam sources around one isolated cluster of four beam targets, their indices interleaved with the class's
    1417 others: the first source in index order wins each target (atomicMin on the claim table), across the several
    128-source chunks the cluster spans after the Morton sort. The class then shrinks below 500 in a later iteration."""
    p = base_pair()
    (xy,) = free_spots(p, B, 1, seed=11)
    rng = np.random.default_rng(12)
    tg = np.array([[0.0, 0.0, 0.0], [0.2, 0.0, 0.0], [0.0, 0.2, 0.0], [0.0, 0.0, 0.2]]) + [xy[0], xy[1], 0.0]
    p["tgt"][B] = np.concatenate([p["tgt"][B], rows(tg, (0, 0, 1))])
    d = rng.normal(size=(600, 3))
    d *= (rng.uniform(0.05, 1.2, 600) / np.linalg.norm(d, axis=1))[:, None]
    p["src"][B], pos = interleave(p["src"][B], rows(d + [xy[0], xy[1], 0.0], (0, 0, 1)), seed=13)
    p["contenders"] = pos
    return p


# 2. class sizes around the rules
def class_sizes(sizes, tgt_sizes=None):
    """Source classes cut to the given sizes (evenly over the class); optional target cuts. No intersection filter, so
    that determine_corres sees exactly these sizes."""
    p = base_pair()
    p["params"].apply_intersection_filter = 0
    for c, n in enumerate(sizes):
        if n is not None:
            p["src"][c] = subsample(p["src"][c], n)
    for c, n in (tgt_sizes or {}).items():
        p["tgt"][c] = subsample(p["tgt"][c], n)
    return p


def sizes_a():
    return class_sizes([501, 129, 500, 3, 127, None])


def sizes_b():
    return class_sizes([499, 128, 2, 0, 3, None], {R: 2})


# 3. exact nearest-neighbour ties
def _tilt(n, deg):
    a = np.deg2rad(deg)
    Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    return (n.astype(F64) @ Rz.T).astype(F32)


def ties():
    """Facade: 400 target points duplicated at other indices (half of the copies before the originals, half after), each
    copy's normal turned by 8 degrees, so that the copy chosen changes ATPA. Beam: eight isolated sources with two targets
    placed symmetrically around each (exactly equal float distances), with different line directions."""
    p = base_pair()
    rng = np.random.default_rng(21)
    t = p["tgt"][F]
    pick = rng.choice(len(t), 400, replace=False)
    dup = t[pick].copy()
    dup[:, 4:7] = _tilt(dup[:, 4:7], 8.0)
    p["tgt"][F] = np.concatenate([dup[:200], t, dup[200:]])
    spots = free_spots(p, B, 8, seed=22)
    v = np.array([0.25, 0.125, 0.0625])
    src, tgt = [], []
    for k, (x, y) in enumerate(spots):
        c = np.array([x, y, 0.5])
        src.append(rows(c, (0, 0, 1)))
        first, second = (c + v, c - v) if k % 2 else (c - v, c + v)
        tgt += [rows(first, (0, 0, 1)), rows(second, (0, np.sin(0.2), np.cos(0.2)))]
    p["src"][B] = np.concatenate([p["src"][B]] + src)
    p["tgt"][B] = np.concatenate([p["tgt"][B]] + tgt)
    return p


# 4. threshold edges
def _exact_offset(z0, dz):
    """(z, z + dz) in float with fl(fl(z + dz) - z) == dz exactly."""
    z = F32(z0)
    for _ in range(1000):
        q = F32(z + F32(dz))
        if F32(q - z) == F32(dz):
            return z, q
        z = np.nextafter(z, F32(10))
    raise AssertionError("no exact offset")


def thresholds():
    """Facade (a class with the duplicate check) at identity: in iteration 0 the sources stand where they were placed.
    Four sources with a lone target at float d2 == thre*thre exactly (the rejector keeps only '<'), four at exactly the
    search bound (2.5*thre)^2 = 12.25 (kept: '<=' in double, then dropped by the rejector but surviving the shrink)."""
    p = base_pair()
    thre = F32(p["params"].dis_thre_unit)
    assert F32(F32(2.5) * thre) == F32(3.5)
    spots = free_spots(p, F, 8, seed=31)
    src, tgt = [], []
    for k, (x, y) in enumerate(spots):
        z, q = _exact_offset(-0.7, thre) if k < 4 else (F32(-1.75), F32(1.75))
        src.append(rows((x, y, z), (0, 0, 1)))
        tgt.append(rows((x, y, q), (0, 0, 1)))
    p["src"][F] = np.concatenate([p["src"][F]] + src)
    p["tgt"][F] = np.concatenate([p["tgt"][F]] + tgt)
    return p


COS_PASS_SRC = (1.0, 3 * 2.0 ** -14, 0.0)  # dot with the target normal = 1 - 2^-26: rounds to 1.0f, on cos_thre
COS_FAIL_SRC = (1.0, 2.0 ** -14, 0.0)  # dot = 1 - 0.75 * 2^-24: rounds to 1 - 2^-24, just below
COS_TGT = (1.0 - 2.0 ** -24, 2.0 ** -12, 0.0)


def cos_edge():
    """normal_bearing = 0: cos_thre = cos(0) = 1.0 exactly, so a correspondence passes the normal test only if its float
    |cos| rounds to 1.0. All normals of both clouds are snapped to their dominant axis (|cos| = 1 or 0); four placed pairs
    have a double dot product just below 1 that rounds to 1.0f (kept), four one that rounds below (rejected). Once the first
    increment has turned the source normals no |cos| rounds to 1 any more: the scene ends with -2 in iteration 1."""
    p = base_pair()
    for side in ("tgt", "src"):
        for c in range(6):
            a = p[side][c]
            if len(a):
                n = np.zeros((len(a), 3), F32)
                k = np.abs(a[:, 4:7]).argmax(1)
                n[np.arange(len(a)), k] = np.sign(a[np.arange(len(a)), 4 + k])
                a[:, 4:7] = n
    p["params"].normal_bearing = 0.0
    spots = free_spots(p, F, 8, seed=41)
    src, tgt = [], []
    for k, (x, y) in enumerate(spots):
        src.append(rows((x, y, 0.25), COS_PASS_SRC if k < 4 else COS_FAIL_SRC))
        tgt.append(rows((x + 0.3, y, 0.25), COS_TGT))
    p["src"][F] = np.concatenate([p["src"][F]] + src)
    p["tgt"][F] = np.concatenate([p["tgt"][F]] + tgt)
    return p


# 5. keep-mode certificates
KEEP_N = 40


def _keep_stage(oracle_mod):
    p = base_pair()
    p["params"].converge_translation, p["params"].converge_rotation_d = 0.0, 0.0
    init = p["init_guess"].copy()
    init[0, 3] += 0.6
    init[1, 3] -= 0.4
    p["init_guess"] = init
    spots = free_spots(p, R, KEEP_N, seed=51, spacing=6.0)
    rng = np.random.default_rng(52)
    # the probes are placed in the source frame; their first targets 0.3 m off where the base registration takes them
    base_traj = _keep_base_positions(oracle_mod)
    srcs = rows(np.c_[spots, rng.uniform(-1.0, 1.0, KEEP_N)], (0, 0, 1))
    p2 = fl.rigid(srcs, base_traj[2])
    ang = rng.uniform(0, 2 * np.pi, KEEP_N)
    first = p2[:, 0:3].astype(F64) + 0.3 * np.c_[np.cos(ang), np.sin(ang), np.zeros(KEEP_N)]
    p["src"][R] = np.concatenate([p["src"][R], srcs])
    p["tgt"][R] = np.concatenate([p["tgt"][R], rows(first, (0, 0, 1))])
    return p


@functools.lru_cache(maxsize=None)
def _keep_base_positions(oracle_mod):
    """The accumulated pose at the start of iterations 0..3 of the base pair under the keep scene's initial guess."""
    p = base_pair()
    p["params"].converge_translation, p["params"].converge_rotation_d = 0.0, 0.0
    init = p["init_guess"].copy()
    init[0, 3] += 0.6
    init[1, 3] -= 0.4
    _, tr = oracle_mod.icp_run(p["tgt"], p["src"], p["params"], init)
    poses = [init]
    for x in tr["x"][:3]:
        poses.append(fl.increment_matrix(x) @ poses[-1])
    return poses


KEEP_EPS = 6e-5


@functools.lru_cache(maxsize=None)
def keep_mode(oracle_mod):
    """Roof (< 500 sources, no shrinking, so a source keeps its row): 40 isolated probes, all 20 iterations, a non-identity
    initial guess. Each probe's first target is its match up to iteration 2, where its certificate is made. A second
    target is then placed on the ray of the probe's motion from iteration 2 to 3, KEEP_EPS closer to its iteration-3
    position than the first: that small move makes it the nearest, just inside what a slightly too large certificate
    radius would wrongly keep. A second target is placed only where the oracle-equivalent trajectory of the scene without
    it shows the first target nearest in iterations 0-2 and the second nearest in iteration 3."""
    p = _keep_stage(oracle_mod)
    rec = probe(oracle_mod, p)
    pos = {it: rec[(it, R)]["src"][-KEEP_N:] for it in range(4)}  # (the probes are the last rows)
    Fq = p["tgt"][R][-KEEP_N:]
    second = []
    for k in range(KEEP_N):
        a, b = pos[2][k, 0:3].astype(F64), pos[3][k, 0:3].astype(F64)
        m = np.linalg.norm(b - a)
        if m < 10 * KEEP_EPS:
            continue
        e = (b - a) / m
        f3 = np.sqrt(fl.l2_simple(pos[3][k:k + 1, 0:3], Fq[k:k + 1, 0:3])[0])
        s = rows(b + (float(f3) - KEEP_EPS) * e, (0, 0, 1))
        d = lambda it, q: fl.l2_simple(pos[it][k:k + 1, 0:3], q[:, 0:3])[0]
        if all(d(it, s) > d(it, Fq[k:k + 1]) for it in range(3)) and d(3, s) < d(3, Fq[k:k + 1]):
            second.append(s)
    assert len(second) >= KEEP_N // 2, len(second)
    p["tgt"][R] = np.concatenate([p["tgt"][R]] + second)
    p["n_second"] = len(second)
    return p


# 6. the intersection filter and the grid
BOUND_SHIFT = (0.5, 0.25, 0.0)


def bound_faces():
    """A target_bound inside the clouds' extent, so that the filter's box is target_bound -/+ 1 m, and an initial guess
    that is a dyadic translation (exact in float). Sources (in every filtered class) and targets are placed exactly on
    the box's x and y faces (excluded: the filter is strict) and one float step inside (included); the included sources
    sit at the edge of the target cloud, where the moving pose carries them towards and away from their matches."""
    p = base_pair()
    tb = np.array(p["params"].target_bound[:])
    lo = np.ceil(tb[:3]) + [6, 3, 0]
    hi = np.floor(tb[3:]) - [6, 3, 0]
    lo[2], hi[2] = tb[2], tb[5]
    p["params"].target_bound[:] = [lo[0], lo[1], lo[2], hi[0], hi[1], hi[2]]
    init = np.eye(4)
    init[:3, 3] = BOUND_SHIFT
    p["init_guess"] = init
    face_lo, face_hi = lo[:2] - 1.0, hi[:2] + 1.0
    rng = np.random.default_rng(61)
    placed = []
    for axis in (0, 1):
        for face, inward in ((face_lo[axis], np.inf), (face_hi[axis], -np.inf)):
            for step in (0, 1):
                v = F32(face) if step == 0 else np.nextafter(F32(face), F32(inward))
                for _ in range(6):
                    xyz = np.empty(3, F32)
                    other = 1 - axis
                    xyz[other] = F32(np.round(rng.uniform(lo[other] + 2, hi[other] - 2) * 64) / 64)
                    xyz[2] = F32(np.round(rng.uniform(-1.0, 1.0) * 64) / 64)
                    xyz[axis] = v
                    placed.append(xyz)
    placed = np.array(placed, F32)
    src_xyz = placed - np.array(BOUND_SHIFT, F32)  # the initial guess moves them back onto the faces exactly
    for c in (G, PL, F):
        p["src"][c] = np.concatenate([p["src"][c], rows(src_xyz, (0, 0, 1))])
        p["tgt"][c] = np.concatenate([p["tgt"][c], rows(placed + np.array([0.05, 0.05, 0.0], F32), (0, 0, 1))])
    p["face_points"] = placed
    p["faces"] = (face_lo, face_hi)
    return p


def deep_grid():
    """No intersection filter, and three facade targets far out (1.4 km across): the class's grid doubles its finest cell
    (the Morton code holds 4096 cells per axis) and so has more levels above the search radius's."""
    p = base_pair()
    p["params"].apply_intersection_filter = 0
    far = rows([(700.0, 3.0, 0.0), (-700.0, -3.0, 0.0), (0.0, 650.0, 1.0)], (1, 0, 0))
    p["tgt"][F] = np.concatenate([p["tgt"][F][:1000], far, p["tgt"][F][1000:]])
    return p


NAMES = ("contention", "sizes_a", "sizes_b", "ties", "thresholds", "cos_edge", "keep_mode", "bound_faces", "deep_grid")


def scenes_by_name(oracle_mod, name):
    return keep_mode(oracle_mod) if name == "keep_mode" else globals()[name]()


def scenes(oracle_mod):
    """name -> scene, in a fixed order"""
    return {n: scenes_by_name(oracle_mod, n) for n in NAMES}


# ---------------------------------------------------------------------------------------------------------------------
def probe(oracle_mod, pair, min_iters=4):
    """Run the numpy restatement of the loop, require the oracle's code, iteration count and per-class counts in every
    iteration and its pose, and return {(iteration, class): dict(src = the moved sources determine_corres saw, tgt, thre, nn = (index, float d2)
    of every source's nearest target (ties to the lower index), out = (shrunk sources, source rows, target rows, d2) of
    the correspondences it returned)}."""
    rec = {}
    inner = fl.correspondences

    def recording(src, tgt, thre, normal_check, cos_thre, normal_shooting=False):
        f = sys._getframe(1).f_locals
        out = inner(src, tgt, thre, normal_check, cos_thre, normal_shooting)
        nn = fl.nearest(tgt, src) if len(src) and len(tgt) else None
        rec[(f["it"], f["c"])] = dict(src=src, tgt=tgt, thre=thre, cos_thre=cos_thre, nn=nn, out=out)
        return out

    fl.correspondences = recording
    try:
        mine, log = fl.run_loop(pair)
    finally:
        fl.correspondences = inner
    res, tr = oracle_mod.icp_run(pair["tgt"], pair["src"], pair["params"], pair["init_guess"])
    assert (mine["code"], mine["iters"]) == (res["code"], res["iters"]) and res["iters"] >= min_iters
    for it, e in enumerate(log):  # the matches recorded here are the oracle's: equal counts in every iteration
        np.testing.assert_array_equal(e["n_corr"], tr["n_corr"][it], err_msg=f"correspondences, iteration {it}")
        np.testing.assert_array_equal(e["n_src"], tr["n_src"][it], err_msg=f"source sizes, iteration {it}")
    np.testing.assert_allclose(mine["T"], res["T"], rtol=0, atol=1e-9)
    rec["result"], rec["trace"], rec["log"] = res, tr, log
    return rec
