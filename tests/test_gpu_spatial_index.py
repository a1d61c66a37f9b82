"""The Morton-sorted multi-level hashed grid the ingest builds on the device (k_gather's cell counts, k_hash_layout,
k_hash_build), and the two searches that read it — mulls_nn_query and the PCA neighbourhoods of k_pca — against brute
force on adversarial clouds: points on cell boundaries with exact ties, duplicates, a dense spot with more than 1024
neighbours, distances exactly at the search radius, grid extents around the doubling of the level-0 cell, clouds far
from the origin, tiny and empty classes, classes sharing cells, batch neighbours, a hash layout at its last attempt, and
sparse target clouds that need a larger hash pool than their context starts with.

The references are plain numpy:
  nn_ref   — minimum of the float32 FLANN distance (dx*dx + dy*dy) + dz*dz, ties to the lowest original index, a target
             counts only if float64(d2) <= float64(float32(rmax))**2. mulls_nn_query must equal it bit for bit.
  pca_ref  — neighbours with d2 < float32(r*r) (strict), sorted by (d2, original index), truncated to k (k <= 0 or
             k > 1024: 1024, abi.h), fp64 covariance / (n-1), numpy.linalg.eigh. pt_num exact, eigenvalues within
             1e-4 x lambda1, and for 1 <= k <= 64 the device's outputs are bit-identical to the oracle's (test_pca.py).
The CPU tests at the end pin both references to the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from mulls_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THRE = 1.5                      # dis_thre_unit of every registration here: nn_query answers within 2.5 x 1.5 = 3.75 m
RMAX = np.float32(2.5) * np.float32(THRE)
FAR = np.array([6000.0, -3000.0, 40.0])


# ---------------------------------------------------------------- references

def flann_d2(tgt, p):
    d = tgt - p
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]  # float32, FLANN's order


def nn_ref(tgt, q, rmax):
    tgt = np.ascontiguousarray(np.asarray(tgt, np.float32)[:, :3])
    q = np.asarray(q, np.float32)[:, :3]
    idx = np.full(len(q), -1, np.int32)
    d2 = np.full(len(q), np.inf, np.float32)
    if len(tgt) == 0:
        return idx, d2
    r2 = np.float64(np.float32(rmax)) ** 2
    for b in range(0, len(q), 256):
        blk = q[b:b + 256]
        d = tgt[None, :, :] - blk[:, None, :]
        dd = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        j = np.argmin(dd, axis=1)  # first minimum = lowest index
        best = dd[np.arange(len(blk)), j]
        ok = best.astype(np.float64) <= r2
        idx[b:b + 256] = np.where(ok, j, -1)
        d2[b:b + 256] = np.where(ok, best, np.float32(np.inf))
    return idx, d2


def pca_ref(cloud, r, k, stride=1):
    xyz = np.ascontiguousarray(np.asarray(cloud, np.float32)[:, :3])
    n = len(xyz)
    r2 = np.float32(np.float64(r) * np.float64(r))
    kk = 1024 if (k <= 0 or k > 1024) else k
    pt_num = np.zeros(n, np.int32)
    lam = np.zeros((n, 3))
    for i in range(0, n, stride):
        d2 = flann_d2(xyz, xyz[i])
        nb = np.nonzero(d2 < r2)[0]
        nb = nb[np.lexsort((nb, d2[nb]))][:kk]
        pt_num[i] = len(nb)
        if len(nb) > 3:
            P = xyz[nb].astype(np.float64)
            D = P - P.mean(0)
            lam[i] = np.linalg.eigvalsh(D.T @ D / (len(nb) - 1))[::-1]
    return pt_num, lam


# ---------------------------------------------------------------- the grid as the ingest lays it out (numpy)

def spread12(v):
    x = np.asarray(v).astype(np.uint64) & np.uint64(0xfff)
    for s, m in ((16, 0x0000ff0000ff), (8, 0x00f00f00f00f), (4, 0x0c30c30c30c3), (2, 0x249249249249)):
        x = (x | (x << np.uint64(s))) & np.uint64(m)
    return x


def morton36(c):
    return spread12(c[:, 0]) | (spread12(c[:, 1]) << np.uint64(1)) | (spread12(c[:, 2]) << np.uint64(2))


def grid_geometry(tgt_all, thre, shooting):
    """k_pair_setup without the intersection filter: (h0, origin, n_levels) of a pair whose targets are tgt_all"""
    lo = tgt_all.min(0).astype(np.float64)
    ext = float((tgt_all.max(0).astype(np.float64) - lo).max())
    h0 = np.float32(0.125)
    while (ext + 8.0 * float(h0)) * 1.001 > float(h0) * 4092:
        h0 = np.float32(h0 * 2)
    origin = lo.astype(np.float32) - np.float32(2) * h0
    rmax = np.float32(2.5) * np.float32(thre) * np.float32(1.0001)
    L = 2
    while L < 12 and np.float32(0.999) * np.float32(0.5) * h0 * np.float32(1 << (L - 1)) < rmax:
        L += 1
    return h0, origin, (12 if shooting else L)


def cell_coords(xyz, h0, origin):
    inv = np.float32(1) / h0
    return np.floor((np.asarray(xyz, np.float32)[:, :3] - origin) * inv).astype(np.int64)


def count_cells(coords, L):
    """grid cells of one class over the levels below L (what k_gather counts into hash_entries)"""
    m = morton36(coords)
    return int(sum(len(np.unique(m >> np.uint64(3 * l))) for l in range(L)))


def table_cap(attempt, cells):
    want = 4 * cells if attempt == 0 else 2 * cells if attempt == 1 else (5 * cells) // 4 + 1
    cap = 16
    while cap < want:
        cap <<= 1
    return cap


def layout(cells, pool):
    """k_hash_layout: (attempt, [(base, mask)] in (pair, class) order, used), or (None, need of attempt 2, 0)"""
    for attempt in range(3):
        used, tables = 0, []
        for e in cells:
            cap = table_cap(attempt, e)
            if used + cap > pool:
                break
            tables.append((used, cap - 1))
            used += cap
        else:
            return attempt, tables, used
    return None, sum(table_cap(2, e) for e in cells), 0


def pool_of(max_pairs, max_tgt):
    return 12 * max_pairs * max_tgt + 64 * max_pairs * 6  # mulls_create


def pair_cells(tgt_classes, thre=THRE, shooting=False):
    allp = np.concatenate([t[:, :3] for t in tgt_classes if len(t)]).astype(np.float32)
    h0, origin, L = grid_geometry(allp, thre, shooting)
    return [count_cells(cell_coords(t, h0, origin), L) if len(t) else 0 for t in tgt_classes], L


# ---------------------------------------------------------------- adversarial clouds

def lattice(step, nx, ny, nz, seed=0):
    """points on a lattice of spacing `step` (every point on a cell boundary when step = h0/2), shuffled so that
    original index != Morton order"""
    ax = np.arange(max(nx, ny, nz), dtype=np.float32) * np.float32(step)
    g = np.stack(np.meshgrid(ax[:nx], ax[:ny], ax[:nz], indexing="ij"), -1).reshape(-1, 3)
    return g[np.random.default_rng(seed).permutation(len(g))].astype(np.float32)


def boundary_lattice():
    return lattice(0.0625, 24, 24, 6, seed=1)


def triplicates(seed=2):
    rng = np.random.default_rng(seed)
    base = np.concatenate([rng.uniform(-8, 8, (2000, 3)), rng.normal(0, 0.3, (1000, 3))]).astype(np.float32)
    return np.tile(base, (3, 1))[rng.permutation(3 * len(base))]


def dense_spot(seed=3):
    rng = np.random.default_rng(seed)
    spot = (rng.uniform(0, 0.1, (5000, 3)) + [1.0, 1.0, 1.0]).astype(np.float32)
    halo = rng.uniform(-3, 5, (2000, 3)).astype(np.float32)
    return np.concatenate([spot, halo])[rng.permutation(7000)]


def queries_for(tgt, seed, n_on=300, n_near=600, n_out=100):
    tgt = np.asarray(tgt, np.float32)[:, :3]
    rng = np.random.default_rng(seed)
    lo, hi = tgt.min(0), tgt.max(0)
    c = ((lo.astype(np.float64) + hi) / 2).astype(np.float32)
    return np.concatenate([
        tgt[rng.integers(0, len(tgt), n_on)],
        tgt[rng.integers(0, len(tgt), n_near)] + rng.normal(0, 0.2, (n_near, 3)).astype(np.float32),
        (c + rng.uniform(-1, 1, (n_out, 3)) * ((hi - lo) / 2 + 6)).astype(np.float32)]).astype(np.float32)


def lattice_queries(tgt):
    """on lattice points, at lattice-cell centres (8-way ties), on level-0 boundaries, and outside the grid"""
    rng = np.random.default_rng(7)
    o = tgt.min(0)
    return np.concatenate([
        tgt[rng.integers(0, len(tgt), 300)],
        tgt[rng.integers(0, len(tgt), 300)] + np.float32(0.03125),
        o + (rng.integers(-8, 40, (300, 3)) * np.float32(0.125)).astype(np.float32),
        o + rng.uniform(-30, 30, (100, 3)).astype(np.float32)]).astype(np.float32)


def radius_hit_cloud(shift=np.zeros(3)):
    """query sites with a target at exactly 3.75 m (inclusive), and sites whose only target lies one float beyond that
    along x: the next float32 after site.x + 3.75, an exactly representable coordinate (also 6 km from the origin)"""
    sites = np.zeros((20, 3), np.float32)
    sites[:, 0] = np.arange(20) * 20.0
    sites = (sites + shift).astype(np.float32)
    offs = np.array([[3.75, 0, 0], [0, -3.75, 0], [3, 2.25, 0], [0, 2.25, -3]], np.float32)  # |off|^2 = 14.0625 exactly
    hit = sites[:10] + offs[np.arange(10) % 4]
    assert np.array_equal(np.abs(hit - sites[:10]), np.abs(offs[np.arange(10) % 4]))  # no rounding anywhere
    beyond = sites[10:].copy()
    beyond[:, 0] = np.nextafter(sites[10:, 0] + np.float32(3.75), np.float32(np.inf))
    return np.concatenate([hit, beyond]).astype(np.float32), sites


def rows(xyz):
    r = np.zeros((len(xyz), 12), np.float32)
    r[:, :3] = np.asarray(xyz, np.float32)[:, :3]
    r[:, 3] = 1.0
    r[:, 6] = 1.0  # normal (0, 0, 1)
    return r


def make_pair(tgt_classes, n_src=300, seed=0, **params):
    rng = np.random.default_rng(seed)
    tgt = [rows(t) for t in tgt_classes]
    src = []
    for t in tgt_classes:
        s = np.asarray(t, np.float32)[rng.integers(0, len(t), min(n_src, len(t)))] if len(t) else np.zeros((0, 3), np.float32)
        src.append(rows(s + rng.normal(0, 0.02, s.shape).astype(np.float32)))
    p = abi.default_params()
    p.max_iter_num = 1
    p.dis_thre_unit = THRE
    p.apply_intersection_filter = 0
    for k, v in params.items():
        setattr(p, k, v)
    return {"tgt": tgt, "src": src, "params": p, "init_guess": np.eye(4)}


def one_class(t, cls=0):
    return [t if c == cls else np.zeros((0, 3), np.float32) for c in range(6)]


def assert_nn(ctx, cls, q, ref_cloud):
    idx, d2 = ctx.nn_query(cls, q)
    ri, rd = nn_ref(ref_cloud, q, RMAX)
    np.testing.assert_array_equal(idx, ri)
    np.testing.assert_array_equal(d2.view(np.uint32), rd.view(np.uint32))
    return ri


def eigenvalues_close(got, pt, lam, float_far):
    """within 1e-4 x lambda1 of the fp64 reference. pcl::PCA's float mean and covariance (the oracle always, the device
    for 1 <= k <= 64) lose about 1e-3 of lambda1 6 km from the origin (float_far): there the device is held to bit
    equality with the oracle instead."""
    if float_far:
        return True
    sel = pt > 3
    return (np.abs(got[sel].astype(np.float64) - lam[sel]) / (lam[sel, :1] + 1e-12)).max(initial=0) < 1e-4


def assert_pca(ctx, oracle_mod, cloud, r, k, stride, far):
    g = ctx.pca_features(rows(cloud), r, k, stride)
    pt, lam = pca_ref(cloud, r, k, stride)
    np.testing.assert_array_equal(g["pt_num"], pt)
    assert eigenvalues_close(g["eigenvalues"], pt, lam, far and 1 <= k <= 64)
    if 1 <= k <= 64:
        # the float covariance of both sides is bit-identical; an eigenvector is only defined where its eigenvalue is
        # separated from the others (a lattice neighbourhood is often isotropic)
        o = oracle_mod.pca_features(rows(cloud), r, k, stride)
        assert np.array_equal(g["eigenvalues"].view(np.uint32), o["eigenvalues"].view(np.uint32))
        lo = o["eigenvalues"].astype(np.float64)
        gap01 = lo[:, 0] - lo[:, 1] > 1e-3 * lo[:, 0]
        gap12 = lo[:, 1] - lo[:, 2] > 1e-3 * lo[:, 0]
        assert np.array_equal(g["principal"][gap01].view(np.uint32), o["principal"][gap01].view(np.uint32))
        assert np.array_equal(g["normal"][gap01 & gap12].view(np.uint32), o["normal"][gap01 & gap12].view(np.uint32))
    return pt


# ---------------------------------------------------------------- GPU: nn_query and PCA

@pytest.fixture(scope="module")
def ctx():
    from mulls_b200.registration import Context

    c = Context(0, 3, 20000, 40000)
    yield c
    c.close()


def register(ctx, pairs):
    ctx.upload(pairs)
    ctx.run_resident()


NN_CLOUDS = {
    "lattice": lambda: (boundary_lattice(), lattice_queries(boundary_lattice())),
    "triplicates": lambda: (triplicates(), queries_for(triplicates(), 11)),
    "dense_spot": lambda: (dense_spot(), queries_for(dense_spot(), 12)),
}


def nn_cloud(name, far):
    """(targets, queries) of an NN cloud, moved to (+6 km, -3 km, +40 m) when far"""
    if name == "radius_hits":
        return radius_hit_cloud(FAR if far else np.zeros(3))
    tgt, q = NN_CLOUDS[name]()
    if far:  # cell boundaries o + x*h stay exact: same answers 6 km from the origin
        tgt = (tgt + FAR).astype(np.float32)
        q = (q + FAR).astype(np.float32)
    return tgt, q


@pytest.mark.gpu
@pytest.mark.parametrize("far", [False, True])
@pytest.mark.parametrize("name", list(NN_CLOUDS) + ["radius_hits"])
def test_nn_query_equals_brute_force(ctx, name, far):
    tgt, q = nn_cloud(name, far)
    register(ctx, [make_pair(one_class(tgt))])
    ri = assert_nn(ctx, 0, q, tgt)
    assert (ri >= 0).sum() > len(q) // 3
    if name == "radius_hits":
        assert (ri[:10] >= 0).all() and (ri[10:] == -1).all()


@pytest.mark.gpu
@pytest.mark.parametrize("ext", [509.0, 511.0, 20000.0])
def test_nn_query_at_grid_extents_around_the_cell_doubling(ctx, ext):
    rng = np.random.default_rng(int(ext))
    body = rng.uniform(0, ext, (6000, 3)).astype(np.float32)
    corners = np.array([[x, y, z] for x in (0, ext) for y in (0, ext) for z in (0, ext)], np.float32)
    clusters = (corners[:, None, :] + rng.uniform(-1, 1, (8, 50, 3)) * 0.8).reshape(-1, 3)
    tgt = np.concatenate([body, corners, np.clip(clusters, 0, ext)]).astype(np.float32)
    h0, _, _ = grid_geometry(tgt, THRE, False)
    assert h0 == {509.0: 0.125, 511.0: 0.25, 20000.0: 8.0}[ext]
    q = np.concatenate([queries_for(tgt, 13), corners + rng.normal(0, 1.0, corners.shape).astype(np.float32),
                        np.clip(clusters[::5] + np.float32(0.3), 0, ext)]).astype(np.float32)
    register(ctx, [make_pair(one_class(tgt))])
    assert_nn(ctx, 0, q, tgt)


@pytest.mark.gpu
def test_nn_query_tiny_empty_and_shared_cell_classes(ctx):
    rng = np.random.default_rng(14)
    big = rng.uniform(-10, 10, (3000, 3)).astype(np.float32)
    tiny = [np.zeros((0, 3), np.float32), big[:1] + 0.01, np.zeros((0, 3), np.float32), big[1:3] + 0.01, big[3:6] + 0.01]
    classes = [big] + tiny
    register(ctx, [make_pair(classes)])
    q = queries_for(big, 15)
    for c in range(6):
        ri = assert_nn(ctx, c, q, classes[c])
        assert (ri == -1).all() if len(classes[c]) == 0 else (ri >= 0).any()
    # one cloud dealt round-robin into the six classes: neighbouring segments of the sorted keys carry the same Morton
    # codes, and each class must answer from itself alone
    cloud = boundary_lattice()
    dealt = [cloud[c::6] for c in range(6)]
    register(ctx, [make_pair(dealt)])
    q = lattice_queries(cloud)
    for c in range(6):
        assert_nn(ctx, c, q, dealt[c])


@pytest.mark.gpu
def test_nn_query_does_not_depend_on_the_batch_position(ctx):
    tgt = triplicates(seed=16)
    q = queries_for(tgt, 17)
    alone = make_pair(one_class(tgt))
    register(ctx, [alone])
    idx0, d20 = ctx.nn_query(0, q)
    others = [make_pair(one_class((tgt + np.float32(d)).astype(np.float32)), seed=s) for s, d in ((1, 0.03), (2, -0.05))]
    register(ctx, [alone] + others)
    idx1, d21 = ctx.nn_query(0, q)
    np.testing.assert_array_equal(idx1, idx0)
    np.testing.assert_array_equal(d21.view(np.uint32), d20.view(np.uint32))
    assert_nn(ctx, 0, q, tgt)


@pytest.mark.gpu
@pytest.mark.parametrize("shooting", [0, 1])
@pytest.mark.parametrize("mode", ["plain", "filter", "keep_less"])
def test_nn_query_parameter_switches(ctx, oracle_mod, shooting, mode):
    rng = np.random.default_rng(18)
    ground = np.c_[rng.uniform(-30, 30, 6000), rng.uniform(-30, 30, 6000), rng.normal(0, 0.05, 6000)]
    facade = np.c_[rng.uniform(-30, 30, 3000), np.full(3000, 12.0) + rng.normal(0, 0.05, 3000), rng.uniform(0, 8, 3000)]
    pillar = rng.normal(0, 0.1, (800, 3)) + [5.0, -4.0, 2.0]
    classes = [ground.astype(np.float32), pillar.astype(np.float32), facade.astype(np.float32),
               boundary_lattice()[:500] + np.float32(3.0), np.zeros((0, 3), np.float32), triplicates()[:300]]
    pair = make_pair(classes, n_src=1500, normal_shooting_on=shooting,
                     apply_intersection_filter=int(mode == "filter"), keep_less_source_points=int(mode == "keep_less"))
    # the filter keeps the targets inside the source bbox + 1 m: a source that covers part of the scene
    for c in range(6):
        s = pair["src"][c]
        pair["src"][c] = np.ascontiguousarray(s[(s[:, 0] < 10) & (s[:, 1] < 8)])
    _, L = pair_cells(classes, shooting=bool(shooting))
    assert L == (12 if shooting else 7)
    register(ctx, [pair])
    if mode == "plain":
        refs = classes
    else:  # the clouds the reference built its kd-trees on
        _, trees = oracle_mod.icp_run_trees(pair["tgt"], pair["src"], pair["params"], pair["init_guess"])
        refs = [t[:, :3] for t in trees]
        if mode == "keep_less":
            assert len(refs[0]) == len(classes[0]) // 2 and len(refs[2]) == len(classes[2]) // 2
        else:
            assert 0 < len(refs[0]) < len(classes[0])
    for c in range(5):  # (the reference builds no kd-tree for the vertex class, which "111110" leaves unused)
        q = queries_for(classes[c], 19 + c) if len(classes[c]) else queries_for(classes[0], 19)
        idx, d2 = ctx.nn_query(c, q)
        ri, rd = nn_ref(refs[c], q, RMAX)
        np.testing.assert_array_equal(d2.view(np.uint32), rd.view(np.uint32))
        np.testing.assert_array_equal(idx < 0, ri < 0)
        hit = ri >= 0
        # indices: ours point into the caller's cloud, the reference's into the filtered clone — the points coincide
        np.testing.assert_array_equal(classes[c][idx[hit]], refs[c][ri[hit]])


@pytest.mark.gpu
def test_nn_query_with_the_layout_at_its_last_attempt(oracle_mod):
    """a context sized exactly to a sparse target cloud whose grid only fits at load factor 0.8"""
    from mulls_b200.registration import Context

    rng = np.random.default_rng(20)
    tgt = rng.uniform(0, 60, (8000, 3)).astype(np.float32)
    cells, _ = pair_cells(one_class(tgt))
    attempt, _, _ = layout(cells, pool_of(1, 8000))
    assert attempt == 2
    c = Context(0, 1, 8000, 8000)
    try:
        register(c, [make_pair(one_class(tgt))])
        assert_nn(c, 0, queries_for(tgt, 21, n_near=2000), tgt)
    finally:
        c.close()


PCA_CASES = [
    # the cut at k = 10 falls inside the 12-point sqrt(2) shell of the lattice: the tie rule decides the covariance
    ("lattice", 0.1, 10, 1), ("lattice", 0.1, 7, 1), ("lattice", 0.1, 0, 1),
    ("triplicates", 0.5, 20, 1), ("triplicates", 0.5, 0, 2),
    # more than 1024 candidates in the radius: the re-scan path
    ("dense_spot", 0.2, 50, 3), ("dense_spot", 0.2, 100, 3), ("dense_spot", 0.2, 1024, 3), ("dense_spot", 0.2, 0, 3),
    # 0.25 m lattice, radius 0.5: the 6 points at d2 == r2 are outside; k = 20 cuts the 8-point sqrt(3) shell
    ("radius_lattice", 0.5, 0, 1), ("radius_lattice", 0.5, 30, 1), ("radius_lattice", 0.5, 20, 1),
]
PCA_CLOUDS = {"lattice": boundary_lattice, "triplicates": triplicates, "dense_spot": dense_spot,
              "radius_lattice": lambda: lattice(0.25, 10, 10, 6, seed=4)}


@pytest.mark.gpu
@pytest.mark.parametrize("far", [False, True])
@pytest.mark.parametrize("name,r,k,stride", PCA_CASES)
def test_pca_neighbourhoods_equal_brute_force(ctx, oracle_mod, name, r, k, stride, far):
    cloud = PCA_CLOUDS[name]()
    if far:
        cloud = (cloud + FAR).astype(np.float32)
    pt = assert_pca(ctx, oracle_mod, cloud, r, k, stride, far)
    if name == "dense_spot":
        assert (pt == (1024 if k in (0, 1024) else k)).sum() > 1000
    if name == "radius_lattice" and k == 0:
        assert pt.max() == 27  # self + 6 + 12 + 8; the 6 at exactly r are out


# ---------------------------------------------------------------- GPU: the table k_hash_build writes

@pytest.fixture(scope="module")
def grid_lib():
    src = os.path.join(ROOT, "tests", "harness", "grid_device.cu")
    out = os.path.join(ROOT, "tests", "harness", "_build", "libgrid_device.so")
    deps = [src] + [os.path.join(ROOT, "mulls_b200", "csrc", f)
                    for f in ("kernels_ingest.cuh", "device_types.cuh", "device_math.cuh", "grid_key.cuh", "search_core.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false",
                               "-I", os.path.join(ROOT, "include"), "-Xcompiler", "-fPIC", "-shared", "-o", out, src])
    lb = C.CDLL(out)
    P = C.c_void_p
    lb.gd_build.restype = C.c_int
    lb.gd_build.argtypes = [P, C.c_uint32, C.c_int, P, P, P, P, C.c_uint32, P, P, P, P]
    return lb


def synthetic_keys(rng, levels):
    """sorted keys of len(levels) pairs: every (pair, segment) gets a mix of clustered and scattered cells (some stay
    empty), plus filtered-out points (~0) at the tail"""
    keys, coords = [], []
    for p in range(len(levels)):
        for seg in range(12):
            n = [0, 1, 40, 700, 2500][rng.integers(0, 5)] if seg not in (4, 9) else 0
            c = np.concatenate([rng.integers(0, 4096, (n // 2, 3)),
                                rng.integers(0, 4096, (1, 3)) + rng.integers(0, 64, (n - n // 2, 3))]) % 4096
            m = morton36(c.astype(np.uint64))
            keys.append((np.uint64(p * 12 + seg) << np.uint64(36)) | m)
            coords.append(c)
    k = np.concatenate(keys)
    c = np.concatenate(coords)
    o = np.argsort(k, kind="stable")
    k, c = k[o], c[o]
    return np.concatenate([k, np.full(37, np.uint64(0xffffffffffffffff))]), np.concatenate([c, np.zeros((37, 3), np.int64)])


def expected_cells(keys, coords, n_pairs, levels):
    """{(pair, class): sorted [(key_lo, key_hi, children, start, count)]} enumerated from the sorted keys, and the
    segment starts / counts"""
    sg = (keys >> np.uint64(36)).astype(np.int64)
    valid = keys != np.uint64(0xffffffffffffffff)
    seg_start = np.zeros(12 * n_pairs, np.uint32)
    seg_count = np.zeros(12 * n_pairs, np.uint32)
    cells = {}
    for p in range(n_pairs):
        for s in range(12):
            sel = np.nonzero(valid & (sg == p * 12 + s))[0]
            seg_start[12 * p + s] = sel[0] if len(sel) else 0
            seg_count[12 * p + s] = len(sel)
            if s >= 6:
                continue
            m = keys[sel] & np.uint64((1 << 36) - 1)
            out = [np.zeros((0, 5), np.int64)]
            for l in range(levels[p]):
                _, first, inv, cnt = np.unique(m >> np.uint64(3 * l), return_index=True, return_inverse=True,
                                               return_counts=True)
                x, y, z = (coords[sel[first]] >> l).T
                ch = np.zeros(len(first), np.int64)
                if l > 0:
                    np.bitwise_or.at(ch, inv, 1 << ((m >> np.uint64(3 * (l - 1))) & np.uint64(7)).astype(np.int64))
                out.append(np.stack([x | (y << 12) | ((z & 0xff) << 24), (z >> 8) | ((l + 1) << 4), ch, first, cnt], 1))
            cells[(p, s)] = sort_rows(np.concatenate(out))
    return cells, seg_start, seg_count


def sort_rows(a):
    return a[np.lexsort(a.T[::-1])]


@pytest.mark.gpu
@pytest.mark.parametrize("attempt", [0, 1, 2, None])
def test_device_hash_table_holds_exactly_the_cells(grid_lib, attempt):
    rng = np.random.default_rng(30 + (attempt if attempt is not None else 3))
    for run in range(4):
        levels = [2 + (3 * run + p) % 11 for p in range(3)]
        keys, coords = synthetic_keys(rng, levels)
        cells, seg_start, seg_count = expected_cells(keys, coords, 3, levels)
        n_cells = [len(cells[(p, c)]) for p in range(3) for c in range(6)]
        need = [sum(table_cap(a, e) for e in n_cells) for a in range(3)]
        pool = need[attempt] if attempt is not None else need[2] - 1
        exp_attempt, tables, exp_used = layout(n_cells, pool)
        assert exp_attempt == attempt
        used = np.zeros(3, np.uint32)
        base = np.zeros(18, np.uint32)
        mask = np.zeros(18, np.uint32)
        table = np.zeros((pool, 4), np.uint32)
        rc = grid_lib.gd_build(keys.ctypes.data, len(keys), 3, seg_start.ctypes.data, seg_count.ctypes.data,
                               np.asarray(n_cells, np.uint32).ctypes.data, np.asarray(levels, np.int32).ctypes.data, pool,
                               used.ctypes.data, base.ctypes.data, mask.ctypes.data, table.ctypes.data)
        assert rc == 0
        if attempt is None:  # overflow: flagged, nothing laid out (k_hash_clear clears nothing), nothing written
            assert list(used) == [0, 1, need[2]]
            continue
        assert list(used[:2]) == [exp_used, 0]
        assert [(int(b), int(m)) for b, m in zip(base, mask)] == tables
        for t, (p, c) in enumerate((p, c) for p in range(3) for c in range(6)):
            w = table[base[t]:base[t] + mask[t] + 1]
            full = (w[:, 0] != 0) | (w[:, 1] != 0)
            w = w[full].astype(np.int64)
            got = np.stack([w[:, 0], w[:, 1] & 0xffff, w[:, 1] >> 16, w[:, 2], w[:, 3]], 1)
            assert np.array_equal(sort_rows(got), cells[(p, c)]), (p, c, levels[p])


# ---------------------------------------------------------------- GPU: a context holds any target within its capacity

@pytest.mark.gpu
@pytest.mark.parametrize("shooting", [0, 1])
def test_sparse_targets_within_capacity(oracle_mod, shooting):
    """20 000 target points spread over a 500 m cube, in a context created for 20 000 target points: the grid needs more
    hash entries than the pool the context starts with, at every load factor. The pool grows and the call runs again —
    one-shot and resident registrations, and PCA neighbourhoods whose radius asks for more levels."""
    from mulls_b200.registration import Context

    tgt = np.random.default_rng(40).uniform(0, 500, (20000, 3)).astype(np.float32)
    cells, L = pair_cells(one_class(tgt), shooting=bool(shooting))
    assert L == (12 if shooting else 7)
    assert layout(cells, pool_of(1, 20000))[0] is None
    pair = make_pair(one_class(tgt), n_src=2000, normal_shooting_on=shooting)
    c = Context(0, 1, 20000, 20000)
    try:
        res, _ = c.run_batch([pair])
        assert res[0]["iters"] >= 1
        assert_nn(c, 0, queries_for(tgt, 41, n_near=2000), tgt)
        register(c, [pair])  # resident, on the grown pool
        assert_nn(c, 0, queries_for(tgt, 42), tgt)
    finally:
        c.close()
    if shooting:
        return
    # PCA: 20 000 points in a 100 m cube, radius 4 m (9 levels, about 5.6 cells per point)
    cloud = np.random.default_rng(43).uniform(0, 100, (20000, 3)).astype(np.float32)
    assert layout(pair_cells(one_class(cloud), thre=4.0)[0], pool_of(1, 20000))[0] is None
    c = Context(0, 1, 16, 20000)
    try:
        g = c.pca_features(rows(cloud), 4.0, 20, 50)
        pt, lam = pca_ref(cloud, 4.0, 20, 50)
        np.testing.assert_array_equal(g["pt_num"], pt)
        assert (pt > 3).sum() > 300
        o = oracle_mod.pca_features(rows(cloud), 4.0, 20, 50)
        assert np.array_equal(g["eigenvalues"].view(np.uint32), o["eigenvalues"].view(np.uint32))
    finally:
        c.close()


# ---------------------------------------------------------------- CPU: the references agree with the oracle

REF_CLOUDS = {"lattice": boundary_lattice, "triplicates": triplicates, "dense_spot": dense_spot,
              "radius_hits": lambda: radius_hit_cloud()[0], "radius_lattice": PCA_CLOUDS["radius_lattice"]}


@pytest.mark.parametrize("far", [False, True])
@pytest.mark.parametrize("name", ["lattice", "triplicates", "dense_spot", "radius_hits"])
def test_nn_ref_equals_oracle(oracle_mod, name, far):
    tgt, q = nn_cloud(name, far)
    ri, rd = nn_ref(tgt, q, RMAX)
    oi, od = oracle_mod.nn(rows(tgt), rows(q), float(RMAX))
    np.testing.assert_array_equal(ri, oi)
    hit = ri >= 0
    np.testing.assert_array_equal(rd[hit].view(np.uint32), od[hit].view(np.uint32))
    assert hit.sum() > len(q) // 3


@pytest.mark.parametrize("far", [False, True])
@pytest.mark.parametrize("name,r,k,stride", PCA_CASES)
def test_pca_ref_equals_oracle(oracle_mod, name, r, k, stride, far):
    """pt_num exact, eigenvalues within 1e-4 x lambda1. The oracle restates the reference's radius search, which has no
    limit for k <= 0: the 1024 of abi.h is the device kernel's, so there the oracle's counts are capped before the
    comparison and only neighbourhoods of at most 1024 points compare eigenvalues."""
    cloud = PCA_CLOUDS[name]()
    if far:
        cloud = (cloud + FAR).astype(np.float32)
    pt, lam = pca_ref(cloud, r, k, stride)
    o = oracle_mod.pca_features(rows(cloud), r, k, stride)
    np.testing.assert_array_equal(pt, np.minimum(o["pt_num"], 1024))
    same = o["pt_num"] <= 1024
    # (the oracle computes pcl::PCA's float covariance for every k, so far from the origin it is held to the fp64
    # reference only through the device: bit-identical to the oracle for k <= 64, within 1e-4 of pca_ref above)
    assert eigenvalues_close(o["eigenvalues"][same], pt[same], lam[same], far)


def test_layout_restatement_reproduces_the_cell_density_of_a_sparse_cloud():
    """the numpy restatement of the cell counts and of k_hash_layout the GPU tests rely on: 20 000 points spread over a
    500 m cube open about 7 grid cells per point, and the grid needs 262 224 entries at the last attempt — more than the
    12 entries per point a context sizes its pool with, so test_sparse_targets_within_capacity drives the pool's growth"""
    rng = np.random.default_rng(40)
    tgt = rng.uniform(0, 500, (20000, 3)).astype(np.float32)
    cells, L = pair_cells(one_class(tgt))
    assert L == 7 and 6.5 < cells[0] / 20000 < 7.5
    attempt, need, _ = layout(cells, 0)
    assert attempt is None and need == sum(table_cap(2, e) for e in cells) == 262224 > pool_of(1, 20000)
