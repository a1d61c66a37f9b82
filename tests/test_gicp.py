"""CPU checks of the voxelized GICP registration (CRegistration::omp_gicp, cregistration.hpp:1024-1098, FastVGICP):
- the CPU restatement (tests/harness/gicp_oracle.cpp, the host instantiation of mulls_b200/csrc/gicp_core.cuh), the
  checker of mulls_omp_gicp, against independent numpy / scipy code: the 20-neighbour lists (ties at the 20th distance,
  duplicates) exactly, covariances against numpy's SVD, voxel coordinates on cell borders exactly, voxel means and
  covariances, the summed loss terms at fixed poses, SO3 exp / log / product against scipy, the LLT solve;
- the whole walk against a numpy walk started from the same x0 (iteration count, final pose);
- the rand() stream: 3 draws for a normal call, 3 + 6 * 64 when no source point ever hits a voxel;
- edge cases: 19 / 20 points, empty clouds, non-finite rows, a filter that empties a cloud, a non-identity guess;
- the drop-in member replays the mulls_slam call sites against a stand-in reference (tests/stubs/gicp_caller.cpp);
- the ctypes structs mirror abi.h."""
import ctypes as C
import inspect
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from test_ndt import bbox, moved, rot, rows, structured_scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
_LIBS = {}
LIBC = C.CDLL("libc.so.6")
LIBC.rand.restype = C.c_int


def gicp_oracle_lib(out_dir=None):
    out_dir = out_dir or os.path.join(ROOT, "tests", "harness", "_build")
    if out_dir in _LIBS:
        return _LIBS[out_dir]
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available: the host instantiation of gicp_core.cuh cannot be built")
    src = os.path.join(ROOT, "tests", "harness", "gicp_oracle.cpp")
    deps = [src] + [os.path.join(ROOT, "mulls_b200", "csrc", f)
                    for f in ("gicp_core.cuh", "ndt_core.cuh", "ransac_core.cuh", "ground_core.cuh")]
    deps.append(os.path.join(ROOT, "include", "mulls_b200", "abi.h"))
    out = os.path.join(out_dir, "libgicp_oracle.so")
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
    dp, fp, ip, vp = C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_int), C.c_void_p
    lb.orc_gicp.restype = C.c_int
    lb.orc_gicp.argtypes = [vp, C.c_long, vp, C.c_long, C.c_float, dp, C.c_int, C.c_float, dp, dp,
                            C.POINTER(abi.GicpResult), C.POINTER(abi.GicpIter), C.c_int]
    lb.orc_gicp_covariances.argtypes = [vp, C.c_long, vp]
    lb.orc_gicp_neighbours.argtypes = [vp, C.c_long, vp]
    lb.orc_gicp_voxels.restype = C.c_long
    lb.orc_gicp_voxels.argtypes = [vp, C.c_long, C.c_float, C.c_long, vp, vp, vp, vp]
    lb.orc_gicp_eval.argtypes = [vp, C.c_long, vp, C.c_long, C.c_float, vp, vp]
    lb.orc_gicp_voxel_coord.argtypes = [vp, C.c_long, C.c_float, vp]
    for f in ("orc_gicp_so3_exp", "orc_gicp_so3_log", "orc_gicp_transform"):
        getattr(lb, f).argtypes = [vp, vp]
    lb.orc_gicp_so3_mul.argtypes = [vp, vp, vp]
    lb.orc_gicp_llt_solve.argtypes = [vp, vp, vp]
    _LIBS[out_dir] = lb
    return lb


def _p(a):
    return a.ctypes.data


def xyz32(a):
    return np.ascontiguousarray(np.asarray(a, F32).reshape(-1, 3))


def oracle_gicp(case, trace_cap=64, seed=1234):
    """the restatement on a case dict (tgt, src, optional guess, tb, sb, filter, res, thre), after srand(seed): a dict
    like Context.omp_gicp's plus `rc` and `draws` (the rand() draws the call consumed)"""
    from mulls_b200 import abi
    lb = gicp_oracle_lib()
    t, s = rows(case["tgt"]), rows(case["src"])
    g = np.ascontiguousarray(case.get("guess", np.eye(4)), np.float64).ravel().copy()
    tb = np.ascontiguousarray(case.get("tb", bbox(case["tgt"])), np.float64)
    sb = np.ascontiguousarray(case.get("sb", bbox(case["src"])), np.float64)
    res = abi.GicpResult()
    tr = (abi.GicpIter * trace_cap)()
    dp = C.POINTER(C.c_double)
    LIBC.srand(seed)
    rc = lb.orc_gicp(_p(t), len(t), _p(s), len(s), case.get("res", 1.0), g.ctypes.data_as(dp), int(case.get("filter", False)),
                     case.get("thre", 10.0), tb.ctypes.data_as(dp), sb.ctypes.data_as(dp), C.byref(res), tr, trace_cap)
    nxt = LIBC.rand()
    out = dict(rc=rc, code=res.code, trans=np.array(res.trans[:]).reshape(4, 4), iterations=res.iterations,
               converged=bool(res.converged), fitness=res.fitness, n_target=res.n_target, n_source=res.n_source,
               x0=np.array(res.x0[:], F32), next_rand=nxt, draws=draws_until(seed, nxt))
    k = min(res.iterations, trace_cap)
    out["trace"] = dict(x=np.array([tr[i].x[:] for i in range(k)], F32).reshape(k, 6),
                        delta=np.array([tr[i].delta[:] for i in range(k)], F32).reshape(k, 6),
                        n_corr=np.array([tr[i].n_corr for i in range(k)], np.int32),
                        random_step=np.array([tr[i].random_step for i in range(k)], np.int32))
    return out


def draws_until(seed, nxt, limit=2000):
    """how many rand() draws after srand(seed) precede the value nxt"""
    LIBC.srand(seed)
    for n in range(limit):
        if LIBC.rand() == nxt:
            return n
    return -1


def cases():
    out = {}
    tgt = structured_scene(6000, 1)
    R, t = rot(0.01, -0.015, 0.03), np.array([0.15, -0.1, 0.05])
    src = moved(tgt[::2] + np.random.default_rng(2).normal(0, 0.02, (3000, 3)).astype(F32), R.T, -R.T @ t)
    out["motion"] = dict(tgt=tgt, src=src)
    out["motion_res03"] = dict(tgt=tgt, src=src, res=0.3)
    out["motion_res07"] = dict(tgt=tgt, src=src, res=0.7)
    out["motion_filter"] = dict(tgt=tgt, src=src, filter=True)
    G = np.eye(4)
    G[:3, :3], G[:3, 3] = rot(0.0, 0.0, 0.02), [0.1, 0.0, 0.0]
    out["guess"] = dict(tgt=tgt, src=src, guess=G)
    nf = src.copy()
    nf[::97, 0] = np.nan
    nf[5::101, 2] = np.inf
    nft = tgt.copy()
    nft[3::89, 1] = -np.inf
    out["non_finite"] = dict(tgt=nft, src=nf)
    dup = np.concatenate([tgt[:3000], tgt[:200]])  # duplicated points: zero distances tie on the index
    out["duplicates"] = dict(tgt=dup, src=src)
    # no source point lands in a target voxel: every solve is non-finite, 64 random steps
    out["no_voxel"] = dict(tgt=tgt, src=src + F32(500.0), thre=1e12)
    out["twenty"] = dict(tgt=tgt[:20], src=src[:20], thre=1e12)
    return out


REFUSED = {  # MULLS_E_UNSUPPORTED
    "nineteen_src": lambda c: dict(tgt=c["tgt"], src=c["src"][:19]),
    "nineteen_tgt": lambda c: dict(tgt=c["tgt"][:19], src=c["src"]),
    "empty_source": lambda c: dict(tgt=c["tgt"], src=np.zeros((0, 3), F32)),
    "empty_target": lambda c: dict(tgt=np.zeros((0, 3), F32), src=c["src"]),
    "filter_empties": lambda c: dict(tgt=c["tgt"], src=c["src"] + F32(1000.0), filter=True),
    "huge_coords": lambda c: dict(tgt=np.concatenate([c["tgt"], [[3e6, 0, 0]]]).astype(F32), src=c["src"], res=1.0),
}


# ---------------------------------------------------------------------------------------------------------------------
# the independent restatement (float64 where the reference is float, so tolerances apply)
# ---------------------------------------------------------------------------------------------------------------------
def np_neighbours(xyz, k=20):
    xyz = xyz32(xyz)
    d = xyz[:, None, :] - xyz[None, :, :]  # query minus point, float32
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    idx = np.broadcast_to(np.arange(len(xyz)), d2.shape)
    return np.stack([np.lexsort((idx[i], d2[i]))[:k] for i in range(len(xyz))])


def np_covariances(xyz):
    xyz = xyz32(xyz).astype(np.float64)
    nb = np_neighbours(xyz)
    out = np.empty((len(xyz), 3, 3))
    for i in range(len(xyz)):
        d = xyz[nb[i]] - xyz[nb[i]].mean(0)
        U, _, Vt = np.linalg.svd(d.T @ d)
        out[i] = U @ np.diag([1.0, 1.0, 1e-2]) @ Vt
    return out


def np_coord(x, res):
    return np.floor(np.asarray(x, F32) / F32(res) - F32(0.5)).astype(np.int64)


def np_voxels(xyz, covs, res):
    c = np_coord(xyz, res)
    vox = {}
    for i, key in enumerate(map(tuple, c)):
        vox.setdefault(key, []).append(i)
    return {k: (len(v), np.asarray(xyz, np.float64)[v].mean(0), covs[v].mean(0)) for k, v in vox.items()}


def np_terms(tgt, src, res, T, tcov=None, scov=None):
    """the 21 + 6 sums and the count at the float transform T (rows 0..2, float32 from the restatement, so that the
    voxel lookups agree), the rest in float64"""
    tcov = np_covariances(tgt) if tcov is None else tcov
    scov = np_covariances(src) if scov is None else scov
    V = np_voxels(tgt, tcov, res)
    T32 = np.asarray(T, F32).reshape(3, 4)
    s32 = xyz32(src)
    ta32 = ((T32[:, 0] * s32[:, :1] + T32[:, 1] * s32[:, 1:2]) + T32[:, 2] * s32[:, 2:3]) + T32[:, 3]
    R, t = T32[:, :3].astype(np.float64), T32[:, 3].astype(np.float64)
    JJ, Je, n = np.zeros((6, 6)), np.zeros(6), 0
    for i, key in enumerate(map(tuple, np_coord(ta32, res))):
        if key not in V:
            continue
        _, mb, cb = V[key]
        ta = R @ s32[i].astype(np.float64) + t
        M = np.linalg.inv(cb + R @ scov[i] @ R.T)
        e = M @ (mb - ta)
        sk = np.array([[0, -ta[2], ta[1]], [ta[2], 0, -ta[0]], [-ta[1], ta[0], 0]])
        J = np.hstack([M @ sk, -M])
        JJ += J.T @ J
        Je += J.T @ e
        n += 1
    return JJ, Je, n


def np_walk(tgt, src, res, x0, max_it=64):
    """FastVGICP's walk in float64 with scipy's SO3, from x0: (iterations, final 4x4)"""
    tcov, scov = np_covariances(tgt), np_covariances(src)
    x = np.asarray(x0, np.float64).copy()
    for it in range(max_it):
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = Rotation.from_rotvec(x[:3]).as_matrix(), x[3:]
        JJ, Je, _ = np_terms(tgt, src, res, T[:3].astype(F32), tcov, scov)
        d = np.linalg.solve(JJ, Je)
        x[:3] = (Rotation.from_rotvec(-d[:3]) * Rotation.from_rotvec(x[:3])).as_rotvec()
        x[3:] -= d[3:]
        Rd = Rotation.from_rotvec(d[:3]).as_matrix() - np.eye(3)
        if max(500.0 * np.abs(Rd).max(), 2000.0 * np.abs(d[3:]).max()) < 1:
            break
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = Rotation.from_rotvec(x[:3]).as_matrix(), x[3:]
    return it + 1, T


# ---------------------------------------------------------------------------------------------------------------------
def lattice_with_ties():
    """integer lattice points (many equal distances at the 20th neighbour) plus duplicates"""
    g = np.stack(np.meshgrid(np.arange(6), np.arange(6), np.arange(3), indexing="ij"), -1).reshape(-1, 3).astype(F32)
    return np.concatenate([g, g[::7]]).astype(F32)


def test_neighbour_lists_in_flann_order():
    lb = gicp_oracle_lib()
    for xyz in (lattice_with_ties(), structured_scene(600, 4)):
        xyz = xyz32(xyz)
        out = np.zeros((len(xyz), 20), np.int32)
        lb.orc_gicp_neighbours(_p(xyz), len(xyz), _p(out))
        np.testing.assert_array_equal(out, np_neighbours(xyz))


def test_covariances_against_numpy_svd():
    lb = gicp_oracle_lib()
    rng = np.random.default_rng(5)
    for xyz in (structured_scene(800, 7), lattice_with_ties() + rng.normal(0, 1e-3, (len(lattice_with_ties()), 3)).astype(F32)):
        xyz = xyz32(xyz)
        out = np.zeros((len(xyz), 9), F32)
        lb.orc_gicp_covariances(_p(xyz), len(xyz), _p(out))
        ref = np_covariances(xyz)
        np.testing.assert_allclose(out.reshape(-1, 3, 3), ref, atol=2e-4)


def test_voxel_coords_on_borders_and_voxels():
    lb = gicp_oracle_lib()
    res = 0.3  # not a power of two: x / res rounds
    k = np.arange(-40, 40, dtype=np.float64)
    border = np.stack([(k + 0.5) * res, (k + 1.5) * res, k * res], 1).astype(F32)  # (k + 0.5) res is a cell border
    coords = np.zeros(border.shape, np.int32)
    lb.orc_gicp_voxel_coord(_p(border), len(border), F32(res), _p(coords))
    np.testing.assert_array_equal(coords, np_coord(border, res))
    xyz = xyz32(np.concatenate([structured_scene(1500, 9), border]))
    n = lb.orc_gicp_voxels(_p(xyz), len(xyz), F32(res), 0, None, None, None, None)
    keys, cnt = np.zeros(n, np.uint64), np.zeros(n, np.int32)
    mean, cov = np.zeros((n, 3), F32), np.zeros((n, 9), F32)
    lb.orc_gicp_voxels(_p(xyz), len(xyz), F32(res), n, _p(keys), _p(cnt), _p(mean), _p(cov))
    # the points on a line have no unique PLANE covariance: the voxels average the restatement's own covariances
    # (checked against numpy above)
    covs = np.zeros((len(xyz), 9), F32)
    lb.orc_gicp_covariances(_p(xyz), len(xyz), _p(covs))
    V = np_voxels(xyz, covs.reshape(-1, 3, 3).astype(np.float64), res)
    assert n == len(V)
    bias = 1 << 20
    for i in range(n):
        key = tuple(int((int(keys[i]) >> s) & ((1 << 21) - 1)) - bias for s in (42, 21, 0))
        c, m, cv = V[key]
        assert cnt[i] == c
        np.testing.assert_allclose(mean[i], m, rtol=1e-6, atol=1e-5)
        np.testing.assert_allclose(cov[i].reshape(3, 3), cv, atol=1e-6)


@pytest.mark.parametrize("res", [1.0, 0.5])
def test_loss_terms_at_fixed_poses(res):
    lb = gicp_oracle_lib()
    tgt = xyz32(structured_scene(2000, 11))
    src = xyz32(moved(tgt[::2], rot(0.005, 0.0, -0.01), np.array([0.05, -0.03, 0.0])))
    tcov, scov = np_covariances(tgt), np_covariances(src)
    for x in (np.array([0.003, -0.002, 0.004, 0.01, 0.02, -0.01], F32), np.zeros(6, F32)):
        out = np.zeros(28)
        lb.orc_gicp_eval(_p(tgt), len(tgt), _p(src), len(src), F32(res), _p(x), _p(out))
        T = np.zeros(12, F32)
        lb.orc_gicp_transform(_p(x), _p(T))
        JJ, Je, n = np_terms(tgt, src, res, T, tcov, scov)
        assert out[27] == n and n > 100
        lo = np.tril_indices(6)
        tri = np.array([JJ[a, b] for a in range(6) for b in range(a + 1)])
        np.testing.assert_allclose(out[:21], tri, rtol=2e-3, atol=2e-3 * np.abs(tri).max())
        np.testing.assert_allclose(out[21:27], Je, rtol=2e-3, atol=2e-3 * np.abs(Je).max())
        del lo


def quat_wxyz(r):
    q = r.as_quat()  # x y z w
    return np.array([q[3], q[0], q[1], q[2]])


@pytest.mark.parametrize("angle", [0.0, 1e-7, 3e-6, 1e-3, 0.5, 2.0, np.pi - 1e-3])
def test_so3_against_scipy(angle):
    lb = gicp_oracle_lib()
    axis = np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8])
    v = (axis * angle).astype(F32)
    q = np.zeros(4, F32)
    lb.orc_gicp_so3_exp(_p(v), _p(q))
    ref = quat_wxyz(Rotation.from_rotvec(v.astype(np.float64)))
    np.testing.assert_allclose(q, ref, atol=2e-7 * max(1.0, angle) + 1e-7)
    back = np.zeros(3, F32)
    lb.orc_gicp_so3_log(_p(q), _p(back))
    np.testing.assert_allclose(back, v, atol=3e-6 * max(1.0, angle))
    w = np.array([-0.2, 0.1, 0.05], F32)
    qw, qm = np.zeros(4, F32), np.zeros(4, F32)
    lb.orc_gicp_so3_exp(_p(w), _p(qw))
    lb.orc_gicp_so3_mul(_p(qw), _p(q), _p(qm))
    ref = quat_wxyz(Rotation.from_rotvec(w.astype(np.float64)) * Rotation.from_rotvec(v.astype(np.float64)))
    if ref[0] * qm[0] < 0:
        ref = -ref
    np.testing.assert_allclose(qm, ref, atol=1e-6)
    assert abs(np.linalg.norm(qm.astype(np.float64)) - 1) < 1e-6


def np_partial_llt(A):
    """the factor gicp_core.cuh's LLT reading (G4) leaves, built from numpy's Cholesky: the first k columns are the
    Cholesky factor of the leading k x k block and its L21 = A21 L11^-T, where k is the first leading block that is
    not positive definite; the rest of the lower triangle is A's, untouched. Returns (L, k)."""
    A = np.asarray(A, np.float64)
    L = np.tril(A).copy()
    k = 6
    for m in range(1, 7):
        try:
            np.linalg.cholesky(A[:m, :m])
        except np.linalg.LinAlgError:
            k = m - 1
            break
    if k:
        L11 = np.linalg.cholesky(A[:k, :k])
        L[:k, :k] = L11
        L[k:, :k] = A[k:, :k] @ np.linalg.inv(L11).T
    return L, k


def test_llt_solve():
    """the LLT step against numpy / scipy: an SPD system as np.linalg.solve; systems whose factorisation stops at a
    zero (k = 1) or negative (k = 2) pivot as triangular solves (scipy) with the factor the reading leaves; the zero
    system, where 0 / 0 at k = 0 makes every entry NaN"""
    from scipy.linalg import solve_triangular

    lb = gicp_oracle_lib()
    rng = np.random.default_rng(8)
    J = rng.normal(size=(40, 6))
    b = rng.normal(size=6)

    def solve(A):
        A = np.ascontiguousarray(A, np.float64)
        x = np.zeros(6)
        lb.orc_gicp_llt_solve(_p(A), _p(b), _p(x))
        return x

    spd = J.T @ J
    np.testing.assert_allclose(solve(spd), np.linalg.solve(spd, b), rtol=1e-9)
    zero_pivot = np.array([[4, 2, 1, 0, 0, 0], [2, 1, 3, 0, 0, 0], [1, 3, 6, 1, 0, 0], [0, 0, 1, 5, 1, 0],
                           [0, 0, 0, 1, 4, 1], [0, 0, 0, 0, 1, 3]], np.float64)  # 1 - (2 / 2)^2 = 0 exactly
    negative_pivot = spd.copy()
    negative_pivot[2, 2] = 1e-3  # the Schur complement at k = 2 is negative
    for A, k_expect in ((zero_pivot, 1), (negative_pivot, 2)):
        L, k = np_partial_llt(A)
        assert k == k_expect
        ref = solve_triangular(L.T, solve_triangular(L, b, lower=True), lower=False)
        np.testing.assert_allclose(solve(A), ref, rtol=1e-10, atol=1e-12 * np.abs(ref).max())
    x = solve(np.zeros((6, 6)))
    assert np.isnan(x).all()  # y_0 = 0 / 0 and every later entry takes it in: the random fallback fires


@pytest.mark.parametrize("name,res", [("motion", 1.0), ("motion", 0.5)])
def test_walk_against_numpy(name, res):
    c = dict(cases()[name], res=res)
    tgt, src = xyz32(c["tgt"])[::2], xyz32(c["src"])[::2]
    o = oracle_gicp(dict(tgt=tgt, src=src, res=res))
    assert o["rc"] == 0 and o["converged"]
    it, T = np_walk(tgt, src, res, o["x0"])
    assert it == o["iterations"]
    np.testing.assert_allclose(o["trans"], T, atol=1e-4)
    R, t = rot(0.01, -0.015, 0.03), np.array([0.15, -0.1, 0.05])
    assert np.linalg.norm(o["trans"][:3, 3] - t) < 0.03


def test_rand_draws():
    c = cases()
    o = oracle_gicp(c["motion"])
    assert o["rc"] == 0 and not o["trace"]["random_step"].any() and o["draws"] == 3
    o2 = oracle_gicp(c["motion"])
    assert np.array_equal(o["trans"], o2["trans"]) and np.array_equal(o["x0"], o2["x0"])
    o3 = oracle_gicp(c["motion"], seed=99)
    assert not np.array_equal(o["x0"], o3["x0"])
    nv = oracle_gicp(c["no_voxel"])
    assert nv["rc"] == 0 and nv["iterations"] == 64 and not nv["converged"]
    assert (nv["trace"]["n_corr"] == 0).all() and nv["trace"]["random_step"].all()
    assert nv["draws"] == 3 + 6 * 64


def test_edge_cases():
    c = cases()
    base = c["motion"]
    for name, mk in REFUSED.items():
        assert oracle_gicp(mk(base))["rc"] == -103, name
    tw = oracle_gicp(c["twenty"])
    assert tw["rc"] == 0 and tw["n_target"] == 20 and tw["n_source"] == 20
    # non-finite rows take part in nothing: the result equals the run without them
    nf = oracle_gicp(c["non_finite"])
    f = c["non_finite"]
    clean = dict(tgt=f["tgt"][np.isfinite(f["tgt"]).all(1)], src=f["src"][np.isfinite(f["src"]).all(1)])
    cl = oracle_gicp(clean)
    assert nf["rc"] == 0 and nf["n_source"] == len(clean["src"]) and nf["n_target"] == len(clean["tgt"])
    assert np.array_equal(nf["trans"], cl["trans"]) and nf["fitness"] == cl["fitness"]
    # a non-identity guess: the same walk as on the source moved by the guess (double, float store), then T * guess
    g = c["guess"]
    G, s = g["guess"], np.asarray(g["src"], np.float64)
    ms = np.stack([((G[r, 0] * s[:, 0] + G[r, 1] * s[:, 1]) + G[r, 2] * s[:, 2]) + G[r, 3] for r in range(3)], 1).astype(F32)
    og, om = oracle_gicp(g), oracle_gicp(dict(tgt=g["tgt"], src=ms))
    assert og["iterations"] == om["iterations"]
    np.testing.assert_allclose(og["trans"], om["trans"] @ G, rtol=0, atol=1e-12)


def test_ignored_arguments_not_in_the_abi():
    """max_iter_num and dis_thre_unit are the reference's arguments with its defaults, and never reach the library"""
    from mulls_b200.registration import Context, CRegistration
    for f in (Context.omp_gicp, CRegistration.omp_gicp):
        p = inspect.signature(f).parameters
        assert p["max_iter_num"].default == 20 and p["dis_thre_unit"].default == 1.5
        assert p["using_voxel_gicp"].default is True and p["voxel_size"].default == 1.0
        assert p["apply_intersection_filter"].default is False and p["fitness_score_thre"].default == 10.0
    hdr = open(os.path.join(ROOT, "include", "mulls_b200", "abi.h")).read()
    decl = hdr[hdr.index("int mulls_omp_gicp("):]
    decl = decl[:decl.index(";")]
    assert "max_iter" not in decl and "dis_thre" not in decl


def test_structs_mirror_abi_h(tmp_path):
    from mulls_b200 import abi
    src = tmp_path / "s.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "mulls_b200/abi.h"\nint main(void) {\n'
                   'printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(mulls_gicp_result), offsetof(mulls_gicp_result, fitness), '
                   'offsetof(mulls_gicp_result, x0), sizeof(mulls_gicp_iter), offsetof(mulls_gicp_iter, n_corr), '
                   'offsetof(mulls_gicp_iter, random_step));\nreturn 0;\n}\n')
    exe = tmp_path / "s"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = list(map(int, subprocess.check_output([str(exe)]).split()))
    assert got == [C.sizeof(abi.GicpResult), abi.GicpResult.fitness.offset, abi.GicpResult.x0.offset,
                   C.sizeof(abi.GicpIter), abi.GicpIter.n_corr.offset, abi.GicpIter.random_step.offset]


def build_gicp_caller(td):
    libdir = os.path.join(ROOT, "mulls_b200", "csrc")
    exe = os.path.join(td, "gicp_caller")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-I", os.path.join(ROOT, "include", "dropin"),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "stubs", "gicp_ref"),
                           "-I", os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests", "stubs", "gicp_caller.cpp"),
                           "-o", exe, "-L", libdir, "-lmulls_b200", f"-Wl,-rpath,{libdir}"])
    return exe


def test_dropin_gicp_compiles_and_links():
    """tests/stubs/gicp_caller.cpp replays mulls_slam.cpp:637-639 and :674-676 against the drop-in and a stand-in
    reference that declares omp_gicp: voxel calls reach the library (without a GPU: -3, Trans1_2 untouched),
    using_voxel_gicp = false and refused calls reach the reference member"""
    import tempfile

    import torch

    with tempfile.TemporaryDirectory() as td:
        exe = build_gicp_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "gicp drop-in compiled and linked" in out.stdout and "failures 0" in out.stdout
    if not torch.cuda.is_available():
        assert "ran on a device: 0" in out.stdout
