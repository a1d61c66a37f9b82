"""CPU checks of the NDT registration (CRegistration::omp_ndt, cregistration.hpp:945-1021, DIRECT7):
- the CPU restatement (tests/harness/ndt_oracle.cpp, the host instantiation of mulls_b200/csrc/ndt_core.cuh), the checker
  of mulls_omp_ndt, against an independent numpy restatement: leaf membership and valid-leaf sets exactly, means to
  1e-12 relative, inverse covariances to float tolerance; score, gradient and Hessian at fixed poses to float tolerance;
- the portable exp: at most 1 ulp from the double exp rounded to float, at most 2 from numpy's float32 exp (itself up to 1 ulp off);
- the walk against a numpy walk (iteration count, step lengths, reversals, final pose), the 6x6 SVD solve against
  numpy, the 37-iteration limit; every step length 0 or in [0.05, 0.1], empty clouds,
  all-small leaves, non-finite points, an intersection filter that empties a cloud and a non-identity initial guess;
- the drop-in member replays the mulls_slam call sites against a stand-in reference (tests/stubs/ndt_caller.cpp)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
_LIBS = {}


def ndt_oracle_lib(out_dir=None):
    out_dir = out_dir or os.path.join(ROOT, "tests", "harness", "_build")
    if out_dir in _LIBS:
        return _LIBS[out_dir]
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available: the host instantiation of ndt_core.cuh cannot be built")
    src = os.path.join(ROOT, "tests", "harness", "ndt_oracle.cpp")
    deps = [src] + [os.path.join(ROOT, "mulls_b200", "csrc", f) for f in ("ndt_core.cuh", "ransac_core.cuh", "ground_core.cuh")]
    deps.append(os.path.join(ROOT, "include", "mulls_b200", "abi.h"))
    out = os.path.join(out_dir, "libndt_oracle.so")
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
    dp, fp, ip = C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_int)
    lb.orc_ndt.restype = C.c_int
    lb.orc_ndt.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_float, dp, C.c_int, C.c_float, dp, dp,
                           C.POINTER(abi.NdtResult), C.POINTER(abi.NdtIter), C.c_int]
    lb.orc_ndt_leaves.restype = C.c_long
    lb.orc_ndt_leaves.argtypes = [C.c_void_p, C.c_long, C.c_float, C.c_long, C.POINTER(C.c_int64), ip, dp, fp, ip]
    lb.orc_ndt_eval.restype = None
    lb.orc_ndt_eval.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_float, dp, dp]
    lb.orc_ndt_expf.restype = None
    lb.orc_ndt_expf.argtypes = [fp, fp, C.c_long]
    lb.orc_ndt_gauss.restype = None
    lb.orc_ndt_gauss.argtypes = [C.c_float, dp, dp]
    _LIBS[out_dir] = lb
    return lb


def rows(xyz):
    xyz = np.asarray(xyz, F32).reshape(-1, 3)
    r = np.zeros((len(xyz), 12), F32)
    r[:, :3] = xyz
    return r


def bbox(xyz):
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    f = np.isfinite(xyz).all(1)
    if not f.any():
        return np.array([1e300, 1e300, 1e300, -1e300, -1e300, -1e300])
    return np.concatenate([xyz[f].min(0), xyz[f].max(0)])


def oracle_ndt(case, trace_cap=64):
    from mulls_b200 import abi
    t, s = rows(case["tgt"]), rows(case["src"])
    g = np.ascontiguousarray(case.get("guess", np.eye(4)), np.float64).ravel().copy()
    tb = np.ascontiguousarray(case.get("tb", bbox(case["tgt"])), np.float64)
    sb = np.ascontiguousarray(case.get("sb", bbox(case["src"])), np.float64)
    res = abi.NdtResult()
    tr = (abi.NdtIter * trace_cap)()
    dp = C.POINTER(C.c_double)
    ndt_oracle_lib().orc_ndt(t.ctypes.data, len(t), s.ctypes.data, len(s), case.get("res", 1.0), g.ctypes.data_as(dp),
                             int(case.get("filter", True)), case.get("thre", 10.0), tb.ctypes.data_as(dp), sb.ctypes.data_as(dp),
                             C.byref(res), tr, trace_cap)
    k = min(res.iterations, trace_cap)
    return dict(code=res.code, trans=np.array(res.trans[:]).reshape(4, 4), iterations=res.iterations,
                converged=bool(res.converged), fitness=res.fitness, n_target=res.n_target, n_source=res.n_source,
                trace=dict(p=np.array([tr[i].p[:] for i in range(k)]).reshape(k, 6), step=np.array([tr[i].step for i in range(k)]),
                           score=np.array([tr[i].score for i in range(k)]), reversed=np.array([tr[i].reversed for i in range(k)])))


# ---------------------------------------------------------------------------------------------------------------------
# scenes (shared with tests/test_gpu_ndt.py)
# ---------------------------------------------------------------------------------------------------------------------
def rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    return np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) @ \
        np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])


def structured_scene(n, seed, noise=0.02, extent=20.0):
    """a noisy box room with pillars: ground, walls, columns"""
    rng = np.random.default_rng(seed)
    k = n // 4
    ground = np.c_[rng.uniform(-extent, extent, (k, 2)), rng.normal(0, noise, k)]
    wx = np.c_[rng.choice([-extent, extent], k) + rng.normal(0, noise, k), rng.uniform(-extent, extent, k), rng.uniform(0, 6, k)]
    wy = np.c_[rng.uniform(-extent, extent, k), rng.choice([-extent, extent], k) + rng.normal(0, noise, k), rng.uniform(0, 6, k)]
    m = n - 3 * k
    ang = rng.uniform(0, 2 * np.pi, m)
    cen = rng.uniform(-extent * 0.7, extent * 0.7, (8, 2))[rng.integers(0, 8, m)]
    pil = np.c_[cen[:, 0] + 0.4 * np.cos(ang), cen[:, 1] + 0.4 * np.sin(ang), rng.uniform(0, 6, m)]
    pil[:, :2] += rng.normal(0, noise, (m, 2))
    return np.vstack([ground, wx, wy, pil]).astype(F32)


def moved(xyz, R, t):
    return (np.asarray(xyz, np.float64) @ R.T + t).astype(F32)


def cases():
    out = {}
    tgt = structured_scene(6000, 1)
    R, t = rot(0.01, -0.015, 0.03), np.array([0.15, -0.1, 0.05])
    # source = target moved by the inverse, so the registration should find (R, t)
    src = moved(tgt[::2] + np.random.default_rng(2).normal(0, 0.02, (3000, 3)).astype(F32), R.T, -R.T @ t)
    out["motion"] = dict(tgt=tgt, src=src)
    out["motion_res03"] = dict(tgt=tgt, src=src, res=0.3)
    out["motion_res07"] = dict(tgt=tgt, src=src, res=0.7)
    G = np.eye(4)
    G[:3, :3], G[:3, 3] = rot(0.0, 0.0, 0.02), [0.1, 0.0, 0.0]
    out["guess"] = dict(tgt=tgt, src=src, guess=G)
    out["empty_source"] = dict(tgt=tgt, src=np.zeros((0, 3), F32))
    out["empty_target"] = dict(tgt=np.zeros((0, 3), F32), src=src)
    rng = np.random.default_rng(3)
    sparse = rng.uniform(-50, 50, (200, 3)).astype(F32)  # every leaf well under 6 points
    out["small_leaves"] = dict(tgt=sparse, src=sparse + F32(0.1))
    nf = src.copy()
    nf[::97, 0] = np.nan
    nf[5::101, 2] = np.inf
    nft = tgt.copy()
    nft[3::89, 1] = -np.inf
    out["non_finite"] = dict(tgt=nft, src=nf, filter=False)
    far = src + F32(1000.0)
    out["filter_empties"] = dict(tgt=tgt, src=far)
    # 3 m off in 4 m leaves: every step is clamped to 0.1, the walk stops on the iteration limit (nr > 35)
    out["limit"] = dict(tgt=tgt, src=moved(src, np.eye(3), np.array([3.0, 0.0, 0.0])), res=4.0, thre=1e9)
    # a large offset: far from the Newton point, the walk takes many clamped steps
    out["far"] = dict(tgt=tgt, src=moved(src, np.eye(3), np.array([5.0, 0.0, 0.0])), res=4.0, thre=1e9)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the independent restatement
# ---------------------------------------------------------------------------------------------------------------------
def np_leaves(xyz, res):
    xyz = np.asarray(xyz, F32)
    xyz = xyz[np.isfinite(xyz).all(1)]
    inv = F32(1.0) / F32(res)
    mn, mx = xyz.min(0), xyz.max(0)
    min_b = np.floor(mn * inv).astype(np.int64)
    max_b = np.floor(mx * inv).astype(np.int64)
    div = max_b - min_b + 1
    ijk = (np.floor(xyz * inv) - min_b.astype(F32)).astype(np.int64)
    key = ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1]
    out = {}
    x64 = xyz.astype(np.float64)
    for k in np.unique(key):
        p = x64[key == k]
        n = len(p)
        mean = p.sum(0) / n
        d = dict(n=n, mean=mean, ok=False)
        if n >= 6:
            # the reference's single-pass form: the biased covariance, scaled by (n - 1) / n once more
            cov = np.cov(p.T, bias=True) * ((n - 1.0) / n)
            w, V = np.linalg.eigh(cov)
            d["lam"] = w
            if w[0] >= 0 and w[1] >= 0 and w[2] > 0:
                if w[0] < 0.01 * w[2]:
                    w = np.maximum(w, 0.01 * w[2])
                    cov = V @ np.diag(w) @ V.T
                d["icov"] = np.linalg.inv(cov)
                d["ok"] = True
        out[int(k)] = d
    return out, min_b, max_b, div, inv


def np_gauss(res):
    """ndt_omp_impl.hpp:89-93, outlier ratio 0.55"""
    c1, c2 = 10 * (1 - 0.55), 0.55 / float(np.float32(res)) ** 3
    d3 = -np.log(c2)
    d1 = -np.log(c1 + c2) - d3
    d2 = -2 * np.log((-np.log(c1 * np.exp(-0.5) + c2) - d3) / d1)
    return d1, d2


def np_solve(H, b):
    """JacobiSVD::solve with Eigen 3.3's default rank threshold (6 eps of the largest singular value)"""
    U, S, Vt = np.linalg.svd(H)
    thr = max(S[0] * 6 * np.finfo(np.float64).eps, np.finfo(np.float64).tiny)
    r = int(np.sum((S >= thr) & (S > 0)))
    return Vt[:r].T @ ((U[:, :r].T @ b) / S[:r])


def np_walk(tgt, src, res):
    """computeTransformation with the dead line search (step clamp(norm, 0.05, 0.1)) on np_eval's derivatives"""
    p = np.zeros(6)
    s, g, H = np_eval(tgt, src, res, p)
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
            s, g, H = np_eval(tgt, src, res, p)
        steps.append(a)
        rev.append(r)
        stop = nr > 35 or (nr and a < 0.1)
        nr += 1
        if stop:
            return dict(iterations=nr, step=np.array(steps), reversed=np.array(rev), p=p)


def np_angles(p):
    def cs(a):
        return (1.0, 0.0) if abs(a) < 1e-4 else (np.cos(a), np.sin(a))
    cx, sx = cs(p[3])
    cy, sy = cs(p[4])
    cz, sz = cs(p[5])
    j = np.array([[-sx * sz + cx * sy * cz, -sx * cz - cx * sy * sz, -cx * cy], [cx * sz + sx * sy * cz, cx * cz - sx * sy * sz, -sx * cy],
                  [-sy * cz, sy * sz, cy], [sx * cy * cz, -sx * cy * sz, sx * sy], [-cx * cy * cz, cx * cy * sz, -cx * sy],
                  [-cy * sz, -cy * cz, 0], [cx * cz - sx * sy * sz, -cx * sz - sx * sy * cz, 0],
                  [sx * cz + cx * sy * sz, cx * sy * cz - sx * sz, 0]])
    h = np.array([[-cx * sz - sx * sy * cz, -cx * cz + sx * sy * sz, sx * cy], [-sx * sz + cx * sy * cz, -cx * sy * sz - sx * cz, -cx * cy],
                  [cx * cy * cz, -cx * cy * sz, cx * sy], [sx * cy * cz, -sx * cy * sz, sx * sy],
                  [-sx * cz - cx * sy * sz, sx * sz - cx * sy * cz, 0], [cx * cz - sx * sy * sz, -sx * sy * cz - cx * sz, 0],
                  [-cy * cz, cy * sz, sy], [-sx * sy * cz, sx * sy * sz, sx * cy], [cx * sy * cz, -cx * sy * sz, -cx * cy],
                  [sy * sz, sy * cz, 0], [-sx * cy * sz, -sx * cy * cz, 0], [cx * cy * sz, cx * cy * cz, 0],
                  [-cy * cz, cy * sz, 0], [-cx * sz - sx * sy * cz, -cx * cz + sx * sy * sz, 0],
                  [-sx * sz + cx * sy * cz, -cx * sy * sz - sx * cz, 0]])
    return j, h


def np_eval(tgt, src, res, p):
    leaves, min_b, max_b, div, _ = np_leaves(tgt, res)
    d1, d2 = np_gauss(res)
    R = rot(p[3], p[4], p[5])
    jt, ht = np_angles(p)
    score, grad, hess = 0.0, np.zeros(6), np.zeros((6, 6))
    for x in np.asarray(src, np.float64):
        y = R @ x + p[:3]
        c = np.floor(y.astype(F32) / F32(res)).astype(np.int64)
        xj, xh = jt @ x, ht @ x
        J = np.zeros((3, 6))
        J[:, :3] = np.eye(3)
        J[:, 3], J[:, 4], J[:, 5] = [0, xj[0], xj[1]], [xj[2], xj[3], xj[4]], [xj[5], xj[6], xj[7]]
        a, b, cc = np.array([0, xh[0], xh[1]]), np.array([0, xh[2], xh[3]]), np.array([0, xh[4], xh[5]])
        d, e, f = xh[6:9], xh[9:12], xh[12:15]
        H = {(3, 3): a, (4, 3): b, (5, 3): cc, (3, 4): b, (4, 4): d, (5, 4): e, (3, 5): cc, (4, 5): e, (5, 5): f}
        for disp in [(0, 0, 0), (1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]:
            q = c + disp
            if (q < min_b).any() or (q > max_b).any():
                continue
            k = int((q - min_b) @ np.array([1, div[0], div[0] * div[1]]))
            lf = leaves.get(k)
            if lf is None or not lf["ok"]:
                continue
            xt = y - lf["mean"]
            Ci = lf["icov"]
            ex = np.exp(-d2 * xt @ Ci @ xt / 2)
            if not (0 <= d2 * ex <= 1):
                continue
            score += -d1 * ex
            g6 = xt @ Ci @ J
            grad += d1 * d2 * ex * g6
            for i in range(6):
                for jj in range(6):
                    hij = H.get((i, jj), np.zeros(3))
                    hess[i, jj] += d1 * d2 * ex * (-d2 * g6[i] * g6[jj] + xt @ Ci @ hij + J[:, jj] @ Ci @ J[:, i])
    return score, grad, hess


# ---------------------------------------------------------------------------------------------------------------------
def test_exp_within_one_ulp():
    xs = np.concatenate([np.linspace(-104, 88, 400001, dtype=F32), -np.logspace(-8, 2, 20001).astype(F32),
                         np.array([0.0, -0.0, -110.0, -103.5, 88.7], F32)])
    out = np.empty_like(xs)
    ndt_oracle_lib().orc_ndt_expf(xs.ctypes.data_as(C.POINTER(C.c_float)), out.ctypes.data_as(C.POINTER(C.c_float)), len(xs))
    ref = np.exp(xs.astype(np.float64)).astype(F32)  # correctly rounded but for double-rounding ties
    ulp = np.abs(out.view(np.int32).astype(np.int64) - ref.view(np.int32).astype(np.int64))
    assert ulp.max() <= 1, xs[np.argmax(ulp)]
    # numpy's float32 exp is itself within 1 ulp of the correctly rounded value, not always on the same side
    ref32 = np.exp(xs)
    d32 = np.abs(out.view(np.int32).astype(np.int64) - ref32.view(np.int32).astype(np.int64))
    assert d32.max() <= 2


@pytest.mark.parametrize("res", [1.0, 0.3])
def test_leaves_equal_numpy(res):
    tgt = structured_scene(4000, 7, extent=20.0 * res)
    lb = ndt_oracle_lib()
    cap = len(tgt)
    keys, n, ok = np.zeros(cap, np.int64), np.zeros(cap, np.int32), np.zeros(cap, np.int32)
    mean, icov = np.zeros((cap, 3)), np.zeros((cap, 9), F32)
    tr = rows(tgt)
    m = lb.orc_ndt_leaves(tr.ctypes.data, len(tgt), res, cap, keys.ctypes.data_as(C.POINTER(C.c_int64)),
                          n.ctypes.data_as(C.POINTER(C.c_int)), mean.ctypes.data_as(C.POINTER(C.c_double)),
                          icov.ctypes.data_as(C.POINTER(C.c_float)), ok.ctypes.data_as(C.POINTER(C.c_int)))
    ref, *_ = np_leaves(tgt, res)
    assert sorted(ref) == keys[:m].tolist()
    checked = 0
    for i in range(m):
        r = ref[int(keys[i])]
        assert abs(n[i]) == r["n"] or (n[i] == -1 and not r["ok"])
        np.testing.assert_allclose(mean[i], r["mean"], rtol=1e-12, atol=1e-12)
        lam = r.get("lam")
        if lam is not None and abs(lam[0]) < 1e-9 * max(abs(lam[2]), 1e-30):
            continue  # an exactly planar leaf: rejected or kept by the sign of rounding noise
        assert bool(ok[i]) == r["ok"], (i, lam)
        if r["ok"]:
            np.testing.assert_allclose(icov[i].reshape(3, 3), r["icov"], rtol=2e-4, atol=2e-4 * np.abs(r["icov"]).max())
            checked += 1
    assert checked > (20 if res == 1.0 else 0)


@pytest.mark.parametrize("res,p", [(1.0, [0, 0, 0, 0, 0, 0]), (1.0, [0.1, -0.05, 0.02, 0.01, -0.02, 0.03]),
                                   (0.3, [0.02, 0.01, 0.0, 0.0, 0.005, -0.01])])
def test_derivatives_equal_numpy(res, p):
    tgt = structured_scene(3000, 11)
    src = structured_scene(600, 12)
    p = np.array(p, np.float64)
    out = np.zeros(43)
    tr, sr = rows(tgt), rows(src)
    ndt_oracle_lib().orc_ndt_eval(tr.ctypes.data, len(tgt), sr.ctypes.data, len(src), res,
                                  p.ctypes.data_as(C.POINTER(C.c_double)), out.ctypes.data_as(C.POINTER(C.c_double)))
    s, g, H = np_eval(tgt, src, res, p)
    assert abs(out[0] - s) <= 1e-4 * abs(s)
    np.testing.assert_allclose(out[1:7], g, rtol=0, atol=2e-4 * np.abs(g).max() + 1e-6)
    np.testing.assert_allclose(out[7:].reshape(6, 6), H, rtol=0, atol=2e-4 * np.abs(H).max())


@pytest.mark.parametrize("name", list(cases()))
def test_walk_outcomes(name):
    c = cases()[name]
    o = oracle_ndt(c)
    tr = o["trace"]
    assert o["iterations"] <= 37
    assert np.all((tr["step"] == 0) | ((tr["step"] >= 0.05) & (tr["step"] <= 0.1)))
    if name in ("empty_source", "empty_target", "small_leaves", "filter_empties"):
        assert o["iterations"] == 0 and o["converged"]
        np.testing.assert_array_equal(o["trans"], np.eye(4))
    if name in ("empty_source", "empty_target", "filter_empties"):
        assert o["code"] == -3 and o["fitness"] == np.finfo(np.float64).max
    if name == "filter_empties":
        assert o["n_target"] == 0 and o["n_source"] == 0
    if name == "far":
        assert o["iterations"] > 5 and o["converged"]
    if name == "limit":
        assert o["iterations"] == 37
    if name == "non_finite":
        assert o["n_source"] == len(c["src"]) and np.isfinite(o["fitness"])
    if name.startswith("motion") or name == "guess":
        assert o["code"] == 1 and o["converged"]


def test_reversed_direction_branch():
    """-g.d > 0 happens where the Hessian is not negative definite: the walk turns the direction around. The scene's
    first iterations do so, and the numpy walk, which tests the sign on its own derivatives, reverses at the same ones"""
    c = walk_scene()
    o = oracle_ndt(c)
    assert o["trace"]["reversed"].sum() > 0
    n = np_walk(c["tgt"], c["src"], c["res"])
    assert o["trace"]["reversed"].tolist() == n["reversed"].tolist()


def test_iteration_limit():
    """nr > 35 stops the walk after 37 iterations (nr_iterations_ counts the last one too), every step clamped to 0.1"""
    o = oracle_ndt(cases()["limit"])
    assert o["iterations"] == 37 and o["converged"]
    assert np.all(o["trace"]["step"] == 0.1)


def walk_scene():
    tgt = structured_scene(2000, 21, extent=8.0)
    R, t = rot(0.0, 0.0, 0.02), np.array([0.3, -0.2, 0.05])
    src = moved(tgt[::5] + np.random.default_rng(22).normal(0, 0.02, (400, 3)).astype(F32), R.T, -R.T @ t)
    return dict(tgt=tgt, src=src, res=1.0)


def test_walk_equals_numpy():
    """the restatement's walk against the numpy walk (double derivatives, numpy SVD, Eigen's rank rule): the same
    iteration count, the same step lengths to float tolerance, the same final pose to 1e-4"""
    c = walk_scene()
    o = oracle_ndt(c)
    n = np_walk(c["tgt"], c["src"], c["res"])
    assert o["iterations"] == n["iterations"] >= 3
    np.testing.assert_allclose(o["trace"]["step"], n["step"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(o["trace"]["p"][-1], n["p"], rtol=0, atol=1e-4)


def test_svd_solve_equals_numpy():
    """ndt_svd_solve (Eigen's two-sided Jacobi SVD, rc_svd<6>) against numpy's SVD with Eigen's rank rule, on random,
    symmetric indefinite and rank-deficient 6x6 systems"""
    lb = ndt_oracle_lib()
    rng = np.random.default_rng(5)
    dp = C.POINTER(C.c_double)
    lb.orc_ndt_solve.restype = None
    lb.orc_ndt_solve.argtypes = [dp, dp, dp]
    mats = []
    for k in range(200):
        A = rng.normal(size=(6, 6)) * 10.0 ** rng.uniform(-3, 3)
        if k % 4 == 1:
            A = A + A.T
        if k % 4 == 2:  # rank 3
            A = rng.normal(size=(6, 3)) @ rng.normal(size=(3, 6))
        if k % 4 == 3:  # a zero row and column
            A = A + A.T
            A[2, :] = 0
            A[:, 2] = 0
        mats.append(A)
    mats.append(np.zeros((6, 6)))
    for A in mats:
        H = np.ascontiguousarray(A, np.float64)
        b = rng.normal(size=6)
        x = np.zeros(6)
        lb.orc_ndt_solve(H.ctypes.data_as(dp), b.ctypes.data_as(dp), x.ctypes.data_as(dp))
        ref = np_solve(H, b)
        np.testing.assert_allclose(x, ref, rtol=1e-7, atol=1e-9 * max(np.abs(ref).max(), 1e-300))


def test_dropin_ndt_compiles_and_links():
    """tests/stubs/ndt_caller.cpp replays mulls_slam.cpp:634-636 and :671-673 against the drop-in and a stand-in
    reference that declares omp_ndt: DIRECT7 calls reach the library (without a GPU: -3, Trans1_2 untouched), KDTREE
    calls the reference member"""
    import tempfile

    import torch

    with tempfile.TemporaryDirectory() as td:
        exe = build_ndt_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "ndt drop-in compiled and linked" in out.stdout and "failures 0" in out.stdout
    if not torch.cuda.is_available():
        assert "ran on a device: 0" in out.stdout


def build_ndt_caller(td):
    libdir = os.path.join(ROOT, "mulls_b200", "csrc")
    exe = os.path.join(td, "ndt_caller")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-I", os.path.join(ROOT, "include", "dropin"),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "stubs", "ndt_ref"),
                           "-I", os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests", "stubs", "ndt_caller.cpp"),
                           "-o", exe, "-L", libdir, "-lmulls_b200", f"-Wl,-rpath,{libdir}"])
    return exe


def test_known_motion_recovered():
    """the source is the target scene moved by (R, t)^-1: Trans1_2 recovers (R, t) to within the last step's 0.05
    (mixed m / rad; the walk never steps shorter) plus the scene's noise"""
    c = cases()["motion"]
    o = oracle_ndt(c)
    R, t = rot(0.01, -0.015, 0.03), np.array([0.15, -0.1, 0.05])
    T = o["trans"]
    assert np.linalg.norm(T[:3, 3] - t) < 0.06
    ang = np.arccos(np.clip((np.trace(T[:3, :3].T @ R) - 1) / 2, -1, 1))
    assert ang < 0.06
