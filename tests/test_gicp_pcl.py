"""CPU checks of the point-wise GICP registration (CRegistration::omp_gicp with using_voxel_gicp=False,
cregistration.hpp:1024-1098, koide_reg::GeneralizedIterativeClosestPoint with PCL's BFGS):
- the CPU restatement (tests/harness/gicp_pcl_oracle.cpp, the host instantiation of mulls_b200/csrc/gicp_pcl_core.cuh),
  the checker of mulls_omp_gicp_pcl, against independent numpy / scipy code: the double covariances against numpy's SVD
  (on the neighbour lists of tests/test_gicp.py, the same search), the Mahalanobis matrices and the 3x3 inverse against
  np.linalg.inv, applyState against scipy's ZYX Euler rotation, the functor's three methods at fixed poses against
  float64 numpy and its gradients against central differences, the BFGS solver on a 6-D quadratic (exact minimum) and
  on a Rosenbrock function against scipy's BFGS;
- the whole walk against a float64 numpy walk (numpy functor, a numpy BFGS) on the known-motion scene;
- edge cases: fewer than 4 correspondences, max_iter_num 0 and 1, non-finite rows, fewer than 20 points;
- max_iter_num reaches the solver; the shim caller (tests/stubs/gicp_pcl_caller.cpp) compiles and links;
- the ctypes structs mirror abi.h."""
import ctypes as C
import inspect
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree
from scipy.spatial.transform import Rotation

from test_gicp import cases, np_neighbours, xyz32
from test_ndt import bbox, moved, rot, rows, structured_scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
_LIBS = {}
FDF = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double))


def gicp_pcl_oracle_lib(out_dir=None):
    out_dir = out_dir or os.path.join(ROOT, "tests", "harness", "_build")
    if out_dir in _LIBS:
        return _LIBS[out_dir]
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available: the host instantiation of gicp_pcl_core.cuh cannot be built")
    src = os.path.join(ROOT, "tests", "harness", "gicp_pcl_oracle.cpp")
    deps = [src, os.path.join(ROOT, "tests", "harness", "gicp_oracle.cpp")]
    deps += [os.path.join(ROOT, "mulls_b200", "csrc", f)
             for f in ("gicp_pcl_core.cuh", "gicp_core.cuh", "ndt_core.cuh", "ransac_core.cuh", "ground_core.cuh")]
    deps.append(os.path.join(ROOT, "include", "mulls_b200", "abi.h"))
    out = os.path.join(out_dir, "libgicp_pcl_oracle.so")
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
    dp, vp = C.POINTER(C.c_double), C.c_void_p
    lb.orc_gicp_pcl.restype = C.c_int
    lb.orc_gicp_pcl.argtypes = [vp, C.c_long, vp, C.c_long, C.c_int, dp, C.c_int, C.c_float, dp, dp,
                                C.POINTER(abi.GicpPclResult), C.POINTER(abi.GicpPclIter), C.c_int]
    lb.orc_gicp_pcl_covariances.argtypes = [vp, C.c_long, vp]
    lb.orc_gicp_pcl_maha.argtypes = [vp, vp, vp, vp]
    lb.orc_gicp_pcl_inv3.argtypes = [vp, vp]
    lb.orc_gicp_pcl_apply_state.argtypes = [vp, vp]
    lb.orc_gicp_pcl_functor.restype = C.c_int
    lb.orc_gicp_pcl_functor.argtypes = [vp, C.c_long, vp, C.c_long, vp, vp, vp, vp, vp, vp, vp, vp]
    lb.orc_gicp_pcl_bfgs.argtypes = [FDF, vp, C.c_int, C.c_double, vp]
    _LIBS[out_dir] = lb
    return lb


def _p(a):
    return a.ctypes.data


def oracle_gicp_pcl(case, max_iter=20, trace_cap=256):
    """the restatement on a case dict (tgt, src, optional guess, tb, sb, filter, thre): a dict like
    Context.omp_gicp_pcl's plus `rc`"""
    from mulls_b200 import abi
    from mulls_b200.registration import _gicp_pcl_trace
    lb = gicp_pcl_oracle_lib()
    t, s = rows(case["tgt"]), rows(case["src"])
    g = np.ascontiguousarray(case.get("guess", np.eye(4)), np.float64).ravel().copy()
    tb = np.ascontiguousarray(case.get("tb", bbox(case["tgt"])), np.float64)
    sb = np.ascontiguousarray(case.get("sb", bbox(case["src"])), np.float64)
    res = abi.GicpPclResult()
    tr = (abi.GicpPclIter * trace_cap)()
    dp = C.POINTER(C.c_double)
    rc = lb.orc_gicp_pcl(_p(t), len(t), _p(s), len(s), int(max_iter), g.ctypes.data_as(dp), int(case.get("filter", False)),
                         case.get("thre", 10.0), tb.ctypes.data_as(dp), sb.ctypes.data_as(dp), C.byref(res), tr, trace_cap)
    out = dict(rc=rc, code=res.code, trans=np.array(res.trans[:]).reshape(4, 4), iterations=res.iterations,
               converged=bool(res.converged), fitness=res.fitness, n_target=res.n_target, n_source=res.n_source)
    out["trace"] = _gicp_pcl_trace(tr, min(res.iterations, trace_cap))
    return out


REFUSED = {  # MULLS_E_UNSUPPORTED
    "nineteen_src": lambda c: dict(tgt=c["tgt"], src=c["src"][:19]),
    "nineteen_tgt": lambda c: dict(tgt=c["tgt"][:19], src=c["src"]),
    "empty_source": lambda c: dict(tgt=c["tgt"], src=np.zeros((0, 3), F32)),
    "empty_target": lambda c: dict(tgt=np.zeros((0, 3), F32), src=c["src"]),
    "filter_empties": lambda c: dict(tgt=c["tgt"], src=c["src"] + F32(1000.0), filter=True),
}


# ---------------------------------------------------------------------------------------------------------------------
# the independent restatement in float64
# ---------------------------------------------------------------------------------------------------------------------
def np_covariances(xyz, nb=None):
    """U diag(1, 1, 1e-3) U^T of each point's 20-neighbour covariance (numpy's SVD); nb: the neighbour lists (default:
    a k-d tree's)"""
    xyz = xyz32(xyz)
    if nb is None:
        nb = cKDTree(xyz.astype(np.float64)).query(xyz.astype(np.float64), 20)[1]
    P = xyz[nb]
    mean = P.astype(np.float64).mean(1)
    # the reference adds float products (pt.x * pt.x is float * float) into double sums
    prod = (P[:, :, :, None] * P[:, :, None, :]).astype(np.float64)
    cov = prod.sum(1) / 20.0 - mean[:, :, None] * mean[:, None, :]
    U, _, _ = np.linalg.svd(cov)
    return U @ np.diag([1.0, 1.0, 1e-3]) @ U.transpose(0, 2, 1)


def euler_R(a):
    """applyState's rotation: Z(a[2]) Y(a[1]) X(a[0])"""
    return Rotation.from_euler("ZYX", [a[2], a[1], a[0]]).as_matrix()


def euler_dR(a):
    """the three derivatives of euler_R by the X, Y and Z angles"""
    def axis(k, t):
        c, s = np.cos(t), np.sin(t)
        R, D = np.eye(3), np.zeros((3, 3))
        i, j = [(1, 2), (0, 2), (0, 1)][k]
        R[i, i], R[j, j], D[i, i], D[j, j] = c, c, -s, -s
        sg = -1 if k != 1 else 1
        R[i, j], R[j, i], D[i, j], D[j, i] = sg * s, -sg * s, sg * c, -sg * c
        return R, D
    (Rx, Dx), (Ry, Dy), (Rz, Dz) = axis(0, a[0]), axis(1, a[1]), axis(2, a[2])
    return Rz @ Ry @ Dx, Rz @ Dy @ Rx, Dz @ Ry @ Rx


class NpFunctor:
    """f = mean(res^T M res) over the correspondences (src_i, tgt_j, M_i) with res = R(x) p + t - q, and its gradient.
    f32: each point's res^T M res in float32 as operator() computes it (the reference's f carries float noise, and its
    line search stops on that noise: a walk that is to end where the reference's ends needs the same f)"""

    def __init__(self, p, q, M, f32=False):
        self.p, self.q, self.M, self.f32 = p, q, M, f32

    def f(self, x):
        if not self.f32:
            return self.fdf(x)[0]
        R = euler_R(x[3:]).astype(F32)
        res = (self.p.astype(F32) @ R.T + x[:3].astype(F32)) - self.q.astype(F32)
        Mr = np.einsum("nij,nj->ni", self.M.astype(F32), res)
        return (res * Mr).sum(1, dtype=F32).astype(np.float64).sum() / len(res)

    def fdf(self, x):
        R = euler_R(x[3:])
        res = self.p @ R.T + x[:3] - self.q
        Mr = np.einsum("nij,nj->ni", self.M, res)
        m = len(res)
        f = np.einsum("ni,ni->", res, Mr) / m
        g = np.zeros(6)
        g[:3] = 2.0 / m * Mr.sum(0)
        for k, D in enumerate(euler_dR(x[3:])):
            g[3 + k] = 2.0 / m * np.einsum("ni,ni->", Mr, self.p @ D.T)
        return f, g


class NpBfgs:
    """GSL's vector_bfgs2 with Fletcher's line search, as gicp_pcl_core.cuh reads PCL's bfgs.h (B1-B5), in numpy"""

    def __init__(self, fdf, f=None):
        self.fdf, self.rho, self.sigma, self.tau1, self.tau2, self.tau3 = fdf, 0.01, 0.01, 9.0, 0.05, 0.5
        self.fonly = f or (lambda x: fdf(x)[0])

    def init(self, x):
        self.f, self.g = self.fdf(x)
        self.x0, self.g0 = x.copy(), self.g.copy()
        self.g0n = np.linalg.norm(self.g0)
        self.p = -self.g / self.g0n
        self.pn, self.fp0, self.delta_f = np.linalg.norm(self.p), -self.g0n, 0.0

    def _f(self, a):  # operator() at x0 + a p
        return self.fonly(self.x0 + a * self.p)

    def _df(self, a):  # the slope of df at x0 + a p
        return self.fdf(self.x0 + a * self.p)[1] @ self.p

    @staticmethod
    def _interp(a, fa, fpa, b, fb, fpb, xmin, xmax):
        ymin, ymax = sorted(((xmin - a) / (b - a), (xmax - a) / (b - a)))
        fpa = fpa * (b - a)
        q = lambda z: fa + z * (fpa + z * (fb - fa - fpa))  # noqa: E731
        y, fmin = (ymin, q(ymin)) if q(ymin) <= q(ymax) else (ymax, q(ymax))
        c = 2 * (fb - fa - fpa)
        if c > a:
            z = -fpa / c
            if ymin < z < ymax and q(z) < fmin:
                y = z
        return a + y * (b - a)

    def _search(self, alpha):
        f0, fp0 = self.f, self.fp0
        ap, fprev, fpprev = 0.0, f0, fp0
        a = b = fa = fb = fpa = fpb = None
        i = 0
        while i < 100:
            i += 1
            fal = self._f(alpha)
            if fal > f0 + alpha * self.rho * fp0 or fal >= fprev:
                a, fa, fpa, b, fb, fpb = ap, fprev, fpprev, alpha, fal, np.nan
                break
            fpal = self._df(alpha)
            if abs(fpal) <= -self.sigma * fp0:
                return alpha
            if fpal >= 0:
                a, fa, fpa, b, fb, fpb = alpha, fal, fpal, ap, fprev, fpprev
                break
            d = alpha - ap
            nxt = self._interp(ap, fprev, fpprev, alpha, fal, fpal, alpha + d, alpha + self.tau1 * d)
            ap, fprev, fpprev, alpha = alpha, fal, fpal, nxt
        while i < 100:
            i += 1
            d = b - a
            alpha = self._interp(a, fa, fpa, b, fb, fpb, a + self.tau2 * d, b - self.tau3 * d)
            fal = self._f(alpha)
            if (a - alpha) * fpa <= np.finfo(float).eps:
                return None
            if fal > f0 + self.rho * alpha * fp0 or fal >= fa:
                b, fb, fpb = alpha, fal, np.nan
            else:
                fpal = self._df(alpha)
                if abs(fpal) <= -self.sigma * fp0:
                    return alpha
                if ((b - a) >= 0 and fpal >= 0) or ((b - a) <= 0 and fpal <= 0):
                    b, fb, fpb = a, fa, fpa
                a, fa, fpa = alpha, fal, fpal
        return 0.0

    def step(self):
        """one minimizeOneStep: 0 success, 1 no progress"""
        if self.pn == 0 or self.g0n == 0 or self.fp0 == 0:
            return 1
        f0 = self.f
        a1 = min(1.0, 2.0 * max(-self.delta_f, 10 * np.finfo(float).eps * abs(f0)) / -self.fp0) if self.delta_f < 0 else 1.0
        alpha = self._search(a1)
        if alpha is None:
            return 1
        x = self.x0 + alpha * self.p
        self.f, self.g = self._f(alpha), self.fdf(x)[1]  # the line search's cached f and df at alpha
        self.delta_f = self.f - f0
        dx, dg = x - self.x0, self.g - self.g0
        dxdg = dx @ dg
        A = B = 0.0
        if dxdg != 0:
            B = dx @ self.g / dxdg
            A = -(1.0 + dg @ dg / dxdg) * B + dg @ self.g / dxdg
        p = self.g - A * dx - B * dg
        self.x0, self.g0, self.g0n = x, self.g.copy(), np.linalg.norm(self.g)
        p *= (-1.0 if p @ self.g >= 0 else 1.0) / self.pn
        self.p, self.pn = p, np.linalg.norm(p)
        self.fp0 = p @ self.g0
        return 0

    def solve(self, x, max_inner, tol=1e-2):
        """estimateRigidTransformationBFGS's do-while: (x, status, steps)"""
        self.init(np.asarray(x, np.float64))
        inner = 0
        while True:
            inner += 1
            r = self.step()
            if r:
                break
            r = 0 if np.linalg.norm(self.g) < tol else -1
            if not (r == -1 and inner < max_inner):
                break
        return self.x0.copy(), r, inner


def np_walk(tgt, src, max_iter=20):
    """computeTransformation in float64: (iterations, converged, final 4x4)"""
    tgt, src = xyz32(tgt).astype(np.float64), xyz32(src).astype(np.float64)
    ct, cs, tree = np_covariances(tgt), np_covariances(src), cKDTree(tgt)
    T, nr = np.eye(4), 0
    while True:
        R = T[:3, :3]
        d, j = tree.query(src @ R.T + T[:3, 3])
        keep = d * d < 25.0
        if keep.sum() < 4:
            return nr, False, T
        M = np.linalg.inv(R @ cs[keep] @ R.T + ct[j[keep]])
        fn = NpFunctor(src[keep], tgt[j[keep]], M, f32=True)
        x0 = np.array([T[0, 3], T[1, 3], T[2, 3], np.arctan2(T[2, 1], T[2, 2]), np.arcsin(-T[2, 0]), np.arctan2(T[1, 0], T[0, 0])])
        x, r, inner = NpBfgs(fn.fdf, fn.f).solve(x0, max_iter)
        if not (r in (0, 1) or inner == max_iter):
            return nr, False, T
        Tn = np.eye(4)
        Tn[:3, :3], Tn[:3, 3] = euler_R(x[3:]), x[:3]
        ratio = np.full((4, 4), 1 / 5e-4)
        ratio[:3, :3] = 1 / 2e-3
        delta = (ratio * np.abs(T - Tn)).max()
        T, nr = Tn, nr + 1
        if nr >= 200 or delta < 1:
            return nr, True, T


# ---------------------------------------------------------------------------------------------------------------------
def test_covariances_against_numpy_svd():
    lb = gicp_pcl_oracle_lib()
    for xyz in (structured_scene(800, 7), structured_scene(600, 4, extent=5.0)):
        xyz = xyz32(xyz)
        out = np.zeros((len(xyz), 9))
        lb.orc_gicp_pcl_covariances(_p(xyz), len(xyz), _p(out))
        ref = np_covariances(xyz, np_neighbours(xyz))
        np.testing.assert_allclose(out.reshape(-1, 3, 3), ref, atol=1e-6)
        assert np.isclose(np.linalg.det(out.reshape(-1, 3, 3)), 1e-3, rtol=1e-6).all()


def test_mahalanobis_and_inverse_against_numpy():
    lb = gicp_pcl_oracle_lib()
    rng = np.random.default_rng(3)
    for _ in range(50):
        A = rng.normal(size=(3, 3))
        inv = np.zeros(9)
        lb.orc_gicp_pcl_inv3(_p(np.ascontiguousarray(A.ravel())), _p(inv))
        np.testing.assert_allclose(inv.reshape(3, 3), np.linalg.inv(A), rtol=1e-9, atol=1e-9 * np.abs(np.linalg.inv(A)).max())
        U1, U2 = (np.linalg.qr(rng.normal(size=(3, 3)))[0] for _ in range(2))
        C1, C2 = U1 @ np.diag([1, 1, 1e-3]) @ U1.T, U2 @ np.diag([1, 1, 1e-3]) @ U2.T
        R = Rotation.from_rotvec(rng.normal(0, 0.3, 3)).as_matrix()
        M = np.zeros(9, F32)
        lb.orc_gicp_pcl_maha(_p(np.ascontiguousarray(R.ravel())), _p(np.ascontiguousarray(C1.ravel())),
                             _p(np.ascontiguousarray(C2.ravel())), _p(M))
        ref = np.linalg.inv(R @ C1 @ R.T + C2)
        np.testing.assert_allclose(M.reshape(3, 3), ref, rtol=1e-5, atol=1e-6 * np.abs(ref).max())


@pytest.mark.parametrize("x", [np.zeros(6), np.array([0.5, -1.0, 2.0, 0.01, -0.02, 0.03]),
                               np.array([0.0, 0.0, 0.0, 1.2, -0.7, 2.5]), np.array([3.0, 1.0, -2.0, -3.0, 1.5, -0.4])])
def test_apply_state_against_scipy(x):
    lb = gicp_pcl_oracle_lib()
    x = np.ascontiguousarray(x, np.float64)
    T = np.zeros(12, F32)
    lb.orc_gicp_pcl_apply_state(_p(x), _p(T))
    T = T.reshape(3, 4)
    np.testing.assert_allclose(T[:, :3], euler_R(x[3:].astype(F32).astype(np.float64)), atol=1e-6)
    assert np.array_equal(T[:, 3], x[:3].astype(F32))


def functor_scene():
    tgt = xyz32(structured_scene(3000, 11))
    src = xyz32(moved(tgt[::3], rot(0.004, -0.003, 0.01), np.array([0.08, -0.05, 0.02])))
    return tgt, src


def oracle_functor(lb, tgt, src, x):
    T0 = np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], F32)
    x = np.ascontiguousarray(x, np.float64)
    f, ffdf = np.zeros(1), np.zeros(1)
    gdf, gfdf = np.zeros(6), np.zeros(6)
    si, ti = np.zeros(len(src), np.int32), np.zeros(len(src), np.int32)
    m = lb.orc_gicp_pcl_functor(_p(tgt), len(tgt), _p(src), len(src), _p(T0), _p(x), _p(f), _p(gdf), _p(ffdf), _p(gfdf),
                                _p(si), _p(ti))
    return f[0], gdf, ffdf[0], gfdf, si[:m], ti[:m]


@pytest.mark.parametrize("x", [np.zeros(6), np.array([-0.08, 0.05, -0.02, -0.004, 0.003, -0.01]),
                               np.array([0.03, 0.02, -0.01, 0.01, -0.005, 0.02])])
def test_functor_at_fixed_poses(x):
    """operator(), df and fdf of the restatement against float64 numpy on the same correspondences (the identity
    transformation_), and the gradients against central differences of numpy's f"""
    lb = gicp_pcl_oracle_lib()
    tgt, src = functor_scene()
    f, gdf, ffdf, gfdf, si, ti = oracle_functor(lb, tgt, src, x)
    assert len(si) > 500 and np.all(np.diff(si) > 0)
    d, j = cKDTree(tgt.astype(np.float64)).query(src.astype(np.float64))
    keep = d * d < 25.0
    np.testing.assert_array_equal(si, np.flatnonzero(keep))
    np.testing.assert_array_equal(ti, j[keep])
    ct, cs = np_covariances(tgt, np_neighbours(tgt)), np_covariances(src, np_neighbours(src))
    M = np.linalg.inv(cs[si] + ct[ti])
    fn = NpFunctor(src[si].astype(np.float64), tgt[ti].astype(np.float64), M)
    fr, gr = fn.fdf(x)
    for a in (f, ffdf):
        np.testing.assert_allclose(a, fr, rtol=1e-4)
    for g in (gdf, gfdf):
        np.testing.assert_allclose(g, gr, rtol=1e-3, atol=1e-4 * np.abs(gr).max())
    h, num = 1e-6, np.zeros(6)
    for k in range(6):
        e = np.zeros(6)
        e[k] = h
        num[k] = (fn.fdf(x + e)[0] - fn.fdf(x - e)[0]) / (2 * h)
    np.testing.assert_allclose(gdf, num, rtol=1e-3, atol=1e-4 * np.abs(num).max())


def run_bfgs(fdf, x0, max_inner, tol):
    lb = gicp_pcl_oracle_lib()
    calls = []

    def cb(x, f, g):
        xv = np.array(x[:6])
        fv, gv = fdf(xv)
        calls.append(xv)
        f[0] = fv
        for i in range(6):
            g[i] = gv[i]

    cfn = FDF(cb)
    x = np.ascontiguousarray(x0, np.float64).copy()
    info = np.zeros(3, np.int32)
    lb.orc_gicp_pcl_bfgs(cfn, _p(x), max_inner, tol, _p(info))
    assert info[2] == len(calls)
    return x, info


def test_bfgs_quadratic_exact_minimum():
    from scipy.optimize import minimize
    rng = np.random.default_rng(4)
    J = rng.normal(size=(12, 6))
    A, b = J.T @ J + 0.5 * np.eye(6), rng.normal(size=6)
    fdf = lambda x: (0.5 * x @ A @ x - b @ x, A @ x - b)  # noqa: E731
    x, info = run_bfgs(fdf, np.zeros(6), 200, 1e-10)
    assert info[0] in (0, 1) and info[1] < 200
    np.testing.assert_allclose(x, np.linalg.solve(A, b), atol=1e-8)
    sp = minimize(lambda v: fdf(v)[0], np.zeros(6), jac=lambda v: fdf(v)[1], method="BFGS", options=dict(gtol=1e-10))
    np.testing.assert_allclose(x, sp.x, atol=1e-6)


def test_bfgs_rosenbrock_against_scipy():
    from scipy.optimize import minimize, rosen, rosen_der
    x0 = np.array([-1.2, 1.0, -0.5, 0.8, 0.3, -0.9])
    x, info = run_bfgs(lambda v: (rosen(v), rosen_der(v)), x0, 5000, 1e-8)
    assert info[0] in (0, 1)
    sp = minimize(rosen, x0, jac=rosen_der, method="BFGS", options=dict(gtol=1e-8))
    np.testing.assert_allclose(x, sp.x, atol=1e-4)
    np.testing.assert_allclose(x, np.ones(6), atol=1e-4)


def test_bfgs_matches_numpy_restatement_on_gicp():
    """the solver with the GICP functor: the restatement's steps follow numpy's BFGS (same readings, float64)"""
    tgt, src = functor_scene()
    d, j = cKDTree(tgt.astype(np.float64)).query(src.astype(np.float64))
    keep = d * d < 25.0
    ct, cs = np_covariances(tgt), np_covariances(src)
    fn = NpFunctor(src[keep].astype(np.float64), tgt[j[keep]].astype(np.float64), np.linalg.inv(cs[keep] + ct[j[keep]]))
    x, info = run_bfgs(fn.fdf, np.zeros(6), 20, 1e-2)
    xn, r, inner = NpBfgs(fn.fdf).solve(np.zeros(6), 20)
    assert (info[0], info[1]) == (r, inner)
    np.testing.assert_allclose(x, xn, atol=1e-12)


def test_walk_against_numpy():
    c = cases()["motion"]
    tgt, src = xyz32(c["tgt"])[::2], xyz32(c["src"])[::2]
    o = oracle_gicp_pcl(dict(tgt=tgt, src=src))
    assert o["rc"] == 0 and o["converged"] and o["iterations"] >= 2
    assert (o["trace"]["evaluations"] > o["trace"]["inner_iterations"]).all()  # the solver moves: line searches ran
    it, conv, T = np_walk(tgt, src)
    assert conv and it == o["iterations"]
    np.testing.assert_allclose(o["trans"], T, atol=1e-4)
    R, t = rot(0.01, -0.015, 0.03), np.array([0.15, -0.1, 0.05])
    assert np.linalg.norm(o["trans"][:3, 3] - t) < 0.03


def test_max_iter_reaches_the_solver():
    """the BFGS step cap binds at 1 and 5 on the known-motion scene: three different results"""
    c = cases()["motion"]
    r = {k: oracle_gicp_pcl(c, max_iter=k) for k in (1, 5, 20)}
    assert (r[1]["trace"]["inner_iterations"] == 1).all() and (r[5]["trace"]["inner_iterations"] <= 5).all()
    assert (r[5]["trace"]["inner_iterations"] == 5).any()
    assert r[20]["trace"]["inner_iterations"].max() > 5
    for a, b in ((1, 5), (5, 20), (1, 20)):
        assert not np.array_equal(r[a]["trans"], r[b]["trans"]), (a, b)


def test_edge_cases():
    c = cases()
    base = c["motion"]
    for name, mk in REFUSED.items():
        assert oracle_gicp_pcl(mk(base))["rc"] == -103, name
    tw = oracle_gicp_pcl(c["twenty"])
    assert tw["rc"] == 0 and tw["n_target"] == 20 and tw["n_source"] == 20
    # fewer than 4 correspondences: the first estimate throws, nothing is counted, the result is the identity
    far = oracle_gicp_pcl(c["no_voxel"])
    assert far["rc"] == 0 and far["iterations"] == 0 and not far["converged"] and np.array_equal(far["trans"], np.eye(4))
    # max_iter_num 0: one step is taken; a walk still running throws and ends the loop unconverged
    z = oracle_gicp_pcl(base, max_iter=0)
    assert z["rc"] == 0 and not z["converged"] and (z["trace"]["status"] != -1).all()
    one = oracle_gicp_pcl(base, max_iter=1)
    assert one["rc"] == 0 and one["iterations"] >= 1 and (one["trace"]["inner_iterations"] == 1).all()
    # non-finite rows take part in nothing
    f = c["non_finite"]
    nf = oracle_gicp_pcl(f)
    cl = oracle_gicp_pcl(dict(tgt=f["tgt"][np.isfinite(f["tgt"]).all(1)], src=f["src"][np.isfinite(f["src"]).all(1)]))
    assert nf["rc"] == 0 and np.array_equal(nf["trans"], cl["trans"]) and nf["fitness"] == cl["fitness"]
    # a non-identity guess: the walk on the moved source, then T * guess
    g = c["guess"]
    G, s = g["guess"], np.asarray(g["src"], np.float64)
    ms = np.stack([((G[r, 0] * s[:, 0] + G[r, 1] * s[:, 1]) + G[r, 2] * s[:, 2]) + G[r, 3] for r in range(3)], 1).astype(F32)
    og, om = oracle_gicp_pcl(g), oracle_gicp_pcl(dict(tgt=g["tgt"], src=ms))
    assert og["iterations"] == om["iterations"]
    np.testing.assert_allclose(og["trans"], om["trans"] @ G, rtol=0, atol=1e-12)


def test_arguments_and_defaults():
    from mulls_b200.registration import Context, CRegistration
    for f in (Context.omp_gicp_pcl, CRegistration.omp_gicp_pcl):
        p = inspect.signature(f).parameters
        assert p["max_iter_num"].default == 20 and p["dis_thre_unit"].default == 1.5
        assert p["apply_intersection_filter"].default is False and p["fitness_score_thre"].default == 10.0
        assert "using_voxel_gicp" not in p and "voxel_size" not in p
    hdr = open(os.path.join(ROOT, "include", "mulls_b200", "abi.h")).read()
    decl = hdr[hdr.index("int mulls_omp_gicp_pcl("):]
    decl = decl[:decl.index(";")]
    assert "max_iter_num" in decl and "dis_thre" not in decl and "voxel" not in decl


def test_structs_mirror_abi_h(tmp_path):
    from mulls_b200 import abi
    src = tmp_path / "s.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "mulls_b200/abi.h"\nint main(void) {\n'
                   'printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(mulls_gicp_pcl_result), '
                   'offsetof(mulls_gicp_pcl_result, fitness), sizeof(mulls_gicp_pcl_iter), offsetof(mulls_gicp_pcl_iter, delta), '
                   'offsetof(mulls_gicp_pcl_iter, n_corr), offsetof(mulls_gicp_pcl_iter, inner_iterations), '
                   'offsetof(mulls_gicp_pcl_iter, status), offsetof(mulls_gicp_pcl_iter, evaluations));\nreturn 0;\n}\n')
    exe = tmp_path / "s"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = list(map(int, subprocess.check_output([str(exe)]).split()))
    I = abi.GicpPclIter
    assert got == [C.sizeof(abi.GicpPclResult), abi.GicpPclResult.fitness.offset, C.sizeof(I), I.delta.offset,
                   I.n_corr.offset, I.inner_iterations.offset, I.status.offset, I.evaluations.offset]


def build_gicp_pcl_caller(td):
    libdir = os.path.join(ROOT, "mulls_b200", "csrc")
    exe = os.path.join(td, "gicp_pcl_caller")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests", "stubs", "gicp_pcl_caller.cpp"),
                           "-o", exe, "-L", libdir, "-lmulls_b200", f"-Wl,-rpath,{libdir}"])
    return exe


def test_shim_compiles_and_links():
    """tests/stubs/gicp_pcl_caller.cpp replays mulls_slam.cpp:637-639 and :674-676 with --voxel_gicp_on=false through
    lo::b200::omp_gicp_pcl (without a GPU: -3, Trans1_2 untouched)"""
    import tempfile

    import torch

    with tempfile.TemporaryDirectory() as td:
        exe = build_gicp_pcl_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "gicp_pcl shim compiled and linked" in out.stdout and "failures 0" in out.stdout
    if not torch.cuda.is_available():
        assert "ran on a device: 0" in out.stdout
