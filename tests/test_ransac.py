"""CPU checks of the RANSAC coarse registration (CRegistration::coarse_reg_ransac, cregistration.hpp:604-661):
- the CPU restatement (tests/harness/ransac_oracle.cpp), the checker of mulls_coarse_reg_ransac, against an independent
  numpy restatement: numpy's legacy-seeded MT19937 for the sample stream, np.linalg.svd for the Umeyama fits, float32
  numpy arithmetic for the transform-and-compare. Sample triples, hypothesis counts, the best hypothesis, the sizes of the
  refinement rounds, the final inlier count and the status agree exactly, the transform to 1e-6 per entry;
- known answers: keypoints under a known rigid motion at 2 %, 10 %, 50 % and 100 % inliers;
- the drop-in CRegistration replays the call sites of test/mulls_reg.cpp and test/mulls_slam.cpp against the stand-in
  headers (tests/stubs/ransac_caller.cpp), and the unchanged tests/stubs/dropin_caller.cpp still compiles."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
INT_MAX = 2 ** 31 - 1


# ---------------------------------------------------------------------------------------------------------------------
# the independent restatement
# ---------------------------------------------------------------------------------------------------------------------
class MtStream:
    """boost::mt19937(12345u): numpy's MT19937 with the legacy (init_genrand) seeding"""

    def __init__(self):
        self.bg = np.random.MT19937()
        self.bg._legacy_seeding(12345)
        self.buf, self.pos = [], 0

    def __call__(self):
        if self.pos == len(self.buf):
            self.buf, self.pos = self.bg.random_raw(4096).tolist(), 0
        self.pos += 1
        return self.buf[self.pos - 1]


def np_roots(m):
    """pcl::computeRoots on a float32 3x3, float32 scalar arithmetic"""
    m = [[F32(v) for v in row] for row in m]
    with np.errstate(all="ignore"):
        c0 = m[0][0] * m[1][1] * m[2][2] + F32(2) * m[0][1] * m[0][2] * m[1][2] - m[0][0] * m[1][2] * m[1][2] - \
            m[1][1] * m[0][2] * m[0][2] - m[2][2] * m[0][1] * m[0][1]
        c1 = m[0][0] * m[1][1] - m[0][1] * m[0][1] + m[0][0] * m[2][2] - m[0][2] * m[0][2] + m[1][1] * m[2][2] - m[1][2] * m[1][2]
        c2 = m[0][0] + m[1][1] + m[2][2]

        def roots2(b, c):
            d = F32(F32(b * b) - 4.0 * float(c))
            d = F32(0) if d < 0 else d
            sd = np.sqrt(d)
            return [F32(0), F32(0.5) * (b - sd), F32(0.5) * (b + sd)]

        if abs(c0) < np.finfo(F32).eps:
            return roots2(c2, c1)
        inv3 = F32(1.0 / 3.0)
        c2_3 = c2 * inv3
        a_3 = (c1 - c2 * c2_3) * inv3
        a_3 = F32(0) if a_3 > 0 else a_3
        half_b = F32(0.5) * (c0 + c2_3 * (F32(2) * c2_3 * c2_3 - c1))
        q = half_b * half_b + a_3 * a_3 * a_3
        q = F32(0) if q > 0 else q
        rho = np.sqrt(-a_3)
        theta = F32(np.arctan2(float(np.sqrt(-q)), float(half_b))) * inv3
        ct, st = F32(np.cos(float(theta))), F32(np.sin(float(theta)))
        s3 = np.sqrt(F32(3))
        r = [c2_3 + F32(2) * rho * ct, c2_3 - rho * (ct + s3 * st), c2_3 - rho * (ct - s3 * st)]
        if r[0] >= r[1]:
            r[0], r[1] = r[1], r[0]
        if r[1] >= r[2]:
            r[1], r[2] = r[2], r[1]
            if r[0] >= r[1]:
                r[0], r[1] = r[1], r[0]
        if r[0] <= 0:
            return roots2(c2, c1)
        return r


def np_sample_threshold(src):
    """computeMeanAndCovarianceMatrix (float32, sequential sums), eigen33's eigenvalues, ((sum sqrt) / 3)^2 in double"""
    x, y, z = (np.ascontiguousarray(src[:, c], F32) for c in range(3))
    with np.errstate(all="ignore"):
        terms = [x * x, x * y, x * z, y * y, y * z, z * z, x, y, z]
        accu = [np.add.accumulate(t)[-1] if len(t) else F32(0) for t in terms]
        accu = [F32(a) / F32(len(x)) for a in accu]
        cov = np.array([[accu[0] - accu[6] * accu[6], accu[1] - accu[6] * accu[7], accu[2] - accu[6] * accu[8]],
                        [0, accu[3] - accu[7] * accu[7], accu[4] - accu[7] * accu[8]],
                        [0, 0, accu[5] - accu[8] * accu[8]]], F32)
        cov[1, 0], cov[2, 0], cov[2, 1] = cov[0, 1], cov[0, 2], cov[1, 2]
        a = np.abs(cov)
        scale = F32(np.nanmax(a)) if not np.all(np.isnan(a)) else F32(0)
        scale = F32(1) if scale <= np.finfo(F32).tiny else scale
        ev = [r * scale for r in np_roots(cov / scale)]
        t = float(np.sqrt(ev[0]) + np.sqrt(ev[1]) + np.sqrt(ev[2])) / 3.0
    return t * t


def np_umeyama(src, tgt):
    """pcl::umeyama(src, tgt, false) in float64 with numpy's SVD, cast to float32 (3x4)"""
    with np.errstate(all="ignore"):
        s, t = np.asarray(src, np.float64), np.asarray(tgt, np.float64)
        ms, mt = s.mean(0), t.mean(0)
        sigma = (t - mt).T @ (s - ms) / len(s)
        if not np.all(np.isfinite(sigma)):
            return np.full((3, 4), np.nan, F32)
        U, _, Vt = np.linalg.svd(sigma)
        S = np.ones(3)
        if np.linalg.det(U) * np.linalg.det(Vt) < 0:
            S[2] = -1
        R = U @ np.diag(S) @ Vt
        T = np.empty((3, 4))
        T[:, :3], T[:, 3] = R, mt - R @ ms
    return T.astype(F32)


def np_sq_errors(T, s, t):
    """float32 T [s, 1] - t, squared norm (dx^2 + dz^2) + dy^2; T (..., 3, 4)"""
    with np.errstate(all="ignore"):
        p = [((T[..., i, 0:1] * s[:, 0] + T[..., i, 1:2] * s[:, 1]) + T[..., i, 2:3] * s[:, 2]) + T[..., i, 3:4] for i in range(3)]
        d = [p[i] - t[:, i] for i in range(3)]
        return (d[0] * d[0] + d[2] * d[2]) + d[1] * d[1]


def np_ransac(target, source, noise_bound=0.2, min_inlier_num=8, max_iter_num=20000):
    """dict: status, T (4x4 float64, None when not written), n_inliers, n_hyp, samples, counts, best, sizes,
    count_margin (per hypothesis: number of squared errors within 1e-4 relative of the threshold)"""
    N = len(target)
    t = np.ascontiguousarray(np.asarray(target, F32)[:, :3])
    s = np.ascontiguousarray(np.asarray(source, F32)[:N, :3])
    out = dict(samples=[], counts=[], margin=[], best=-1, sizes=[], n_hyp=0)
    best_T, remaining = np.eye(4), 0
    thr = float(noise_bound) * float(noise_bound)
    if N > 0:
        sthr = np_sample_threshold(s)
        rnd = MtStream()
        shuf = list(range(N))

        def good(a, b):
            with np.errstate(all="ignore"):
                d = s[a] - s[b]
                return float((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]) > sthr

        it, n_best, k, model = 0, -INT_MAX, 1.0, None
        max_skip = (max_iter_num * 10) % 2 ** 32
        while it < k and 0 < max_skip:
            sel = None
            if N >= 3:
                for _ in range(1000):
                    for i in range(3):
                        o = i + (rnd() >> 1) % (N - i)
                        shuf[i], shuf[o] = shuf[o], shuf[i]
                    if good(shuf[1], shuf[0]) and good(shuf[2], shuf[0]) and good(shuf[2], shuf[1]):
                        sel = shuf[:3]
                        break
            if sel is None:
                break
            T = np_umeyama(s[sel], t[sel])
            e = np_sq_errors(T, s, t).astype(np.float64)
            with np.errstate(invalid="ignore"):
                cnt = int(np.sum(e < thr))
                out["margin"].append(int(np.sum(np.abs(e - thr) <= 1e-4 * thr)))
            out["samples"].append(list(sel))
            out["counts"].append(cnt)
            if cnt > n_best:
                n_best, model, out["best"] = cnt, T, it
                w = n_best / N
                p = min(max(np.finfo(float).eps, 1.0 - w ** 3), 1.0 - np.finfo(float).eps)
                k = np.log(0.01) / np.log(p)
            it += 1
            if it > max_iter_num:
                break
        out["n_hyp"] = it
        if model is None:
            remaining = N
        else:
            def select(T, th):
                e = np_sq_errors(T, s, t).astype(np.float64)
                with np.errstate(invalid="ignore"):
                    m = e < th * th
                return np.flatnonzero(m), e[m]

            inliers_, _ = select(model, noise_bound)
            err_thr, it_r, changed, osc = float(noise_bound), 0, False, False
            prev, new, sizes = inliers_, np.zeros(0, np.int64), []
            new_T = model
            while True:
                new_T = np_umeyama(s[prev], t[prev]) if len(prev) else np.full((3, 4), np.nan, F32)
                sizes.append(len(prev))
                new, errs = select(new_T, err_thr)
                if len(new) == 0:
                    it_r += 1
                    if it_r >= 1000:
                        break
                else:
                    med = np.sort(errs)[len(errs) >> 1]
                    err_thr = np.sqrt(min(thr, 9.0 * (2.1981 * med)))
                    changed = False
                    prev, new = new, prev
                    if len(new) != len(prev):
                        if len(sizes) >= 4 and sizes[-1] == sizes[-3] and sizes[-2] == sizes[-4]:
                            osc = True
                            break
                        changed = True
                    elif not np.array_equal(prev, new):
                        changed = True
                if not changed:
                    break
                it_r += 1
                if it_r >= 1000:
                    break
            out["sizes"] = sizes
            if len(new) == 0:
                ok, fin, fin_T = False, None, None
            elif osc:
                ok, fin, fin_T = True, inliers_, model
            elif not changed:
                ok, fin, fin_T = True, prev, new_T
            else:
                ok, fin, fin_T = False, None, None
            if not ok:
                remaining = 0
            elif len(fin) < 3:
                remaining = N
            else:
                remaining = len(fin)
                best_T = np.eye(4)
                best_T[:3] = fin_T.astype(np.float64)
    lo = min_inlier_num % 2 ** 64
    hi = ((2 * min_inlier_num + 2 ** 31) % 2 ** 32 - 2 ** 31) % 2 ** 64
    out["n_inliers"] = remaining
    out["status"] = (1 if remaining >= hi else 0) if remaining >= lo else -1
    out["T"] = best_T if out["status"] >= 0 else None
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the CPU restatement (tests/harness/ransac_oracle.cpp)
# ---------------------------------------------------------------------------------------------------------------------
_LIBS = {}


def ransac_oracle_lib(out_dir=None):
    out_dir = out_dir or os.path.join(ROOT, "tests", "harness", "_build")
    if out_dir in _LIBS:
        return _LIBS[out_dir]
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available: the host instantiation of ransac_core.cuh cannot be built")
    src = os.path.join(ROOT, "tests", "harness", "ransac_oracle.cpp")
    deps = [src] + [os.path.join(ROOT, "mulls_b200", "csrc", f) for f in ("ransac_core.cuh", "ground_core.cuh")]
    out = os.path.join(out_dir, "libransac_oracle.so")
    if not os.path.exists(out) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(out):
        os.makedirs(out_dir, exist_ok=True)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        subprocess.check_call([nvcc, "-x", "cu", "-O2", "-std=c++17", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a",
                               "-ccbin", cxx, "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-w", "-o", out, src])
    lb = C.CDLL(out)
    ip = C.POINTER(C.c_int)
    lb.orc_ransac.restype = C.c_int
    lb.orc_ransac.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_float, C.c_int, C.c_int, C.POINTER(C.c_double),
                              ip, ip, ip, ip, C.c_long, ip, ip, C.c_int, ip, ip]
    lb.orc_mt_draws.restype = None
    lb.orc_mt_draws.argtypes = [C.POINTER(C.c_uint32), C.c_long]
    lb.orc_sample_threshold.restype = C.c_double
    lb.orc_sample_threshold.argtypes = [C.c_void_p, C.c_long]
    _LIBS[out_dir] = lb
    return lb


def oracle_ransac(target, source, noise_bound=0.2, min_inlier_num=8, max_iter_num=20000, tran=None, trace_cap=25000, lib_dir=None):
    """the restatement's result as np_ransac's dict; T is the given matrix (marker when None) when status is -1"""
    t = np.ascontiguousarray(target, F32)
    s = np.ascontiguousarray(source, F32)
    T = np.array(np.full((4, 4), 7.0) if tran is None else tran, np.float64).ravel().copy()
    samples = np.zeros((trace_cap, 3), np.int32)
    counts = np.zeros(trace_cap, np.int32)
    sizes = np.zeros(1000, np.int32)
    st, ni, nh, ns_, best = (C.c_int(0) for _ in range(5))
    ip = C.POINTER(C.c_int)
    ransac_oracle_lib(lib_dir).orc_ransac(t.ctypes.data, len(t), s.ctypes.data, len(s), float(noise_bound), int(min_inlier_num),
                                          int(max_iter_num), T.ctypes.data_as(C.POINTER(C.c_double)), C.byref(st), C.byref(ni),
                                          C.byref(nh), samples.ctypes.data_as(ip), trace_cap, counts.ctypes.data_as(ip),
                                          sizes.ctypes.data_as(ip), len(sizes), C.byref(ns_), C.byref(best))
    h = min(nh.value, trace_cap)
    return dict(status=st.value, T=T.reshape(4, 4), n_inliers=ni.value, n_hyp=nh.value, samples=samples[:h].tolist(),
                counts=counts[:h].tolist(), best=best.value, sizes=sizes[: min(ns_.value, 1000)].tolist())


def assert_same(o, n, check_T=True):
    assert o["n_hyp"] == n["n_hyp"], (o["n_hyp"], n["n_hyp"])
    assert o["samples"] == n["samples"]
    for k, (co, cn, m) in enumerate(zip(o["counts"], n["counts"], n["margin"])):
        assert abs(co - cn) <= m, (k, co, cn, m)  # equal unless a residual sits on the threshold
    assert o["best"] == n["best"]
    assert o["sizes"] == n["sizes"], (o["sizes"][:20], n["sizes"][:20])
    assert (o["status"], o["n_inliers"]) == (n["status"], n["n_inliers"])
    if n["status"] >= 0:
        assert not check_T or np.allclose(o["T"], n["T"], rtol=0, atol=1e-6), (o["T"], n["T"])
    else:
        assert np.all(o["T"] == 7.0)  # untouched


# ---------------------------------------------------------------------------------------------------------------------
# the correspondence sets (shared with tests/test_gpu_ransac.py)
# ---------------------------------------------------------------------------------------------------------------------
def rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    return np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) @ \
        np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])


def rows(xyz):
    r = np.zeros((len(xyz), 12), F32)
    r[:, :3] = xyz
    r[:, 8] = np.arange(len(xyz)) % 255  # payload the call ignores
    return r


def scene(n, ratio, seed, noise=0.01, extent=40.0):
    """(target, source, T_true): keypoint pairs where round(ratio * n) targets are R s + t moved by `noise` in a random
    direction (every inlier error about noise, far below the default noise bound 0.2), the rest uniform in the box"""
    rng = np.random.default_rng(seed)
    src = rng.uniform(-extent, extent, (n, 3))
    R, tr = rot(*rng.uniform(-0.5, 0.5, 3)), rng.uniform(-5, 5, 3)
    tgt = src @ R.T + tr
    d = rng.normal(size=(n, 3))
    tgt += noise * d / np.linalg.norm(d, axis=1, keepdims=True)
    k = int(round(ratio * n))
    out = rng.permutation(n)[: n - k]
    tgt[out] = rng.uniform(-extent, extent, (len(out), 3))
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, tr
    return rows(tgt), rows(src), T


def cases():
    """(name, target, source, kwargs) for both restatements and the device"""
    out = []
    for r in (0.02, 0.1, 0.5, 1.0):
        t, s, _ = scene(400, r, int(r * 100))
        out.append((f"known_{int(r * 100)}pct", t, s, {}))
    t, s, _ = scene(50, 1.0, 3)
    out += [("n0", t[:0], s[:0], {}), ("n0_min0", t[:0], s[:0], dict(min_inlier_num=0)), ("n2", t[:2], s[:2], dict(min_inlier_num=2)),
            ("n3", t[:3], s[:3], dict(min_inlier_num=3))]
    for k, name in ((8, "exactly_min"), (15, "two_min_minus_1"), (16, "two_min")):
        t, s, _ = scene(60, k / 60, 40 + k)
        out.append((name, t, s, {}))
    t, s, _ = scene(200, 0.0, 5)
    out.append(("all_outliers", t, s, dict(max_iter_num=3000)))
    t, s, _ = scene(300, 1.0, 6)
    out.append(("all_inliers", t, s, {}))
    # collinear sources: collinear triples pass isSampleGood
    rng = np.random.default_rng(7)
    src = np.outer(rng.uniform(-20, 20, 120), [0.6, 0.8, 0.0]) + [1.0, 2.0, 3.0]
    out.append(("collinear", rows(src @ rot(0.1, 0.2, 0.3).T + 1.0), rows(src), dict(max_iter_num=2000)))
    # duplicate sources: the threshold is 0, no sample is good, 1000 attempts exhaust the selection
    out.append(("duplicates", rows(rng.uniform(-5, 5, (30, 3))), rows(np.tile([[1.0, 2.0, 3.0]], (30, 1))), {}))
    for what, val in (("nan", np.nan), ("inf", np.inf), ("ninf", -np.inf)):
        t, s, _ = scene(120, 0.5, 8)
        s2 = s.copy()
        s2[17, 1] = val
        out.append((f"{what}_in_source", t, s2, {}))
        t2 = t.copy()
        t2[[3, 50, 99], 2] = val
        out.append((f"{what}_in_target", t2, s, {}))
    t, s, _ = scene(150, 0.3, 9)
    for mi in (0, 1, -1):
        out.append((f"max_iter_{mi}", t, s, dict(max_iter_num=mi)))
    for nb, name in ((0.0, "zero"), (-0.2, "negative"), (np.nan, "nan")):
        out.append((f"noise_bound_{name}", t, s, dict(noise_bound=nb, max_iter_num=500)))
    out.append(("min_inlier_0_refine_fails", t, s, dict(noise_bound=0.0, min_inlier_num=0, max_iter_num=50)))
    out.append(("min_inlier_0", t, s, dict(min_inlier_num=0)))
    out.append(("min_inlier_negative", t, s, dict(min_inlier_num=-3)))
    t, s, _ = scene(300, 0.6, 10, noise=0.15)
    out.append(("noisy_refinement", t, s, {}))
    t, s, _ = scene(120, 0.4, 11)
    out.append(("source_longer", t, np.concatenate([s, rows(np.full((5, 3), np.nan))]), {}))
    # refinements that stop on the oscillation test (sizes 14 13 14 13, and ... 34 33 34 33): refineModel returns true
    # but keeps computeModel's inliers and model (found by a seed search over noisy scenes)
    t, s, _ = scene(50, 0.970919387749674, 170, noise=0.264787681546382)
    out.append(("oscillating_a", t, s, dict(max_iter_num=200)))
    t, s, _ = scene(76, 0.8352342762699921, 2077, noise=0.18495069422172322)
    out.append(("oscillating_b", t, s, {}))
    return out


CASES = cases()


def test_mt_stream_and_threshold_are_the_shared_ones():
    lb = ransac_oracle_lib()
    out = np.zeros(40000, np.uint32)
    lb.orc_mt_draws(out.ctypes.data_as(C.POINTER(C.c_uint32)), len(out))
    bg = np.random.MT19937()
    bg._legacy_seeding(12345)
    assert np.array_equal(out.astype(np.uint64), bg.random_raw(40000))  # past the 16 384 the ground filter tabulates
    assert int(out[0]) == 3992670690
    for name, t, s, _ in CASES:
        if len(t) >= 1:
            sc = np.ascontiguousarray(s, F32)
            a, b = lb.orc_sample_threshold(sc.ctypes.data, len(t)), np_sample_threshold(sc[: len(t), :3])
            assert (np.isnan(a) and np.isnan(b)) or abs(a - b) <= 1e-6 * abs(b), (name, a, b)


@pytest.mark.parametrize("name,target,source,kw", CASES, ids=[c[0] for c in CASES])
def test_oracle_equals_numpy_restatement(name, target, source, kw):
    # collinear correspondences leave the rotation about their line to the SVD's own steps: everything but the matrix
    # must agree there
    assert_same(oracle_ransac(target, source, **kw), np_ransac(target, source, **kw), check_T=name != "collinear")


def test_case_outcomes_cover_the_branches():
    res = {name: oracle_ransac(t, s, **kw) for name, t, s, kw in CASES}
    assert res["n0"]["status"] == -1 and res["n0_min0"]["status"] == 1 and res["n0_min0"]["n_hyp"] == 0
    assert np.array_equal(res["n0_min0"]["T"], np.eye(4))
    assert res["n2"]["n_hyp"] == 0 and res["n2"]["n_inliers"] == 2 and res["n2"]["status"] == 0
    assert res["exactly_min"]["n_inliers"] == 8 and res["exactly_min"]["status"] == 0
    assert res["two_min_minus_1"]["n_inliers"] == 15 and res["two_min_minus_1"]["status"] == 0
    assert res["two_min"]["n_inliers"] == 16 and res["two_min"]["status"] == 1
    assert res["all_inliers"]["n_hyp"] == 1 and res["all_inliers"]["n_inliers"] == 300
    assert res["duplicates"]["n_hyp"] == 0 and res["duplicates"]["n_inliers"] == 30 and np.array_equal(res["duplicates"]["T"], np.eye(4))
    for what in ("nan", "inf", "ninf"):  # the threshold is NaN: no sample is good, all correspondences with the identity
        r = res[f"{what}_in_source"]
        assert r["n_hyp"] == 0 and r["n_inliers"] == 120 and np.array_equal(r["T"], np.eye(4))
        assert res[f"{what}_in_target"]["n_hyp"] > 0
    assert res["max_iter_0"]["n_hyp"] == 0 and res["max_iter_0"]["n_inliers"] == 150
    assert res["max_iter_1"]["n_hyp"] == 2 and res["max_iter_-1"]["n_hyp"] == 1
    assert res["noise_bound_zero"]["status"] == -1 and res["noise_bound_zero"]["n_inliers"] == 0
    assert res["noise_bound_negative"]["status"] == res["known_50pct"]["status"] or res["noise_bound_negative"]["n_inliers"] > 0
    assert res["min_inlier_0_refine_fails"]["status"] == 1 and np.array_equal(res["min_inlier_0_refine_fails"]["T"], np.eye(4))
    assert res["min_inlier_negative"]["status"] == -1
    for name in ("oscillating_a", "oscillating_b"):
        z = res[name]["sizes"]
        assert len(z) >= 4 and z[-1] == z[-3] and z[-2] == z[-4] and z[-1] != z[-2], (name, z)
        assert res[name]["n_inliers"] == z[0] != z[-1], (name, res[name]["n_inliers"], z)  # computeModel's inliers


# at 2 % inliers a sample is all inliers with probability 8e-6: 20 000 hypotheses find one in about 15 % of the scenes
# (PCL's result is then every correspondence with the identity), so that scene gets the iterations it needs
@pytest.mark.parametrize("ratio,n,max_iter,status", [(0.02, 500, 2000000, 0), (0.1, 1000, 20000, 1), (0.5, 1000, 20000, 1),
                                                     (1.0, 1000, 20000, 1)])
def test_known_motion_is_recovered(ratio, n, max_iter, status):
    t, s, T = scene(n, ratio, 77 + int(ratio * 100))
    o = oracle_ransac(t, s, max_iter_num=max_iter)
    assert o["status"] == status
    k = int(round(ratio * len(t)))
    assert o["n_inliers"] <= k and o["n_inliers"] >= 0.9 * k
    assert np.abs(o["T"][:3, :3] - T[:3, :3]).max() < 2e-3 and np.abs(o["T"][:3, 3] - T[:3, 3]).max() < 0.02


def test_20000_correspondences():
    t, s, _ = scene(20000, 0.1, 12)
    o = oracle_ransac(t, s)
    assert_same(o, np_ransac(t, s))
    assert o["status"] == 1


# ---------------------------------------------------------------------------------------------------------------------
# the drop-in CRegistration against the stand-in headers
# ---------------------------------------------------------------------------------------------------------------------
def build_caller(td, name="ransac_caller"):
    libdir = os.path.join(ROOT, "mulls_b200", "csrc")
    exe = os.path.join(td, name)
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-I", os.path.join(ROOT, "include", "dropin"),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "stubs", "ref"),
                           "-I", os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests", "stubs", name + ".cpp"),
                           "-o", exe, "-L", libdir, "-lmulls_b200", f"-Wl,-rpath,{libdir}"])
    return exe


def test_dropin_ransac_compiles_and_links():
    """Without a GPU every call reports the missing device, returns -1 and leaves tran_mat alone."""
    import torch

    with tempfile.TemporaryDirectory() as td:
        exe = build_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
        build_caller(td, "dropin_caller")  # the unchanged caller of the stand-in's coarse_reg_ransac(int)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "ransac drop-in compiled and linked" in out.stdout and "failures 0" in out.stdout
    if not torch.cuda.is_available():
        assert "ran on a device: 0" in out.stdout
