"""CPU checks of the NCC keypoint matching (CRegistration::find_feature_correspondence_ncc, cregistration.hpp:409-601):
- the CPU restatement (tests/harness/ncc_oracle.cpp), the checker of mulls_ncc_correspondences, against an independent
  numpy restatement (float32 sums in component order), bit for bit in every mode on adversarial keypoint clouds and on
  real vertex clouds of the oracle's front end;
- the drop-in CRegistration replays test/mulls_reg.cpp:173-174 and test/mulls_slam.cpp:534-535 against the stand-in
  headers (tests/stubs/ncc_caller.cpp)."""
import ctypes as C
import functools
import importlib.util
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLT_MAX = np.float32(np.finfo(np.float32).max)
INT_MIN = -(2 ** 31)
INT_MAX = 2 ** 31 - 1

# (name, fixed_num_corr, corr_num, reciprocal_on)
MODES = [("plain", False, 2000, False), ("reciprocal", False, 2000, True), ("fixed", True, 1000, True)]


# ---------------------------------------------------------------------------------------------------------------------
# the independent restatement
# ---------------------------------------------------------------------------------------------------------------------
def x86_int(f):
    """(int) of float32 values as x86-64 converts them: truncation in [-2^31, 2^31), INT_MIN otherwise and for NaN"""
    f = np.asarray(f, np.float32)
    ok = (f >= np.float32(-2147483648.0)) & (f < np.float32(2147483648.0))
    out = np.full(f.shape, INT_MIN, np.int64)
    out[ok] = np.trunc(f[ok]).astype(np.int64)
    return out


def cdiv(a, b):
    q = np.abs(a) // b
    return np.where(a < 0, -q, q)


def cmod(a, b):
    return a - b * cdiv(a, b)


def intensity_range(target):
    """max_ / min_ (utility.hpp:31-32) folded in order from FLT_MAX and 0"""
    mn, mx = FLT_MAX, np.float32(0.0)
    for v in np.asarray(target, np.float32)[:, 8]:
        mn = mn if mn < v else v
        mx = mx if mx > v else v
    return np.float32(mn), np.float32(mx)


def np_descriptors(rows, mn, mx):
    rows = np.asarray(rows, np.float32)
    D = np.empty((len(rows), 11), np.float32)
    for base, col in ((0, 4), (4, 5)):
        c = x86_int(rows[:, col])
        D[:, base + 0] = cdiv(c, 1000000)
        D[:, base + 1] = cdiv(cmod(c, 1000000), 10000)
        D[:, base + 2] = cdiv(cmod(c, 10000), 100)
        D[:, base + 3] = cmod(c, 100)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        q = (rows[:, 8] - mn) / (mx - mn)  # float32
        D[:, 8] = (q.astype(np.float64) * 255.0).astype(np.float32)
        D[:, 9] = rows[:, 7] * np.float32(100)
        D[:, 10] = rows[:, 3] * np.float32(30)
    return D


def np_distances(target, source):
    mn, mx = intensity_range(target)
    T, S = np_descriptors(target, mn, mx), np_descriptors(source, mn, mx)
    d = np.zeros((len(T), len(S)), np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for k in range(11):
            d = d + np.abs(T[:, None, k] - S[None, :, k])
    return d


def np_keys(d):
    k = np.ascontiguousarray(d, np.float32).view(np.uint32).copy()
    k[np.isnan(d)] = 0xFFFFFFFF
    return k


def cap_walk(order, n_s, n_t):
    ct, cs = np.zeros(n_t, np.int64), np.zeros(n_s, np.int64)
    ti, si = [], []
    for idx in order.tolist():
        i, j = divmod(idx, n_s)
        if ct[i] > 6 or cs[j] > 6:
            continue
        ct[i] += 1
        cs[j] += 1
        ti.append(i)
        si.append(j)
    return np.array(ti, np.int32), np.array(si, np.int32)


def np_ncc(target, source, fixed_num_corr, corr_num, reciprocal_on):
    """None (fewer than 10 keypoints), "E_ARG" (fixed mode over INT_MAX pairs) or (tgt_idx, src_idx)"""
    nt, ns = len(target), len(source)
    if nt < 10 or ns < 10:
        return None
    if fixed_num_corr and nt * ns > INT_MAX:
        return "E_ARG"
    d = np_distances(target, source)
    if not fixed_num_corr:
        with np.errstate(invalid="ignore"):
            cand = np.where(d < FLT_MAX, d, np.inf)
        has = np.isfinite(cand).any(1)
        j = np.where(has, np.argmin(cand, axis=1), 0)
        best = np.where(has, d[np.arange(nt), j], FLT_MAX).astype(np.float32)
        keep = np.ones(nt, bool)
        if reciprocal_on:
            with np.errstate(invalid="ignore"):
                colmin = np.fmin.reduce(d, axis=0)
            colmin = np.where(np.isnan(colmin), np.float32(np.inf), colmin)
            keep = ~(best > colmin[j])
        return np.flatnonzero(keep).astype(np.int32), j[keep].astype(np.int32)
    M = nt * ns
    K = M if corr_num < 0 else min(corr_num, M)
    order = np.argsort(np_keys(d).ravel(), kind="stable")[:K]
    return cap_walk(order, ns, nt)


# ---------------------------------------------------------------------------------------------------------------------
# the CPU restatement (tests/harness/ncc_oracle.cpp)
# ---------------------------------------------------------------------------------------------------------------------
_LIBS = {}


def ncc_oracle_lib(out_dir=None):
    out_dir = out_dir or os.path.join(ROOT, "tests", "harness", "_build")
    if out_dir in _LIBS:
        return _LIBS[out_dir]
    src = os.path.join(ROOT, "tests", "harness", "ncc_oracle.cpp")
    out = os.path.join(out_dir, "libncc_oracle.so")
    if not os.path.exists(out) or os.path.getmtime(src) > os.path.getmtime(out):
        os.makedirs(out_dir, exist_ok=True)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        subprocess.check_call([cxx, "-O3", "-fPIC", "-fopenmp", "-ffp-contract=off", "-std=c++17", "-w", "-shared", "-o", out, src])
    lb = C.CDLL(out)
    ip = C.POINTER(C.c_int32)
    lb.orc_ncc.restype = C.c_int
    lb.orc_ncc.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_int, ip, ip, C.c_size_t,
                           C.POINTER(C.c_size_t)]
    _LIBS[out_dir] = lb
    return lb


def result_cap(nt, ns, fixed_num_corr):
    """the most pairs a call can return: one per target row, or at most 7 per keypoint"""
    return 7 * min(nt, ns) if fixed_num_corr else nt


def oracle_ncc(target, source, fixed_num_corr, corr_num, reciprocal_on, threads=0, lib_dir=None):
    """None (the reference's false), -101 (refused) or (tgt_idx, src_idx). threads 0: min(6, cores) as the reference"""
    t = np.ascontiguousarray(target, np.float32)
    s = np.ascontiguousarray(source, np.float32)
    cap = result_cap(len(t), len(s), fixed_num_corr)
    ti, si = np.zeros(max(cap, 1), np.int32), np.zeros(max(cap, 1), np.int32)
    n = C.c_size_t(0)
    ip = C.POINTER(C.c_int32)
    rc = ncc_oracle_lib(lib_dir).orc_ncc(t.ctypes.data, len(t), s.ctypes.data, len(s), int(bool(fixed_num_corr)), int(corr_num),
                                         int(bool(reciprocal_on)), int(threads), ti.ctypes.data_as(ip), si.ctypes.data_as(ip), cap,
                                         C.byref(n))
    if rc == 0:
        return None
    if rc < 0:
        return rc
    return ti[: n.value].copy(), si[: n.value].copy()


def assert_same_pairs(got, exp):
    if exp is None or got is None:
        assert got is None and exp is None, (got, exp)
        return
    assert len(got[0]) == len(exp[0]), (len(got[0]), len(exp[0]))
    assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])


# ---------------------------------------------------------------------------------------------------------------------
# the keypoint clouds (shared with tests/test_gpu_ncc.py)
# ---------------------------------------------------------------------------------------------------------------------
def kpts(n, rng, close=None, far=None, intensity=None, curv=None, height=None):
    """48-byte rows as encode_stable_points leaves vertex keypoints: normal[0] / normal[1] the encoded close / far
    neighbourhood categories, normal[3] the curvature, data[3] the height above ground"""
    r = np.zeros((n, 12), np.float32)
    r[:, :3] = rng.uniform(-50, 50, (n, 3))
    pct = lambda: (rng.integers(0, 101, (n, 4)) * np.array([1000000, 10000, 100, 1])).sum(1)  # noqa: E731
    r[:, 4] = pct() if close is None else close
    r[:, 5] = pct() if far is None else far
    r[:, 7] = rng.uniform(0, 1, n) if curv is None else curv
    r[:, 3] = rng.uniform(0, 3, n) if height is None else height
    r[:, 8] = rng.uniform(0, 255, n) if intensity is None else intensity
    r[:, 9] = rng.uniform(0, 1, n)  # untouched payload
    return r


def _chain_mod():
    spec = importlib.util.spec_from_file_location("make_golden_chain", os.path.join(ROOT, "tests", "golden", "make_golden_chain.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@functools.lru_cache(maxsize=None)
def real_vertex_clouds():
    """pc_vertex of scans 0 and 1 of tests/golden/demo_chain.npz through the oracle's front end"""
    mod = _chain_mod()
    z = np.load(os.path.join(ROOT, "tests", "golden", "demo_chain.npz"))
    gp, cp = mod.chain_params()
    out = []
    for k in (0, 1):
        raw = mod.decode_scan(z[f"scan{k}_dmm"], z[f"scan{k}_i"])
        out.append(np.ascontiguousarray(mod.oracle_features(raw, gp, cp)["vertex"], np.float32))
    return out[0], out[1]


def cpu_clouds():
    """(name, target rows, source rows)"""
    rng = np.random.default_rng(11)
    out = [("random", kpts(300, rng), kpts(250, rng))]
    # every target row but the first (whose intensity spans the range) has the sources' descriptor: all distances tie
    t = kpts(60, rng, close=12345678, far=2030405, intensity=1.0, curv=0.25, height=1.0)
    t[0, 8] = 0.0
    s = kpts(50, rng, close=12345678, far=2030405, intensity=1.0, curv=0.25, height=1.0)
    out.append(("all_equal", t, s))
    out.append(("integer_only", kpts(200, rng, intensity=rng.integers(0, 2, 200), curv=rng.integers(0, 3, 200),
                                     height=rng.integers(0, 2, 200)),
                kpts(180, rng, intensity=rng.integers(0, 2, 180), curv=rng.integers(0, 3, 180), height=rng.integers(0, 2, 180))))
    out.append(("constant_intensity", kpts(80, rng, intensity=7.0), kpts(70, rng)))
    out.append(("constant_zero_intensity", kpts(40, rng, intensity=0.0), kpts(45, rng, intensity=0.0)))
    for where, at in (("start", [0]), ("middle", [37]), ("end", [99]), ("several", [3, 50, 60])):
        t = kpts(100, rng)
        t[at, 8] = np.nan
        out.append((f"nan_intensity_{where}", t, kpts(90, rng)))
    out.append(("negative_intensity", kpts(120, rng, intensity=rng.uniform(-5, -1, 120)), kpts(110, rng)))
    t = kpts(150, rng, intensity=rng.uniform(-2, 2, 150))
    t[[10, 20, 30], 8] = [0.0, -0.0, 0.0]
    out.append(("signed_zero_intensity", t, kpts(90, rng, intensity=rng.uniform(-2, 2, 90))))
    t, s = kpts(200, rng), kpts(180, rng)
    odd = np.array([np.nan, np.inf, -np.inf, 3.0e9, -3.0e9, 2.0 ** 31, -(2.0 ** 31), 16777217.0, 123456789.0, 99999999.0,
                    -123456.0, 2147483520.0], np.float32)
    for c in (4, 5):
        t[: len(odd), c] = odd
        s[-len(odd):, c] = odd[::-1]
    out.append(("odd_normals", t, s))
    out.append(("nine_targets", kpts(9, rng), kpts(20, rng)))
    out.append(("nine_sources", kpts(20, rng), kpts(9, rng)))
    out.append(("ten_ten", kpts(10, rng), kpts(10, rng)))
    t, s = kpts(60, rng), kpts(55, rng)
    t[[2, 5], 7] = np.nan  # rows of NaN distances
    t[[7, 9], 7] = np.inf  # rows of +inf distances
    s[[0, 4], 3] = np.nan  # NaN columns
    out.append(("no_finite_distance", t, s))
    out.append(("shape_10x20000", kpts(10, rng), kpts(20000, rng)))
    out.append(("shape_20000x10", kpts(20000, rng), kpts(10, rng)))
    return out


CLOUDS = cpu_clouds()


@pytest.mark.parametrize("mode,fixed,corr,recip", MODES, ids=[m[0] for m in MODES])
@pytest.mark.parametrize("name,target,source", CLOUDS, ids=[c[0] for c in CLOUDS])
def test_oracle_equals_numpy_restatement(name, target, source, mode, fixed, corr, recip):
    exp = np_ncc(target, source, fixed, corr, recip)
    assert_same_pairs(oracle_ncc(target, source, fixed, corr, recip), exp)
    if exp is not None and len(target) * len(source) <= 200000:
        assert_same_pairs(oracle_ncc(target, source, fixed, corr, recip, threads=1), exp)


@pytest.mark.parametrize("mode,fixed,corr,recip", MODES, ids=[m[0] for m in MODES])
def test_real_vertex_clouds(mode, fixed, corr, recip):
    t, s = real_vertex_clouds()
    assert len(t) >= 100 and len(s) >= 100
    assert np.any(t[:, 4] > 2 ** 24)  # encoded categories above 2^24: rounded ints
    exp = np_ncc(t, s, fixed, corr, recip)
    assert len(exp[0]) > 0
    assert_same_pairs(oracle_ncc(t, s, fixed, corr, recip), exp)


@pytest.mark.parametrize("corr_num", [-1, 0, 1, "M", "M+1", 4000])
@pytest.mark.parametrize("name", ["random", "all_equal", "no_finite_distance"])
def test_fixed_corr_num_edges(name, corr_num):
    t, s = dict((c[0], (c[1], c[2])) for c in CLOUDS)[name]
    M = len(t) * len(s)
    k = {"M": M, "M+1": M + 1}.get(corr_num, corr_num)
    exp = np_ncc(t, s, True, k, False)
    assert_same_pairs(oracle_ncc(t, s, True, k, False), exp)
    if k == 0:
        assert len(exp[0]) == 0


def test_cap_binds_on_ties():
    t, s = dict((c[0], (c[1], c[2])) for c in CLOUDS)["all_equal"]
    ti, si = oracle_ncc(t, s, True, -1, False)
    assert np.bincount(ti).max() == 7 and np.bincount(si).max() == 7
    # rows 1.. take the sources seven at a time until every source holds 7; row 0 (distance 255 to all) comes last
    assert len(ti) == 7 * len(s) and not np.any(ti == 0)
    assert list(zip(ti[:8].tolist(), si[:8].tolist())) == [(1, j) for j in range(7)] + [(2, 0)]


def test_over_int_max_pairs_is_refused():
    t = kpts(46341, np.random.default_rng(3))  # 46341^2 > INT_MAX >= 46340^2
    assert oracle_ncc(t, t, True, 10, False) == -101
    assert np_ncc(t, t, True, 10, False) == "E_ARG"
    assert oracle_ncc(t[:10], t, True, 10, False) is not None


# ---------------------------------------------------------------------------------------------------------------------
# the drop-in CRegistration: test/mulls_reg.cpp:173-174, test/mulls_slam.cpp:534-535, against the stand-in headers
# ---------------------------------------------------------------------------------------------------------------------
def build_ncc_caller(td):
    libdir = os.path.join(ROOT, "mulls_b200", "csrc")
    exe = os.path.join(td, "ncc_caller")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-I", os.path.join(ROOT, "include", "dropin"),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "stubs", "ref"),
                           "-I", os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests", "stubs", "ncc_caller.cpp"),
                           "-o", exe, "-L", libdir, "-lmulls_b200", f"-Wl,-rpath,{libdir}"])
    return exe


def test_dropin_ncc_compiles_and_links():
    """Without a GPU every call reports the missing device, returns false and leaves the output clouds empty."""
    import torch

    with tempfile.TemporaryDirectory() as td:
        exe = build_ncc_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "ncc drop-in compiled and linked" in out.stdout and "failures 0" in out.stdout
    if not torch.cuda.is_available():
        assert "ran on a device: 0" in out.stdout
