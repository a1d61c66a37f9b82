"""CPU checks of the TEASER++ coarse registration (CRegistration::coarse_reg_teaser, cregistration.hpp:664-759):
- the clique step of the CPU restatement (tests/harness/teaser_oracle.cpp, the checker of mulls_coarse_reg_teaser)
  against a pure-Python Bron-Kerbosch search with pivoting and the lexicographic rule (teaser_core.cuh T9), on random
  graphs and on graphs with several maximum cliques of one size; its core numbers against a pure-Python peeling;
- the whole restatement against an independent numpy restatement (numpy's SVD for the Jacobi SVD, Python's sort for the
  voting): status, clique, rotation inliers and the counts identical, the matrix to 1e-9;
- adversarial correspondence sets and known motions at 5 %, 20 %, 50 % and 100 % inliers;
- the drop-in CRegistration replays the call sites of test/mulls_reg.cpp and test/mulls_slam.cpp against the stand-in
  headers (tests/stubs/teaser_caller.cpp), and the unchanged tests/stubs/dropin_caller.cpp still compiles."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from mulls_b200 import abi
from test_ransac import build_caller, rot, rows, scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


# ---------------------------------------------------------------------------------------------------------------------
# the CPU restatement
# ---------------------------------------------------------------------------------------------------------------------
_LIBS = {}


def teaser_oracle_lib():
    if "lib" in _LIBS:
        return _LIBS["lib"]
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available: the host instantiation of teaser_core.cuh cannot be built")
    out_dir = os.path.join(ROOT, "tests", "harness", "_build")
    src = os.path.join(ROOT, "tests", "harness", "teaser_oracle.cpp")
    deps = [src, os.path.join(ROOT, "include", "mulls_b200", "abi.h")] + \
        [os.path.join(ROOT, "mulls_b200", "csrc", f) for f in ("teaser_core.cuh", "ransac_core.cuh", "ground_core.cuh")]
    out = os.path.join(out_dir, "libteaser_oracle.so")
    if not os.path.exists(out) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(out):
        os.makedirs(out_dir, exist_ok=True)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        subprocess.check_call([nvcc, "-x", "cu", "-O2", "-std=c++17", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a",
                               "-ccbin", cxx, "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-w", "-o", out, src])
    lb = C.CDLL(out)
    ip, up = C.POINTER(C.c_int), C.POINTER(C.c_uint64)
    lb.orc_tm_clique.restype = C.c_int
    lb.orc_tm_clique.argtypes = [C.c_int, up, ip]
    lb.orc_tm_core.restype = None
    lb.orc_tm_core.argtypes = [C.c_int, up, ip]
    lb.orc_tm_graph.restype = None
    lb.orc_tm_graph.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_float, up]
    lb.orc_teaser.restype = C.c_int
    lb.orc_teaser.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_float, C.c_int, C.POINTER(C.c_double), ip,
                              C.POINTER(abi.TeaserInfo), ip, C.POINTER(C.c_uint8)]
    _LIBS["lib"] = lb
    return lb


def info_dict(info):
    return {k: getattr(info, k) for k, _ in abi.TeaserInfo._fields_ if k not in ("pad", "search_launches")}


def oracle_teaser(target, source, noise_bound=0.2, min_inlier_num=8, tran=None):
    """dict: status, T (the given matrix, a marker when None, where status is -1), info, clique, mask"""
    t = np.ascontiguousarray(target, F32)
    s = np.ascontiguousarray(source, F32)
    T = np.array(np.full((4, 4), 7.0) if tran is None else tran, np.float64).ravel().copy()
    n = max(len(t), 1)
    clique = np.zeros(n, np.int32)
    mask = np.zeros(n, np.uint8)
    st, info = C.c_int(0), abi.TeaserInfo()
    teaser_oracle_lib().orc_teaser(t.ctypes.data, len(t), s.ctypes.data, len(s), float(noise_bound), int(min_inlier_num),
                                   T.ctypes.data_as(C.POINTER(C.c_double)), C.byref(st), C.byref(info),
                                   clique.ctypes.data_as(C.POINTER(C.c_int)), mask.ctypes.data_as(C.POINTER(C.c_uint8)))
    d = info_dict(info)
    m = d["clique_size"] if len(t) == len(s) and len(t) > 3 else 0
    return dict(status=st.value, T=T.reshape(4, 4), info=d, clique=clique[:m].tolist(),
                mask=mask[:m].tolist() if m > 1 else [])


def bits_of(adj_bool):
    """(n, n) bool -> (n, W) uint64 rows"""
    n = len(adj_bool)
    W = (n + 63) // 64
    out = np.zeros((n, W), np.uint64)
    for i in range(n):
        for j in np.flatnonzero(adj_bool[i]):
            out[i, j >> 6] |= np.uint64(1) << np.uint64(j & 63)
    return out


def oracle_clique(adj_bool):
    rows_ = np.ascontiguousarray(bits_of(adj_bool))
    out = np.zeros(max(len(adj_bool), 1), np.int32)
    m = teaser_oracle_lib().orc_tm_clique(len(adj_bool), rows_.ctypes.data_as(C.POINTER(C.c_uint64)), out.ctypes.data_as(C.POINTER(C.c_int)))
    return out[:m].tolist()


def oracle_core(adj_bool):
    rows_ = np.ascontiguousarray(bits_of(adj_bool))
    out = np.zeros(max(len(adj_bool), 1), np.int32)
    teaser_oracle_lib().orc_tm_core(len(adj_bool), rows_.ctypes.data_as(C.POINTER(C.c_uint64)), out.ctypes.data_as(C.POINTER(C.c_int)))
    return out[: len(adj_bool)].tolist()


# ---------------------------------------------------------------------------------------------------------------------
# the independent restatement
# ---------------------------------------------------------------------------------------------------------------------
def py_max_clique(adj_bool):
    """Bron-Kerbosch with Tomita's pivot over every maximal clique; the largest, lexicographically smallest ascending"""
    n = len(adj_bool)
    nb = [set(np.flatnonzero(adj_bool[i]).tolist()) for i in range(n)]
    best = [None]

    def bk(R, P, X):
        if not P and not X:
            c = sorted(R)
            if best[0] is None or len(c) > len(best[0]) or (len(c) == len(best[0]) and c < best[0]):
                best[0] = c
            return
        if best[0] is not None and len(R) + len(P) < len(best[0]):
            return
        u = max(P | X, key=lambda v: len(P & nb[v]))
        for v in sorted(P - nb[u]):
            bk(R | {v}, P & nb[v], X & nb[v])
            P = P - {v}
            X = X | {v}

    if n:
        bk(set(), set(range(n)), set())
    return best[0] or []


def py_core(adj_bool):
    n = len(adj_bool)
    deg = adj_bool.sum(1).astype(int)
    alive = np.ones(n, bool)
    core = np.zeros(n, int)
    k = 0
    for _ in range(n):
        d = np.where(alive, deg, n + 1)
        v = int(np.argmin(d))
        k = max(k, int(d[v]))
        core[v] = k
        alive[v] = False
        deg[adj_bool[v] & alive] -= 1
    return core.tolist()


def np_graph(p6, noise_bound):
    s, d = p6[:, :3], p6[:, 3:]
    with np.errstate(invalid="ignore"):
        ds, dd = s[None, :, :] - s[:, None, :], d[None, :, :] - d[:, None, :]
        a = np.sqrt((ds[..., 0] * ds[..., 0] + ds[..., 1] * ds[..., 1]) + ds[..., 2] * ds[..., 2])
        b = np.sqrt((dd[..., 0] * dd[..., 0] + dd[..., 1] * dd[..., 1]) + dd[..., 2] * dd[..., 2])
        adj = np.abs(a - b) <= 2.0 * noise_bound
    np.fill_diagonal(adj, False)
    return adj


def np_vote(x, r):
    h = sorted([(x[i] - r, i + 1) for i in range(len(x))] + [(x[i] + r, -(i + 1)) for i in range(len(x))])
    with np.errstate(divide="ignore"):
        w = np.float64(1.0) / np.float64(r * r)
    rs = 0.0
    for _ in range(len(x)):
        rs += r
    dxw = dwc = sxi = sxs = 0.0
    card = 0
    best = None
    with np.errstate(all="ignore"):
        for v, key in h:
            idx, eps = abs(key) - 1, (1 if key > 0 else -1)
            X = float(x[idx])
            card += eps
            dwc += eps * w
            dxw += eps * w * X
            rs -= eps * r
            sxi += eps * X
            sxs += eps * X * X
            xh = np.float64(dxw) / np.float64(dwc)
            cost = card * xh * xh + sxs - 2 * sxi * xh + rs
            if best is None or cost < best[0]:
                best = (cost, xh)
    return float(best[1])


def np_teaser(target, source, noise_bound=0.2, min_inlier_num=8):
    t, s = np.asarray(target, F32), np.asarray(source, F32)
    out = dict(status=-1, T=None, clique=[], mask=[], info=dict(n_edges=0, max_core=0, clique_size=0, rotation_inliers=0,
                                                                 gnc_iterations=0))
    if len(t) != len(s) or len(t) <= 3:
        return out
    nb = float(F32(noise_bound))
    p6 = np.concatenate([s[:, :3], t[:, :3]], 1).astype(np.float64)
    adj = np_graph(p6, nb)
    clique = py_max_clique(adj)
    info = out["info"]
    info.update(n_edges=int(adj.sum()) // 2, max_core=max(py_core(adj)), clique_size=len(clique))
    out["clique"] = clique
    if len(clique) <= 1:
        return out
    M = len(clique)
    c = np.array(clique)
    tims = p6[np.roll(c, -1)] - p6[c]
    X, Y = tims[:, :3], tims[:, 3:]
    nb2 = (2.0 * nb) ** 2
    nb2 = 1e-2 if nb2 < 1e-16 else nb2
    w = np.ones(M)
    mu, prev = 1.0, np.inf
    it = 0
    for i in range(100):
        it = i + 1
        H = (X * w[:, None]).T @ Y
        U, _, Vt = np.linalg.svd(H)
        V = Vt.T.copy()
        if np.linalg.det(U) * np.linalg.det(V) < 0:
            V[:, 2] *= -1
        R = V @ U.T
        d = Y - X @ R.T
        r = (d[:, 0] ** 2 + d[:, 1] ** 2) + d[:, 2] ** 2
        if i == 0:
            mu = 1 / (2 * r.max() / nb2 - 1)
            if mu <= 0:
                break
        cost = float(np.sum(w * r))
        th1, th2 = (mu + 1) / mu * nb2, mu / (mu + 1) * nb2
        with np.errstate(divide="ignore", invalid="ignore"):
            mid = np.sqrt(nb2 * mu * (mu + 1) / r) - mu
        w = np.where(r >= th1, 0.0, np.where(r <= th2, 1.0, mid))
        diff = abs(cost - prev)
        mu *= 1.4
        prev = cost
        if diff < 0.005:
            break
    mask = (w >= 0.5).astype(int)
    info.update(rotation_inliers=int(mask.sum()), gnc_iterations=it)
    out["mask"] = mask.tolist()
    src, dst = p6[c, :3], p6[c, 3:]
    x = dst - src @ R.T
    tr = [np_vote(x[:, a], nb) for a in range(3)]
    cnt = int(mask.sum())
    if min_inlier_num >= 0 and cnt >= min_inlier_num:
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, tr
        out["T"] = T
        out["status"] = 1 if cnt >= 2 * min_inlier_num else 0
    return out


def assert_same(o, n, atol=1e-9):
    assert o["info"] == n["info"], (o["info"], n["info"])
    assert o["clique"] == n["clique"]
    assert o["mask"] == n["mask"]
    assert o["status"] == n["status"]
    if n["status"] >= 0:
        a, b = o["T"], n["T"]
        fin = np.isfinite(b)
        assert np.array_equal(np.isfinite(a), fin)
        assert np.allclose(a[fin], b[fin], rtol=0, atol=atol), (a, b)
    else:
        assert np.all(o["T"] == 7.0)  # untouched


# ---------------------------------------------------------------------------------------------------------------------
# the correspondence sets (shared with tests/test_gpu_teaser.py)
# ---------------------------------------------------------------------------------------------------------------------
def cases():
    """(name, target, source, kwargs)"""
    out = []
    for r in (0.05, 0.2, 0.5, 1.0):
        t, s, _ = scene(120, r, 300 + int(r * 100))
        out.append((f"known_{int(r * 100)}pct", t, s, {}))
    t, s, _ = scene(50, 1.0, 3)
    out += [("n3", t[:3], s[:3], {}), ("n4", t[:4], s[:4], dict(min_inlier_num=2)), ("n4_min0", t[:4], s[:4], dict(min_inlier_num=0)),
            ("sizes_differ", t[:20], s[:21], {})]
    rng = np.random.default_rng(11)
    # no edges: source and target spread on incommensurate scales
    src = rng.uniform(-50, 50, (40, 3))
    out.append(("no_edges", rows(src * 0.01), rows(src), dict(noise_bound=0.01)))
    # a complete graph: every pair consistent under a noise bound larger than the scene
    t, s, _ = scene(60, 0.3, 12, extent=1.0)
    out.append(("complete", t, s, dict(noise_bound=5.0)))
    # two disjoint maximum cliques of 12: two rigid groups with their own motions, far apart, plus outliers
    a = rng.uniform(-5, 5, (12, 3))
    b = rng.uniform(-5, 5, (12, 3)) + 200.0
    o = rng.uniform(-300, 300, (16, 3))
    src = np.concatenate([o[:8], a, o[8:12], b, o[12:]])
    tgt = np.concatenate([rng.uniform(-300, 300, (8, 3)), a @ rot(0.3, 0, 0).T + 1, rng.uniform(-300, 300, (4, 3)),
                          b @ rot(0, 0.5, 0).T - 7, rng.uniform(-300, 300, (4, 3))])
    out.append(("two_max_cliques", rows(tgt), rows(src), dict(noise_bound=0.05, min_inlier_num=4)))
    # noise-free: every residual of the first fit is tiny, mu <= 0 ends GNC at once
    t, s, _ = scene(80, 0.5, 13, noise=0.0)
    out.append(("noise_free", t, s, {}))
    out.append(("noise_bound_zero", t, s, dict(noise_bound=0.0)))
    # duplicated points: zero-length TIMs inside the clique
    t, s, _ = scene(60, 0.8, 14)
    t2, s2 = t.copy(), s.copy()
    t2[5:10], s2[5:10] = t2[4], s2[4]
    out.append(("duplicates", t2, s2, {}))
    # a collinear clique: a degenerate H
    line = np.outer(rng.uniform(-20, 20, 40), [0.6, 0.8, 0.0]) + [1.0, 2.0, 3.0]
    out.append(("collinear", rows(line @ rot(0.1, 0.2, 0.3).T + 1.0), rows(line), {}))
    # 180 degree rotations about z and about a skew axis
    t, s, _ = scene(60, 1.0, 15)
    src = s[:, :3].astype(np.float64)
    out.append(("rot180_z", rows(src @ np.diag([-1.0, -1.0, 1.0]).T + [3, 4, 5]), s, {}))
    ax = np.array([1.0, 2.0, 2.0]) / 3.0
    R180 = 2 * np.outer(ax, ax) - np.eye(3)
    out.append(("rot180_skew", rows(src @ R180.T), s, {}))
    # voting ties: a pure translation on an integer lattice with noise_bound 0.5, boundaries landing on equal values
    grid = np.array([[i, j, k] for i in range(4) for j in range(3) for k in range(2)], np.float64)
    out.append(("vote_ties", rows(grid + [1.0, 0.0, 0.5]), rows(grid), dict(noise_bound=0.5)))
    # noise_bound 0 where every TIM length matches exactly: a complete graph, ranges of 0 and a NaN translation
    out.append(("noise_bound_zero_exact", rows(grid + [1.0, 0.0, 0.5]), rows(grid), dict(noise_bound=0.0)))
    # a NaN row
    t, s, _ = scene(60, 0.7, 16)
    s2 = s.copy()
    s2[7, 0] = np.nan
    out.append(("nan_row", t, s2, {}))
    t, s, _ = scene(60, 0.7, 17)
    out.append(("min_inlier_negative", t, s, dict(min_inlier_num=-3)))
    out.append(("min_inlier_0", t, s, dict(min_inlier_num=0)))
    return out


CASES = cases()


# ---------------------------------------------------------------------------------------------------------------------
# the tests
# ---------------------------------------------------------------------------------------------------------------------
def random_graph(n, p, seed):
    rng = np.random.default_rng(seed)
    a = rng.random((n, n)) < p
    a = np.triu(a, 1)
    return a | a.T


def planted_graph(n, k, copies, seed):
    """a sparse random graph with `copies` planted cliques of k vertices, shuffled"""
    rng = np.random.default_rng(seed)
    a = random_graph(n, 0.1, seed)
    perm = rng.permutation(n)
    for c in range(copies):
        idx = perm[c * k: (c + 1) * k]
        a[np.ix_(idx, idx)] = True
    np.fill_diagonal(a, False)
    return a


GRAPHS = [(n, p, seed) for seed, (n, p) in enumerate([(60, 0.05), (60, 0.2), (60, 0.35), (55, 0.5), (50, 0.65), (45, 0.8),
                                                      (30, 0.95), (40, 0.9), (1, 0.5), (2, 1.0), (64, 0.3), (65, 0.3)])]


@pytest.mark.parametrize("n,p,seed", GRAPHS)
def test_clique_equals_bron_kerbosch(n, p, seed):
    a = random_graph(n, p, seed)
    assert oracle_clique(a) == py_max_clique(a)
    assert oracle_core(a) == py_core(a)


@pytest.mark.parametrize("k,copies,seed", [(6, 2, 1), (5, 3, 2), (8, 4, 3), (4, 6, 4)])
def test_clique_lex_rule_among_equal_maxima(k, copies, seed):
    a = planted_graph(60, k, copies, seed)
    got = oracle_clique(a)
    assert got == py_max_clique(a)
    assert len(got) >= k


@pytest.mark.parametrize("name,target,source,kw", CASES, ids=[c[0] for c in CASES])
def test_oracle_equals_numpy_restatement(name, target, source, kw):
    # a collinear clique leaves the rotation about its line to the SVD's own steps: everything but the matrix must agree
    assert_same(oracle_teaser(target, source, **kw), np_teaser(target, source, **kw), atol=1e9 if name == "collinear" else 1e-9)


def test_case_outcomes_cover_the_branches():
    res = {name: oracle_teaser(t, s, **kw) for name, t, s, kw in CASES}
    assert res["n3"]["status"] == -1 and res["n3"]["info"]["n_edges"] == 0
    assert res["n4"]["info"]["clique_size"] == 4 and res["n4"]["status"] >= 0
    assert res["sizes_differ"]["status"] == -1 and res["sizes_differ"]["info"]["clique_size"] == 0
    assert res["no_edges"]["info"]["n_edges"] == 0 and res["no_edges"]["status"] == -1
    assert res["complete"]["info"]["n_edges"] == 60 * 59 // 2 and res["complete"]["clique"] == list(range(60))
    c = res["two_max_cliques"]["clique"]
    assert c == list(range(8, 20)), c  # the first group: the lexicographically smaller of two 12-cliques
    assert res["noise_free"]["info"]["gnc_iterations"] == 1 and res["noise_free"]["status"] == 1
    assert res["noise_bound_zero"]["status"] == -1
    z = res["noise_bound_zero_exact"]
    assert z["info"]["clique_size"] == 24 and z["status"] == 1 and not np.any(np.isfinite(z["T"][:3, 3]))
    assert res["collinear"]["info"]["clique_size"] == 40
    for name in ("rot180_z", "rot180_skew"):
        assert res[name]["status"] == 1
    assert 7 not in res["nan_row"]["clique"]
    assert res["min_inlier_negative"]["status"] == -1 and res["min_inlier_0"]["status"] == 1


def test_vote_ties_are_in_key_order():
    """the lattice case has equal boundaries; the sort puts them in ascending signed key order (T9)"""
    _, t, s, kw = next(c for c in CASES if c[0] == "vote_ties")
    o = oracle_teaser(t, s, **kw)
    assert o["status"] == 1
    assert np.allclose(o["T"][:3, 3], [1.0, 0.0, 0.5], atol=0.5)


@pytest.mark.parametrize("ratio,n", [(0.05, 400), (0.2, 400), (0.5, 400), (1.0, 400)])
def test_known_motion_is_recovered(ratio, n):
    t, s, T = scene(n, ratio, 700 + int(ratio * 100))
    o = oracle_teaser(t, s)
    k = int(round(ratio * n))
    assert o["status"] == 1
    assert k * 0.9 <= o["info"]["clique_size"] <= k + 2
    assert np.abs(o["T"][:3, :3] - T[:3, :3]).max() < 2e-3 and np.abs(o["T"][:3, 3] - T[:3, 3]).max() < 0.05


def test_dropin_teaser_compiles_and_links():
    """Without a GPU every call reports the missing device, returns -1 and leaves tran_mat alone."""
    import torch

    with tempfile.TemporaryDirectory() as td:
        exe = build_caller(td, "teaser_caller")
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
        build_caller(td, "dropin_caller")
    assert out.returncode == 0, out.stdout + out.stderr
    assert "teaser drop-in compiled and linked" in out.stdout and "failures 0" in out.stdout
    if not torch.cuda.is_available():
        assert "ran on a device: 0" in out.stdout
