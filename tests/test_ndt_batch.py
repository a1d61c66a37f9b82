"""CPU checks of the batched NDT registration (mulls_omp_ndt_batch):
- the Newton walk as a step function (ndt_walk_start / ndt_walk_advance of mulls_b200/csrc/ndt_core.cuh), advanced for
  every case of tests/test_ndt.py at once, one evaluation of each live walk per round as the batch call advances them
  (tests/harness/ndt_lockstep.cpp), ends each walk bit for bit as ndt_walk ends it for that case alone (orc_ndt): the
  iteration count, convergence, point counts, every Trans1_2 bit and every trace row;
- the C++ shim lo::b200::omp_ndt_batch compiles and links with the reference's omp_ndt arguments and defaults
  (tests/stubs/ndt_batch_caller.cpp)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from test_ndt import ROOT, bbox, cases, oracle_ndt, rows

_LIB = {}


def lockstep_lib():
    if "lib" in _LIB:
        return _LIB["lib"]
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available: the host instantiation of ndt_core.cuh cannot be built")
    src = os.path.join(ROOT, "tests", "harness", "ndt_lockstep.cpp")
    deps = [src, os.path.join(ROOT, "tests", "harness", "ndt_oracle.cpp"), os.path.join(ROOT, "include", "mulls_b200", "abi.h")]
    deps += [os.path.join(ROOT, "mulls_b200", "csrc", f) for f in ("ndt_core.cuh", "ransac_core.cuh", "ground_core.cuh")]
    out_dir = os.path.join(ROOT, "tests", "harness", "_build")
    out = os.path.join(out_dir, "libndt_lockstep.so")
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
    lb.orc_ndt_lockstep.restype = C.c_int
    lb.orc_ndt_lockstep.argtypes = [C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_long), C.POINTER(C.c_void_p),
                                    C.POINTER(C.c_long), C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int),
                                    C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(abi.NdtResult),
                                    C.POINTER(abi.NdtIter), C.c_int]
    _LIB["lib"] = lb
    return lb


def lockstep(case_list, cap=64):
    from mulls_b200 import abi
    n = len(case_list)
    t = [rows(c["tgt"]) for c in case_list]
    s = [rows(c["src"]) for c in case_list]
    tp = (C.c_void_p * n)(*[a.ctypes.data for a in t])
    sp = (C.c_void_p * n)(*[a.ctypes.data for a in s])
    nt = (C.c_long * n)(*[len(a) for a in t])
    ns = (C.c_long * n)(*[len(a) for a in s])
    res = (C.c_float * n)(*[c.get("res", 1.0) for c in case_list])
    flt = (C.c_int * n)(*[int(c.get("filter", True)) for c in case_list])
    g = np.concatenate([np.asarray(c.get("guess", np.eye(4)), np.float64).ravel() for c in case_list])
    tb = np.concatenate([np.asarray(c.get("tb", bbox(c["tgt"])), np.float64) for c in case_list])
    sb = np.concatenate([np.asarray(c.get("sb", bbox(c["src"])), np.float64) for c in case_list])
    out = (abi.NdtResult * n)()
    tr = (abi.NdtIter * (n * cap))()
    dp = C.POINTER(C.c_double)
    rounds = lockstep_lib().orc_ndt_lockstep(n, tp, nt, sp, ns, res, g.ctypes.data_as(dp), flt, tb.ctypes.data_as(dp),
                                             sb.ctypes.data_as(dp), out, tr, cap)
    results = []
    for i in range(n):
        r = out[i]
        k = min(r.iterations, cap)
        rw = [tr[i * cap + j] for j in range(k)]
        results.append(dict(trans=np.array(r.trans[:]).reshape(4, 4), iterations=r.iterations, converged=bool(r.converged),
                            n_target=r.n_target, n_source=r.n_source,
                            trace=dict(p=np.array([x.p[:] for x in rw]).reshape(k, 6), step=np.array([x.step for x in rw]),
                                       score=np.array([x.score for x in rw]), reversed=np.array([x.reversed for x in rw]))))
    return rounds, results


def test_lockstep_walks_equal_single_walks():
    cs = cases()
    names = list(cs)
    rounds, got = lockstep([cs[k] for k in names])
    iters = []
    for name, d in zip(names, got):
        o = oracle_ndt(cs[name])
        for k in ("iterations", "converged", "n_target", "n_source"):
            assert d[k] == o[k], (name, k, d[k], o[k])
        assert np.array_equal(d["trans"].view(np.uint64), o["trans"].view(np.uint64)), name
        assert np.array_equal(d["trace"]["reversed"], o["trace"]["reversed"]), name
        for k in ("p", "step", "score"):
            assert np.array_equal(d["trace"][k].view(np.uint64), o["trace"][k].view(np.uint64)), (name, k)
        iters.append(d["iterations"])
    # the walks end at different rounds: the live list shrinks while the longest walk (37 iterations) goes on
    assert len(set(iters)) >= 3 and max(iters) == 37 and min(iters) == 0
    assert rounds == max(iters) + 1


def test_lockstep_order_and_duplicates():
    """a walk does not depend on its neighbours in the batch: the same case three times, between others, ends alike"""
    cs = cases()
    batch = [cs["motion"], cs["far"], cs["motion"], cs["empty_source"], cs["motion"]]
    _, got = lockstep(batch)
    for i in (2, 4):
        assert got[i]["iterations"] == got[0]["iterations"]
        assert np.array_equal(got[i]["trans"].view(np.uint64), got[0]["trans"].view(np.uint64))
        assert np.array_equal(got[i]["trace"]["score"].view(np.uint64), got[0]["trace"]["score"].view(np.uint64))


def build_ndt_batch_caller(td):
    libdir = os.path.join(ROOT, "mulls_b200", "csrc")
    exe = os.path.join(td, "ndt_batch_caller")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests", "stubs", "ndt_batch_caller.cpp"),
                           "-o", exe, "-L", libdir, "-lmulls_b200", f"-Wl,-rpath,{libdir}"])
    return exe


def test_batch_shim_compiles_and_links():
    """lo::b200::omp_ndt_batch with the reference's omp_ndt arguments, once in full and once with the defaults only
    (without a GPU: every code -3, Trans1_2 untouched)"""
    import tempfile

    import torch

    with tempfile.TemporaryDirectory() as td:
        exe = build_ndt_batch_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "ndt batch shim compiled and linked" in out.stdout and "failures 0" in out.stdout
    if not torch.cuda.is_available():
        assert "ran on a device: 0" in out.stdout
