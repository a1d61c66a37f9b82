"""GPU checks of mulls_omp_ndt_batch: every pair of a batch equals, bit for bit, what mulls_omp_ndt returns for that pair
alone (code, iterations, convergence, point counts, every Trans1_2 and fitness bit, every trace row):
- every case of tests/test_ndt.py, batched by resolution, against the single call and the CPU restatement;
- the 15 consecutive pairs of tests/golden/demo_chain.npz in one batch, raw and voxel-downsampled on the device at 0.5 m;
- a shuffled batch, P = 1, and the same pair three times in one batch;
- the refusals, each naming the pair where one pair is the cause, and a refused batch writes no result;
- a batch uploaded again after the call registers as before it (the call replaces the resident batch);
- the C++ shim lo::b200::omp_ndt_batch (tests/stubs/ndt_batch_caller.cpp) returns what the library does."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from mulls_b200 import abi, synth
from mulls_b200.registration import Context
from test_gpu_ndt import assert_bit_equal, demo_pairs, device_ndt
from test_ndt import bbox, cases, oracle_ndt, rows

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, 16, 200000, 200000)
    yield c
    c.close()


def batch(ctx, cs, res=1.0, trace_cap=64, **kw):
    return ctx.omp_ndt_batch([c["tgt"] for c in cs], [c["src"] for c in cs], [c.get("tb", bbox(c["tgt"])) for c in cs],
                             [c.get("sb", bbox(c["src"])) for c in cs], res, True,
                             [c.get("guess", np.eye(4)) for c in cs], kw.get("filter", True), kw.get("thre", 10.0),
                             trace_cap=trace_cap)


def groups():
    """the cases of tests/test_ndt.py by (resolution, filter, threshold): the parameters a batch shares"""
    out = {}
    for name, c in cases().items():
        out.setdefault((c.get("res", 1.0), c.get("filter", True), c.get("thre", 10.0)), []).append(name)
    return out


@pytest.mark.parametrize("key", list(groups()), ids=lambda k: f"res{k[0]}_filter{int(k[1])}_thre{k[2]:g}")
def test_cases_equal_single_call_and_restatement(ctx, key):
    names = groups()[key]
    cs = [cases()[n] for n in names]
    got = batch(ctx, cs, key[0], filter=key[1], thre=key[2])
    for n, c, d in zip(names, cs, got):
        assert_bit_equal(d, device_ndt(ctx, c))
        assert_bit_equal(d, oracle_ndt(c))


def test_pairs_end_at_different_iterations(ctx):
    """the walks of one batch end at different rounds: a pair whose walk has ended leaves the evaluation while the
    others go on"""
    cs = cases()
    names = ["motion", "guess", "empty_source", "empty_target", "small_leaves", "filter_empties"]
    got = batch(ctx, [cs[n] for n in names])
    iters = [d["iterations"] for d in got]
    assert len(set(iters)) >= 2 and min(iters) == 0 and max(iters) >= 2, iters
    for n, d in zip(names, got):
        assert_bit_equal(d, oracle_ndt(cs[n]))


def chain(ctx, voxel):
    _, scans = demo_pairs()
    if voxel:
        scans = [ctx.voxel_downsample(np.c_[s, np.zeros((len(s), 4), np.float32)], voxel)[:, :3].copy() for s in scans]
    return [dict(tgt=scans[k], src=scans[k + 1]) for k in range(15)]


@pytest.mark.parametrize("voxel", [None, 0.5])
def test_demo_chain_equals_single_calls(ctx, voxel):
    cs = chain(ctx, voxel)
    got = batch(ctx, cs)
    for c, d in zip(cs, got):
        assert_bit_equal(d, device_ndt(ctx, c))
        assert d["n_source"] > 1000 and d["iterations"] >= 1


def test_order_and_duplicates(ctx):
    cs = cases()
    names = ["motion", "far", "guess", "non_finite", "motion_res07"]
    base = [cs[n] for n in names if cs[n].get("res", 1.0) == 1.0 and cs[n].get("filter", True)]
    ref = batch(ctx, base)
    perm = np.random.default_rng(4).permutation(len(base))
    shuffled = batch(ctx, [base[i] for i in perm])
    for j, i in enumerate(perm):
        assert_bit_equal(shuffled[j], ref[i])
    one = batch(ctx, [cs["guess"]])
    assert len(one) == 1
    assert_bit_equal(one[0], device_ndt(ctx, cs["guess"]))
    three = batch(ctx, [cs["motion"]] * 3)
    for d in three:
        assert_bit_equal(d, three[0])
    assert_bit_equal(three[0], device_ndt(ctx, cs["motion"]))


def raw_call(ctx, n, tv, sv, out, res=1.0, direct=1, g=None, tb=None, sb=None):
    dp = C.POINTER(C.c_double)
    return ctx.lib.mulls_omp_ndt_batch(ctx.handle, n, tv, sv, res, direct, None if g is None else g.ctypes.data_as(dp), 1, 10.0,
                                       None if tb is None else tb.ctypes.data_as(dp), None if sb is None else sb.ctypes.data_as(dp),
                                       out, None, 0)


def test_refusals(ctx):
    c = cases()["motion"]
    t, s = rows(c["tgt"]), rows(c["src"])
    with pytest.raises(RuntimeError, match="error -103:"):  # MULLS_E_UNSUPPORTED
        ctx.omp_ndt_batch([c["tgt"]] * 2, [c["src"]] * 2, [bbox(c["tgt"])] * 2, [bbox(c["src"])] * 2, use_direct_search=False)
    small = Context(0, 2, 5000, 5000)
    try:
        with pytest.raises(RuntimeError, match="error -102: .*3 pairs exceed max_pairs"):  # MULLS_E_CAPACITY
            small.omp_ndt_batch([c["tgt"][:100]] * 3, [c["src"][:100]] * 3, [bbox(c["tgt"])] * 3, [bbox(c["src"])] * 3)
        big = np.concatenate([c["tgt"]] * 2)  # 12 000 target points in pair 1
        with pytest.raises(RuntimeError, match="error -102: .*pair 1:"):
            small.omp_ndt_batch([c["tgt"][:100], big], [c["src"][:100]] * 2, [bbox(c["tgt"])] * 2, [bbox(c["src"])] * 2)
        # a refused batch writes no result
        tv = (abi.CloudView * 2)(abi.cloud_view(rows(c["tgt"][:100])), abi.cloud_view(rows(big)))
        sv = (abi.CloudView * 2)(abi.cloud_view(rows(c["src"][:100])), abi.cloud_view(rows(c["src"][:100])))
        out = (abi.NdtResult * 2)()
        out[0].code = out[1].code = 12345
        g, b = np.tile(np.eye(4).ravel(), 2), np.tile(bbox(c["tgt"]), 2)
        assert raw_call(small, 2, tv, sv, out, g=g, tb=b, sb=b) == -102
        assert out[0].code == 12345 and out[1].code == 12345 and out[0].iterations == 0
    finally:
        small.close()
    tv = (abi.CloudView * 2)(abi.cloud_view(t), abi.CloudView())
    sv = (abi.CloudView * 2)(abi.cloud_view(s), abi.CloudView(None, 5))  # NULL rows with n > 0 in pair 1
    out = (abi.NdtResult * 2)()
    g, b = np.tile(np.eye(4).ravel(), 2), np.tile(bbox(c["tgt"]), 2)
    assert raw_call(ctx, 2, tv, sv, out, g=g, tb=b, sb=b) == -101  # MULLS_E_ARG
    assert "pair 1" in ctx.lib.mulls_last_error(ctx.handle).decode()
    sv = (abi.CloudView * 2)(abi.cloud_view(s), abi.cloud_view(s))
    assert raw_call(ctx, 2, tv, sv, out, g=None, tb=b, sb=b) == -101  # NULL guesses
    assert raw_call(ctx, 2, tv, sv, out, g=g, tb=None, sb=b) == -101  # NULL bounds
    assert raw_call(ctx, 2, tv, sv, None, g=g, tb=b, sb=b) == -101  # NULL results
    assert raw_call(ctx, 2, tv, sv, out, res=0.0, g=g, tb=b, sb=b) == -101  # resolution <= 0
    assert raw_call(ctx, 0, tv, sv, out, g=g, tb=b, sb=b) == -101  # P = 0
    with pytest.raises(RuntimeError, match="error -101"):
        ctx.omp_ndt_batch([], [], [], [])


def test_registration_after_batch_unchanged(ctx):
    """mulls_omp_ndt_batch replaces the resident batch (its fitness search builds the targets' grids through the
    ingest): a batch uploaded again after the call registers exactly as before it"""
    pair = synth.make_pair(1000, "small")
    r0, _ = ctx.run_batch([pair], want_trace=True)
    batch(ctx, [cases()["motion"], cases()["guess"]])
    r1, _ = ctx.run_batch([pair], want_trace=True)
    assert r0[0]["code"] == r1[0]["code"] and r0[0]["iters"] == r1[0]["iters"]
    assert np.array_equal(np.asarray(r0[0]["T"]), np.asarray(r1[0]["T"]))


def test_shim_on_device(ctx):
    """lo::b200::omp_ndt_batch (tests/stubs/ndt_batch_caller.cpp) returns each pair's code and Trans1_2 as the library does"""
    from test_ndt_batch import build_ndt_batch_caller

    cs = chain(ctx, None)[:3]
    got = batch(ctx, cs)
    with tempfile.TemporaryDirectory() as td:
        exe = build_ndt_batch_caller(td)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0 and "failures 0" in out.stdout and "ran on a device: 1" in out.stdout, out.stdout + out.stderr
        args = []
        for i, c in enumerate(cs):
            tp, sp = os.path.join(td, f"t{i}.bin"), os.path.join(td, f"s{i}.bin")
            rows(c["tgt"]).tofile(tp)
            rows(c["src"]).tofile(sp)
            args += [tp, sp]
        op = os.path.join(td, "o.bin")
        r = subprocess.run([exe, op, "1.0"] + args, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        o = np.fromfile(op, np.float64).reshape(len(cs), 17)
    for d, row in zip(got, o):
        assert int(row[0]) == d["code"]
        assert np.array_equal(row[1:].reshape(4, 4), d["trans"])
