"""The ICP iteration against the oracle where the small-batch tests do not reach: the adversarial scenes of
icp_scenes.py through each loop implementation, a mixed resident batch in the graph body, and the bench's own 64-pair
batch.

The loop runs three ways (DESIGN §4.3): the cooperative kernel k_icp_loop (use_graph on, every chunk and pair co-resident),
the recorded graph's WHILE body (use_graph on, a batch larger than the cooperative kernel holds), and the host launch loop
(use_graph = 0). Which one ran is read off the kernel launch count: the cooperative kernel is one launch for all iterations,
the host loop enqueues at least four kernels per iteration, and the graph body records six. Every comparison uses
test_gpu_parity.assert_parity: code, iteration count and per-class counts equal in every iteration, ATPA / ATPb to 1e-9 of
their scale, pose to 1e-4 m / 1e-4 rad."""
import multiprocessing
import os
import time
from concurrent.futures import ProcessPoolExecutor, ThreadPoolExecutor

import numpy as np
import pytest

import icp_scenes as S
from mulls_b200 import abi, synth
from test_gpu_parity import assert_parity

pytestmark = pytest.mark.gpu

BENCH_PAIRS = 64
GRAPH_FILL = (1001, 1005, 1006)  # three C2 pairs: ~2 800 source chunks; an H100 holds at most 16 x 132 co-resident blocks


def sizes(pairs):
    return (max(max(sum(len(c) for c in q["src"]) for q in pairs), 1),
            max(max(sum(len(c) for c in q["tgt"]) for q in pairs), 1))


def context(pairs):
    from mulls_b200.registration import Context

    return Context(0, len(pairs), *sizes(pairs))


def oracle_all(oracle_mod, pairs):
    """The oracle once per pair, on the host's cores (the ctypes call releases the GIL)."""
    def one(q):
        return oracle_mod.icp_run(q["tgt"], q["src"], q["params"], q["init_guess"], threads=1)

    with ThreadPoolExecutor(max(1, min(len(pairs), os.cpu_count() or 1))) as ex:
        return list(ex.map(one, pairs))


def _gen(seed):
    p = synth.make_pair(seed, "c2")
    return dict(tgt=p["tgt"], src=p["src"], params=bytes(p["params"]), init_guess=p["init_guess"])


def c2_pairs(seeds):
    workers = max(1, min(len(seeds), (os.cpu_count() or 2) // 2, 16))
    with ProcessPoolExecutor(workers, mp_context=multiprocessing.get_context("spawn")) as ex:  # (no fork of a CUDA process)
        raw = list(ex.map(_gen, seeds))
    for r in raw:
        r["params"] = abi.IcpParams.from_buffer_copy(r["params"])
    return raw


def same_bits(a, ta, b, tb, what):
    for k in ("code", "iters", "n_corr", "n_src", "T", "info", "sigma", "confidence"):
        np.testing.assert_array_equal(np.asarray(a[k]), np.asarray(b[k]), err_msg=f"{what}: {k}")
    for k in ("n_iter", "atpa", "atpb", "x", "n_corr", "n_src"):
        np.testing.assert_array_equal(np.asarray(ta[k]), np.asarray(tb[k]), err_msg=f"{what}: trace {k}")


@pytest.fixture(scope="module")
def scenes(oracle_mod):
    sc = S.scenes(oracle_mod)
    names = list(sc)
    return dict(zip(names, zip(sc.values(), oracle_all(oracle_mod, list(sc.values())))))


@pytest.fixture(scope="module")
def fill(oracle_mod):
    pairs = c2_pairs(GRAPH_FILL)
    return pairs, oracle_all(oracle_mod, pairs)


@pytest.mark.parametrize("name", S.NAMES)
def test_scene_cooperative_kernel_and_host_loop(scenes, name):
    pair, (o, ot) = scenes[name]
    ctx = context([pair])
    g, gt = ctx.run_batch([pair], want_trace=True)
    coop = ctx.stats()["kernel_launches"]
    assert_parity(g[0], gt[0], o, ot)
    ctx.set_tunable("use_graph", 0)
    h, ht = ctx.run_batch([pair], want_trace=True)
    host = ctx.stats()["kernel_launches"]
    assert_parity(h[0], ht[0], o, ot)
    ctx.close()
    # same ingest both times; the host loop adds >= 4 launches per iteration, the cooperative kernel one for them all
    assert coop + 4 * o["iters"] <= host + 1, (coop, host, o["iters"])


def test_scenes_in_the_graph_body(scenes, fill):
    """All scenes resident on one context with three C2 pairs: too many chunks for the cooperative kernel, so the graph's
    WHILE body runs them, with the chunks of stopped pairs dropping out of the live lists at different iterations."""
    pairs, ora = fill
    batch = [pairs[0]] + [scenes[n][0] for n in S.NAMES] + pairs[1:]
    expect = [ora[0]] + [scenes[n][1] for n in S.NAMES] + ora[1:]
    ctx = context(batch)
    ctx.upload(batch)
    res, tr = ctx.run_resident(want_trace=True)
    iters = max(r["iters"] for r in res)
    assert ctx.stats()["kernel_launches"] >= 6 * iters
    ctx.close()
    for r, t, (o, ot) in zip(res, tr, expect):
        assert_parity(r, t, o, ot)
    assert len({r["iters"] for r in res}) >= 3


def mixed_pairs(fill):
    """C2 pairs, iteration limits 1 and 3, codes -1 / -2 / -3 (the recipes of test_status_codes_and_early_exits),
    ragged and empty classes, keep_less_source_points, motion undistortion."""
    small = S.base_pair()
    out = [fill[0][0], fill[0][1]]
    for it in (1, 3):
        p = abi.IcpParams.from_buffer_copy(small["params"])
        p.max_iter_num = it
        out.append(dict(small, params=p))
    far = np.eye(4)
    far[0, 3] = 500.0
    out.append(dict(small, init_guess=far))  # -2
    p = abi.IcpParams.from_buffer_copy(small["params"])
    p.sigma_thre = 1e-4
    out.append(dict(small, params=p))  # -3
    p = abi.IcpParams.from_buffer_copy(small["params"])
    p.dis_thre_unit, p.dis_thre_min, p.max_bearable_rotation_d = 1.4, 0.5, 0.001
    out.append(dict(small, params=p))  # -1
    s = small["src"]
    out.append(dict(small, src=[s[0][:1001], s[1][:3], s[2][:2502], s[3][:0], s[4][:7], s[5]]))
    p = abi.IcpParams.from_buffer_copy(small["params"])
    p.keep_less_source_points, p.use_more_points, p.random_seed = 1, 1, 7
    out.append(dict(small, params=p))
    rng = np.random.default_rng(7)
    src = [c.copy() for c in s]
    for c in src:
        c[:, 9] = rng.uniform(-0.05, 1.05, len(c)).astype(np.float32)
    p = abi.IcpParams.from_buffer_copy(small["params"])
    p.apply_motion_undistortion_while_registration = 1
    init = np.eye(4)
    init[:3, :3] = synth.rpy_matrix(0.002, -0.001, 0.012)
    init[:3, 3] = (0.9, 0.04, 0.01)
    out.append(dict(small, src=src, params=p, init_guess=init))
    return out


def test_mixed_batch_in_the_graph_body(oracle_mod, fill):
    batch = mixed_pairs(fill)
    ora = [fill[1][0], fill[1][1]] + oracle_all(oracle_mod, batch[2:])
    assert [o["code"] for o, _ in ora[4:7]] == [-2, -3, -1]
    assert [o["iters"] for o, _ in ora[2:4]] == [1, 3]
    ctx = context(batch)
    ctx.upload(batch)
    res, tr = ctx.run_resident(want_trace=True)
    assert ctx.stats()["kernel_launches"] >= 6 * max(r["iters"] for r in res)
    for r, t, (o, ot) in zip(res, tr, ora):
        assert_parity(r, t, o, ot)
    # the same pairs at other positions of the batch
    order = list(range(len(batch)))[::-1]
    ctx.upload([batch[k] for k in order])
    res2, tr2 = ctx.run_resident(want_trace=True)
    for i, k in enumerate(order):
        same_bits(res[k], tr[k], res2[i], tr2[i], f"pair {k} at position {i}")
    ctx.close()
    # and each pair alone
    for k, q in enumerate(batch):
        one = context([q])
        a, ta = one.run_batch([q], want_trace=True)
        one.close()
        same_bits(res[k], tr[k], a[0], ta[0], f"pair {k} alone")


def test_normal_shooting_batch(oracle_mod, fill):
    """Normal shooting switches its whole context off the cooperative kernel: a resident batch of its own."""
    small = S.base_pair()
    p = abi.IcpParams.from_buffer_copy(small["params"])
    p.normal_shooting_on = 1
    shoot = dict(small, params=p)
    batch = [shoot, fill[0][0], S.sizes_a(), shoot]
    ora = oracle_all(oracle_mod, [shoot, S.sizes_a()])
    ora = [ora[0], fill[1][0], ora[1], ora[0]]
    ctx = context(batch)
    ctx.upload(batch)
    res, tr = ctx.run_resident(want_trace=True)
    ctx.close()
    for r, t, (o, ot) in zip(res, tr, ora):
        assert_parity(r, t, o, ot)
    same_bits(res[0], tr[0], res[3], tr[3], "the shooting pair at two positions")


@pytest.fixture(scope="module")
def bench_batch(oracle_mod):
    t0 = time.perf_counter()
    pairs = c2_pairs([1000 + i for i in range(BENCH_PAIRS)])
    t1 = time.perf_counter()
    ora = oracle_all(oracle_mod, pairs)
    t2 = time.perf_counter()
    print(f"\nbench batch: {BENCH_PAIRS} C2 pairs generated in {t1 - t0:.1f} s, oracle in {t2 - t1:.1f} s "
          f"on {os.cpu_count()} host cores")
    return pairs, ora


def test_bench_batch_against_the_oracle(bench_batch):
    """synth.make_pair(1000 + i, "c2"), i < 64, resident on one context (the bench's 1_context arm), default
    convergence, every pair with its trace."""
    pairs, ora = bench_batch
    ctx = context(pairs)
    ctx.upload(pairs)
    res, tr = ctx.run_resident(want_trace=True)
    assert ctx.stats()["kernel_launches"] >= 6 * max(r["iters"] for r in res)
    ctx.close()
    for k, (r, t, (o, ot)) in enumerate(zip(res, tr, ora)):
        assert r["code"] == 1, k
        assert_parity(r, t, o, ot)


def test_bench_batch_fixed_twenty_iterations(oracle_mod, bench_batch):
    """The bench's fixed20 arm: convergence thresholds 0, every pair runs all 20 iterations (keep mode from the fourth)."""
    pairs = []
    for q in bench_batch[0]:
        p = abi.IcpParams.from_buffer_copy(q["params"])
        p.converge_translation, p.converge_rotation_d = 0.0, 0.0
        pairs.append(dict(q, params=p))
    t0 = time.perf_counter()
    ora = oracle_all(oracle_mod, pairs)
    print(f"\nfixed 20 iterations: oracle for {len(pairs)} pairs in {time.perf_counter() - t0:.1f} s")
    ctx = context(pairs)
    ctx.upload(pairs)
    res, tr = ctx.run_resident(want_trace=True)
    ctx.close()
    for r, t, (o, ot) in zip(res, tr, ora):
        assert r["iters"] == 20
        assert_parity(r, t, o, ot)
