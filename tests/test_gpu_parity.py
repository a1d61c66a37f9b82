"""GPU parity tests: the CUDA path (through the C-ABI) against the CPU oracle on the same inputs.

Bar (BASELINE.json north_star): pose within 1e-4 m / 1e-4 rad of the reference-shaped CPU path;
return code, executed iteration count and per-class correspondence/source counts EXACTLY equal in
every iteration. The normal equations are compared to 1e-9 relative (fp64 sums in a different,
deterministic, order)."""
import os

import numpy as np
import pytest

from conftest import load_golden_pair
from mulls_b200 import abi, synth

pytestmark = pytest.mark.gpu

POSE_TOL_M = 1e-4
POSE_TOL_RAD = 1e-4


@pytest.fixture(scope="module")
def ctx():
    from mulls_b200.registration import Context

    c = Context(0, 8, 700000, 700000)
    yield c
    c.close()


def assert_parity(gpu, gtrace, ora, otrace):
    assert gpu["code"] == ora["code"]
    assert gpu["iters"] == ora["iters"]
    assert gpu["n_corr"] == ora["n_corr"]
    assert gpu["n_src"] == ora["n_src"]
    if gtrace is not None:
        assert gtrace["n_iter"] == otrace["n_iter"]
        np.testing.assert_array_equal(gtrace["n_corr"], otrace["n_corr"])
        np.testing.assert_array_equal(gtrace["n_src"], otrace["n_src"])
        for i in range(otrace["n_iter"]):
            scale = max(np.abs(otrace["atpa"][i]).max(), 1e-300)
            np.testing.assert_allclose(gtrace["atpa"][i], otrace["atpa"][i], rtol=0, atol=1e-9 * scale)
            bs = max(np.abs(otrace["atpb"][i]).max(), 1e-300)
            np.testing.assert_allclose(gtrace["atpb"][i], otrace["atpb"][i], rtol=0, atol=1e-9 * bs)
    dt, dr = synth.pose_error(gpu["T"], ora["T"])
    assert dt <= POSE_TOL_M and dr <= POSE_TOL_RAD, (dt, dr)
    np.testing.assert_allclose(gpu["sigma"], ora["sigma"], rtol=1e-5)
    np.testing.assert_allclose(gpu["confidence"], ora["confidence"], rtol=1e-6)
    iscale = max(np.abs(ora["info"]).max(), 1e-300)
    np.testing.assert_allclose(gpu["info"], ora["info"], rtol=0, atol=1e-6 * iscale)


def run_both(ctx, oracle_mod, pair):
    g, gt = ctx.run_batch([pair], want_trace=True)
    o, ot = oracle_mod.icp_run(pair["tgt"], pair["src"], pair["params"], pair["init_guess"])
    return g[0], gt[0], o, ot


def test_small_pair(ctx, oracle_mod, small_pair):
    assert_parity(*run_both(ctx, oracle_mod, small_pair))


@pytest.mark.parametrize("name", ["synth_small.npz", "demo_pair.npz", "demo_pair_reg.npz"])
def test_golden_fixtures(ctx, golden_dir, name):
    """Against the committed golden outputs (no oracle call: the fixture is the expectation)."""
    pair, exp = load_golden_pair(os.path.join(golden_dir, name))
    g, gt = ctx.run_batch([pair], want_trace=True)
    g, gt = g[0], gt[0]
    assert g["code"] == int(exp["code"]) and g["iters"] == int(exp["iters"])
    np.testing.assert_array_equal(gt["n_corr"], exp["trace_n_corr"])
    np.testing.assert_array_equal(gt["n_src"], exp["trace_n_src"])
    dt, dr = synth.pose_error(g["T"], exp["T"])
    assert dt <= POSE_TOL_M and dr <= POSE_TOL_RAD
    for i in range(int(exp["iters"])):
        scale = np.abs(exp["trace_atpa"][i]).max()
        np.testing.assert_allclose(gt["atpa"][i], exp["trace_atpa"][i], rtol=0, atol=1e-9 * scale)


def test_full_size_c2(ctx, oracle_mod):
    """BASELINE config 2: 120k-point 64-beam scan pair."""
    pair = synth.make_pair(1001, "c2")
    assert sum(len(s) for s in pair["src"]) == 120000
    g, gt, o, ot = run_both(ctx, oracle_mod, pair)
    assert_parity(g, gt, o, ot)
    dt, dr = synth.pose_error(g["T"], pair["T_gt"])
    assert dt < 0.02 and dr < 2e-3  # and both recover the ground-truth motion


def test_scan_to_map_c3_shape(ctx, oracle_mod):
    """BASELINE config 3 shape (source vs 5-scan map, non-identity initial guess), at 1/4 size."""
    pair = synth.make_pair(1002, "c3", n_points=30000)
    assert_parity(*run_both(ctx, oracle_mod, pair))


def test_reference_call_site_parameter_sets(ctx, oracle_mod, small_pair):
    """The parameter sets of the reference's call sites (SURVEY Appendix C)."""
    base = small_pair
    variants = []
    p = abi.IcpParams.from_buffer_copy(base["params"])  # mulls_reg.cpp:194-195 with run script values
    p.max_iter_num, p.dis_thre_unit, p.dis_thre_min = 10, 3.0, 0.75
    p.weight_strategy, p.pt2pt_residual_window, p.pt2pl_residual_window, p.pt2li_residual_window = b"1101", 0.1, 0.1, 0.1
    p.normal_bearing, p.converge_translation, p.converge_rotation_d = 45.0, 0.001, 0.01
    variants.append(p)
    p = abi.IcpParams.from_buffer_copy(base["params"])  # mulls_slam.cpp:642-648 (features 111000)
    p.used_feature_type, p.sigma_thre = b"111000", 0.35
    variants.append(p)
    p = abi.IcpParams.from_buffer_copy(base["params"])  # map-to-map style: 3 iterations, wider thresholds
    p.max_iter_num, p.dis_thre_unit, p.dis_thre_min, p.weight_strategy = 3, 2.1, 0.75, b"1101"
    p.normal_bearing = 30.0
    variants.append(p)
    p = abi.IcpParams.from_buffer_copy(base["params"])  # equal weights, no intersection filter, vertex on
    p.weight_strategy, p.apply_intersection_filter, p.used_feature_type = b"0000", 0, b"111111"
    variants.append(p)
    for p in variants:
        pair = dict(base, params=p)
        assert_parity(*run_both(ctx, oracle_mod, pair))


def test_status_codes_and_early_exits(ctx, oracle_mod, small_pair):
    cases = []
    init = np.eye(4)
    init[0, 3] = 500.0
    cases.append((small_pair["params"], init))  # -2
    p = abi.IcpParams.from_buffer_copy(small_pair["params"])
    p.sigma_thre = 1e-4
    cases.append((p, np.eye(4)))  # -3
    p = abi.IcpParams.from_buffer_copy(small_pair["params"])
    p.max_iter_num = 1
    cases.append((p, np.eye(4)))
    p = abi.IcpParams.from_buffer_copy(small_pair["params"])
    p.max_iter_num = 0
    cases.append((p, small_pair["init_guess"]))  # code 0
    p = abi.IcpParams.from_buffer_copy(small_pair["params"])
    p.dis_thre_unit, p.dis_thre_min, p.max_bearable_rotation_d = 1.4, 0.5, 0.001  # -1: rotation step too large
    cases.append((p, np.eye(4)))
    codes = []
    for p, init in cases:
        pair = dict(small_pair, params=p, init_guess=init)
        g, gt, o, ot = run_both(ctx, oracle_mod, pair)
        assert_parity(g, gt, o, ot)
        codes.append(g["code"])
    assert codes[0] == -2 and codes[1] == -3 and codes[3] == 0 and codes[4] == -1


def test_vertex_class_and_point_to_point(ctx, oracle_mod, small_pair):
    """pt2pt metric (off in the shipped configs) incl. the aliased residual weight (Q2)."""
    tgt = list(small_pair["tgt"])
    src = list(small_pair["src"])
    tgt[abi.VERTEX] = small_pair["tgt"][abi.PILLAR][::3].copy()
    src[abi.VERTEX] = small_pair["src"][abi.PILLAR][::3].copy()
    p = abi.IcpParams.from_buffer_copy(small_pair["params"])
    p.used_feature_type = b"111111"
    pair = dict(small_pair, tgt=tgt, src=src, params=p)
    assert_parity(*run_both(ctx, oracle_mod, pair))


def test_empty_ragged_and_tiny_classes(ctx, oracle_mod, small_pair):
    tgt = [t.copy() for t in small_pair["tgt"]]
    src = [s.copy() for s in small_pair["src"]]
    tgt[abi.ROOF] = tgt[abi.ROOF][:2]      # < K_min on the target side
    src[abi.BEAM] = src[abi.BEAM][:0]      # empty source class
    src[abi.PILLAR] = src[abi.PILLAR][:450]  # < 500: no duplicate check, no shrinking
    pair = dict(small_pair, tgt=tgt, src=src)
    g, gt, o, ot = run_both(ctx, oracle_mod, pair)
    assert_parity(g, gt, o, ot)
    assert (gt["n_src"][:, abi.PILLAR] == 450).all()
    # everything empty: -2 at the first iteration
    empty = [np.zeros((0, 12), np.float32)] * 6
    pair = dict(small_pair, tgt=empty, src=empty)
    g, gt, o, ot = run_both(ctx, oracle_mod, pair)
    assert g["code"] == o["code"] == -2


def test_batch_equals_single_and_is_deterministic(ctx, oracle_mod, small_pair):
    """A pair gives bit-identical results alone, inside a batch, and when run twice (fixed-order reductions)."""
    other = synth.make_pair(1003, "small")
    p2 = abi.IcpParams.from_buffer_copy(small_pair["params"])
    p2.max_iter_num = 5
    third = dict(other, params=p2)
    alone, _ = ctx.run_batch([small_pair])
    batch, _ = ctx.run_batch([other, small_pair, third])
    again, _ = ctx.run_batch([other, small_pair, third])
    np.testing.assert_array_equal(alone[0]["T"], batch[1]["T"])
    np.testing.assert_array_equal(alone[0]["info"], batch[1]["info"])
    for a, b in zip(batch, again):
        np.testing.assert_array_equal(a["T"], b["T"])
        assert a["n_corr"] == b["n_corr"] and a["code"] == b["code"]
    o, _ = oracle_mod.icp_run(third["tgt"], third["src"], third["params"], third["init_guess"])
    assert batch[2]["iters"] == o["iters"] == 5 and batch[2]["n_corr"] == o["n_corr"]


def test_resident_rerun_matches_one_shot(ctx, small_pair):
    one, _ = ctx.run_batch([small_pair])
    ctx.upload([small_pair])
    r1, _ = ctx.run_resident()
    r2, _ = ctx.run_resident()
    np.testing.assert_array_equal(one[0]["T"], r1[0]["T"])
    np.testing.assert_array_equal(r1[0]["T"], r2[0]["T"])
    st = ctx.stats()
    assert st["kernel_launches"] > 0 and st["algorithmic_bytes"] > 0 and st["iterations"] == one[0]["iters"]


def test_reference_interface_mirror(oracle_mod, small_pair):
    """CRegistration.mm_lls_icp(constraint, ...) — the reference's call, argument for argument."""
    from mulls_b200.registration import CloudBlock, Constraint, CRegistration

    P = small_pair["params"]
    con = Constraint(block1=CloudBlock.from_class_list(small_pair["tgt"], local_bound=tuple(P.target_bound)),
                     block2=CloudBlock.from_class_list(small_pair["src"]))
    creg = CRegistration(0, 200000, 200000)
    code = creg.mm_lls_icp(con, P.max_iter_num, P.dis_thre_unit, P.converge_translation, P.converge_rotation_d,
                           P.dis_thre_min, P.dis_thre_update_rate, P.used_feature_type.decode(),
                           P.weight_strategy.decode(), P.z_xy_balanced_ratio, P.pt2pt_residual_window,
                           P.pt2pl_residual_window, P.pt2li_residual_window, np.eye(4), True, False, False,
                           P.normal_bearing, False, False, P.sigma_thre, P.min_neccessary_corr_ratio,
                           P.max_bearable_rotation_d)
    o, _ = oracle_mod.icp_run(small_pair["tgt"], small_pair["src"], P, np.eye(4))
    assert code == o["code"] == 1
    dt, dr = synth.pose_error(con.Trans1_2, o["T"])
    assert dt <= POSE_TOL_M and dr <= POSE_TOL_RAD


def test_motion_undistortion_variant(ctx, oracle_mod, small_pair):
    """apply_motion_undistortion_while_registration (cregistration.hpp:1248-1258): per-point slerp by the
    timestamp ratio in `curvature`, intersection filter off, vertex cloud gets the initial guess twice."""
    rng = np.random.default_rng(7)
    src = [s.copy() for s in small_pair["src"]]
    for s in src:
        s[:, 9] = rng.uniform(-0.05, 1.05, len(s)).astype(np.float32)  # a few ratios outside [0,1]: left untouched
    tgt = list(small_pair["tgt"])
    tgt[abi.VERTEX] = small_pair["tgt"][abi.PILLAR][::3].copy()
    src[abi.VERTEX] = src[abi.PILLAR][::3].copy()
    p = abi.IcpParams.from_buffer_copy(small_pair["params"])
    p.apply_motion_undistortion_while_registration = 1
    p.used_feature_type = b"111111"
    init = np.eye(4)
    init[:3, :3] = synth.rpy_matrix(0.002, -0.001, 0.012)
    init[:3, 3] = (0.9, 0.04, 0.01)
    pair = dict(small_pair, tgt=tgt, src=src, params=p, init_guess=init)
    assert_parity(*run_both(ctx, oracle_mod, pair))
    # a rotation-free initial guess exercises the linear branch of the slerp
    init2 = np.eye(4)
    init2[:3, 3] = (0.7, 0.0, 0.0)
    assert_parity(*run_both(ctx, oracle_mod, dict(pair, init_guess=init2)))


def test_4dof_global_heading_search(oracle_mod, small_pair):
    """mm_lls_icp_4dof_global (cregistration.hpp:1584-1681): the heading trials run as one batched call; the
    winner and its outputs must equal the oracle run trial by trial in the reference's loop order."""
    from mulls_b200.registration import CloudBlock, Constraint, CRegistration, heading_trial_guesses

    # rotate the source by 90 degrees about its station so that only one heading trial can succeed
    yaw = np.eye(4)
    yaw[:3, :3] = synth.rpy_matrix(0.0, 0.0, np.pi / 2)
    src = []
    for s in small_pair["src"]:
        a = s.copy()
        a[:, 0:3] = (s[:, 0:3].astype(np.float64) @ yaw[:3, :3].T).astype(np.float32)
        a[:, 4:7] = (s[:, 4:7].astype(np.float64) @ yaw[:3, :3].T).astype(np.float32)
        src.append(a)
    con = Constraint(block1=CloudBlock.from_class_list(small_pair["tgt"]), block2=CloudBlock.from_class_list(src))
    con.block2.local_station = (0.0, 0.0, 0.0)
    creg = CRegistration(0, 100000, 100000)
    ok = creg.mm_lls_icp_4dof_global(con, 45.0, max_iter_num=12, dis_thre_unit=1.5)
    # oracle, sequentially
    heads, mats = heading_trial_guesses(con.block2.local_station, 45.0)
    p = abi.default_params()
    p.max_iter_num, p.dis_thre_unit, p.converge_translation, p.converge_rotation_d = 12, 1.5, 0.005, 0.005
    p.dis_thre_min, p.dis_thre_update_rate, p.used_feature_type, p.weight_strategy = 0.5, 1.05, b"111110", b"1001"
    p.target_bound[:] = list(con.block1.local_bound)
    best, best_h, best_r = 0.0, None, None
    for h, m in zip(heads, mats):
        r, _ = oracle_mod.icp_run(con.block1.clone_feature(False), con.block2.clone_feature(True), p, m, want_trace=False)
        if r["code"] > 0:
            score = np.float32(r["confidence"]) / np.float32(r["sigma"])
            if score > best:
                best, best_h, best_r = float(score), h, r
    assert ok == (best_r is not None) and ok
    assert creg.best_heading_d == best_h
    dt, dr = synth.pose_error(con.Trans1_2, best_r["T"])
    assert dt <= POSE_TOL_M and dr <= POSE_TOL_RAD
    np.testing.assert_allclose(con.sigma, best_r["sigma"], rtol=1e-5)


def test_keep_less_source_points(ctx, oracle_mod, small_pair):
    """keep_less_source_pts (cregistration.hpp:2866-2892) with the reproducible sampling rule; also the
    map-to-map call-site shape of test/mulls_slam.cpp:477-482 (3 iterations, wider thresholds)."""
    for seed, iters in ((7, 20), (123456, 3)):
        p = abi.IcpParams.from_buffer_copy(small_pair["params"])
        p.keep_less_source_points, p.use_more_points, p.random_seed, p.max_iter_num = 1, 1, seed, iters
        g, gt, o, ot = run_both(ctx, oracle_mod, dict(small_pair, params=p))
        assert_parity(g, gt, o, ot)
        nt = [len(t) for t in small_pair["tgt"]]
        assert gt["n_src"][0][abi.GROUND] <= nt[abi.GROUND] // 2 // 4  # source ground <= |target ground / 2| / 4
    # different seeds pick different subsets
    p1 = abi.IcpParams.from_buffer_copy(small_pair["params"])
    p1.keep_less_source_points, p1.random_seed = 1, 1
    p2 = abi.IcpParams.from_buffer_copy(small_pair["params"])
    p2.keep_less_source_points, p2.random_seed = 1, 2
    r1, _ = ctx.run_batch([dict(small_pair, params=p1)])
    r2, _ = ctx.run_batch([dict(small_pair, params=p2)])
    assert not np.array_equal(r1[0]["T"], r2[0]["T"])


def test_pipelined_context_equals_single_context(small_pair):
    """PipelinedContext: the batch is split over independent contexts (own stream + host thread each); results are
    bit-identical to one context, for one-shot and resident runs, with fewer pairs than contexts too."""
    from mulls_b200.registration import Context, PipelinedContext

    pairs = [small_pair, synth.make_pair(1003, "small"), small_pair, synth.make_pair(1004, "small"), small_pair]
    one = Context(0, 5, 100000, 100000)
    ref, _ = one.run_batch(pairs)
    pipe = PipelinedContext(0, 3, 2, 100000, 100000)
    got, tr = pipe.run_batch(pairs, want_trace=True)
    assert len(got) == len(tr) == len(pairs)
    for a, b in zip(ref, got):
        np.testing.assert_array_equal(a["T"], b["T"])
        assert a["code"] == b["code"] and a["n_corr"] == b["n_corr"]
    assert tr[4]["n_iter"] == got[4]["iters"]
    pipe.upload(pairs)
    again, _ = pipe.run_resident()
    assert len(again) == len(pairs)
    for a, b in zip(ref, again):
        np.testing.assert_array_equal(a["T"], b["T"])
        assert a["code"] == b["code"] and a["n_corr"] == b["n_corr"]
    st = pipe.stats()
    assert sum(s["iterations"] for s in st) == sum(r["iters"] for r in ref)
    assert sum(s["kernel_launches"] for s in st) > 0
    few, _ = pipe.run_batch(pairs[:2])  # fewer pairs than contexts
    np.testing.assert_array_equal(few[1]["T"], ref[1]["T"])
    one.close()
    pipe.close()


def test_normal_shooting_correspondences(ctx, oracle_mod, small_pair):
    """normal_shooting_on (cregistration.hpp:1730-1739): exact 10-NN, minimum distance to the source normal line,
    for ground / facade / roof; also with the intersection filter off (sources outside the target grid)."""
    p = abi.IcpParams.from_buffer_copy(small_pair["params"])
    p.normal_shooting_on = 1
    assert_parity(*run_both(ctx, oracle_mod, dict(small_pair, params=p)))
    p2 = abi.IcpParams.from_buffer_copy(p)
    p2.apply_intersection_filter = 0
    init = np.eye(4)
    init[:3, 3] = (0.4, -0.3, 0.02)
    assert_parity(*run_both(ctx, oracle_mod, dict(small_pair, params=p2, init_guess=init)))
    tiny = dict(small_pair, params=p, tgt=[t[:7] for t in small_pair["tgt"]])  # fewer than 10 targets per class
    g, gt, o, ot = run_both(ctx, oracle_mod, tiny)
    assert g["code"] == o["code"] and g["n_corr"] == o["n_corr"]


def test_host_packed_wire_format_is_bit_identical(oracle_mod, small_pair):
    """The "host_pack" tunable repacks the 48-byte rows to the 28 B (32 B with motion undistortion) wire format on
    the host cores before the DMA (csrc/host_pack.h). Every result bit must be the same as with the raw rows: one
    context, a pipelined context (its contexts share the worker pool), resident re-runs, the undistortion variant (format 2),
    ragged / empty classes, and the resident-map path (device rows for the target, packed source)."""
    from mulls_b200.map_manager import LocalMap
    from mulls_b200.registration import Context, PipelinedContext

    rng = np.random.default_rng(11)
    src_u = [s.copy() for s in small_pair["src"]]
    for s in src_u:
        s[:, 9] = rng.uniform(-0.05, 1.05, len(s)).astype(np.float32)
    pu = abi.IcpParams.from_buffer_copy(small_pair["params"])
    pu.apply_motion_undistortion_while_registration = 1
    init = np.eye(4)
    init[:3, :3] = synth.rpy_matrix(0.002, -0.001, 0.012)
    init[:3, 3] = (0.9, 0.04, 0.01)
    undist = dict(small_pair, src=src_u, params=pu, init_guess=init)
    ragged = dict(small_pair, src=[small_pair["src"][0][:1001], small_pair["src"][1][:3], small_pair["src"][2][:2502],
                                   small_pair["src"][3][:0], small_pair["src"][4][:7], small_pair["src"][5]])
    pairs = [small_pair, undist, synth.make_pair(1003, "small"), ragged, small_pair]

    raw = Context(0, 5, 100000, 100000)
    ref, ref_tr = raw.run_batch(pairs, want_trace=True)
    o, _ = oracle_mod.icp_run(undist["tgt"], undist["src"], undist["params"], undist["init_guess"])
    assert ref[1]["code"] == o["code"] and ref[1]["n_corr"] == o["n_corr"]

    def same(got, got_tr=None):
        for i, (a, b) in enumerate(zip(ref, got)):
            assert a["code"] == b["code"] and a["iters"] == b["iters"] and a["n_corr"] == b["n_corr"], i
            np.testing.assert_array_equal(a["T"], b["T"])
            np.testing.assert_array_equal(a["info"], b["info"])
            if got_tr is not None:
                np.testing.assert_array_equal(ref_tr[i]["atpa"], got_tr[i]["atpa"])

    raw.set_tunable("host_pack", 1)
    raw.set_tunable("pack_threads", 3)
    same(*raw.run_batch(pairs, want_trace=True))
    raw.upload(pairs)
    same(raw.run_resident()[0])
    same(raw.run_resident()[0])
    one, _ = raw.run_batch([ragged])
    np.testing.assert_array_equal(one[0]["T"], ref[3]["T"])
    raw.close()

    pipe = PipelinedContext(0, 3, 2, 100000, 100000)
    pipe.set_tunable("host_pack", 1)
    same(*pipe.run_batch(pairs, want_trace=True))
    pipe.upload(pairs)
    same(pipe.run_resident()[0])
    pipe.close()

    # resident map as the target (rows stay in HBM as 48-byte rows), packed source
    pr = synth.make_pair(21, "small")
    ctx = Context(0, 1, 60000, 60000)
    lm = LocalMap(ctx, 1 << 16)
    lm.set(pr["tgt"], np.eye(4))
    r0, t0 = lm.icp_run(pr["src"], pr["params"], pr["init_guess"], want_trace=True)
    ctx.set_tunable("host_pack", 1)
    r1, t1 = lm.icp_run(pr["src"], pr["params"], pr["init_guess"], want_trace=True)
    assert r0["code"] == r1["code"] == 1
    assert np.array_equal(r0["T"], r1["T"]) and np.array_equal(t0["atpa"], t1["atpa"])
    lm.close()
    ctx.close()


def test_graph_loop_equals_host_loop(oracle_mod, small_pair):
    """The iteration loop as ONE CUDA-graph launch (device-side WHILE, the default) and as the host launch loop
    (use_graph = 0, the path the bench times per kernel) give bit-identical results and traces — also when the pairs
    of a batch stop at different iterations, when one fails early (-1 / -2), and for max_iter = 1."""
    from mulls_b200.registration import Context

    pairs = [small_pair]
    p = abi.IcpParams.from_buffer_copy(small_pair["params"])
    p.max_iter_num = 1
    pairs.append(dict(small_pair, params=p))
    p = abi.IcpParams.from_buffer_copy(small_pair["params"])
    p.max_iter_num = 3
    pairs.append(dict(small_pair, params=p))
    far = np.eye(4)
    far[0, 3] = 40.0  # nothing within the correspondence threshold: code -2 in the first iteration
    pairs.append(dict(small_pair, init_guess=far))
    out = {}
    for mode in (1, 0):
        ctx = Context(0, len(pairs), 30000, 30000)
        ctx.set_tunable("use_graph", mode)
        with pytest.raises(RuntimeError):  # the search parameters are constants of the kernels, not tunables
            ctx.set_tunable("leaf_count", 16)
        out[mode] = ctx.run_batch(pairs, want_trace=True)
        again = ctx.run_batch(pairs, want_trace=True)  # the recorded graph is re-launched, not rebuilt
        for a, b in zip(out[mode][0], again[0]):
            assert np.array_equal(a["T"], b["T"]) and a["iters"] == b["iters"]
        ctx.close()
    for (a, ta), (b, tb) in zip(zip(*out[1]), zip(*out[0])):
        assert a["code"] == b["code"] and a["iters"] == b["iters"] and a["n_corr"] == b["n_corr"]
        assert np.array_equal(a["T"], b["T"]) and np.array_equal(a["info"], b["info"])
        assert ta["n_iter"] == tb["n_iter"]
        np.testing.assert_array_equal(ta["atpa"], tb["atpa"])
        np.testing.assert_array_equal(ta["n_src"], tb["n_src"])
    assert [r["code"] for r in out[1][0]] == [1, 1, 1, -2] and [r["iters"] for r in out[1][0]][1:3] == [1, 3]
    o, ot = oracle_mod.icp_run(small_pair["tgt"], small_pair["src"], small_pair["params"], small_pair["init_guess"])
    assert_parity(out[1][0][0], out[1][1][0], o, ot)


def test_nn_query_stands_in_for_the_target_kdtrees(ctx, oracle_mod, small_pair):
    """mulls_nn_query = block1->tree_*->nearestKSearch(p, 1) (src/map_manager.cpp:221-258 on the trees of
    cregistration.hpp:1213-1232): on the clouds the oracle's mm_lls_icp built its trees on, the same neighbour and the
    same float distance for scan points and for arbitrary points, 'nothing' beyond the registration's search radius."""
    g, _ = ctx.run_batch([small_pair])
    res, trees = oracle_mod.icp_run_trees(small_pair["tgt"], small_pair["src"], small_pair["params"], small_pair["init_guess"])
    rng = np.random.default_rng(5)
    rmax = 2.5 * small_pair["params"].dis_thre_unit
    for c in (abi.PILLAR, abi.FACADE, abi.BEAM, abi.GROUND):
        tree_cloud = trees[c]
        if len(tree_cloud) < 3:
            continue
        q = np.concatenate([small_pair["src"][c][:400, :3] + rng.normal(0, 0.2, (len(small_pair["src"][c][:400]), 3)),
                            rng.uniform(-30, 30, (200, 3))]).astype(np.float32)
        rows = np.zeros((len(q), 12), np.float32)
        rows[:, :3] = q
        oi, od = oracle_mod.nn(tree_cloud, rows, 1e9)
        idx, d2 = ctx.nn_query(c, q)
        inside = od.astype(np.float64) <= np.float64(np.float32(rmax)) ** 2
        assert inside.sum() > 100
        np.testing.assert_array_equal(d2[inside], od[inside])
        # indices: the oracle's are into its filtered clone, ours into the caller's cloud — the POINTS must coincide
        np.testing.assert_array_equal(small_pair["tgt"][c][idx[inside], :3], tree_cloud[oi[inside], :3])
        assert np.all(idx[~inside] == -1) and np.all(np.isinf(d2[~inside]))
    fresh = type(ctx)(0, 1, 1000, 1000)
    with pytest.raises(RuntimeError):
        fresh.nn_query(0, np.zeros((1, 3), np.float32))
    fresh.close()


def test_kept_matches_over_twenty_forced_iterations(ctx, oracle_mod, small_pair):
    """k_search keeps a match without searching once its certificate allows (DESIGN.md 4.2): with the convergence test
    switched off every iteration from the fourth on runs in keep mode, the last ones keeping nearly everything — counts and
    normal equations must still equal the oracle's in each of the 20 iterations, through the graph and the host loop."""
    p = abi.IcpParams.from_buffer_copy(small_pair["params"])
    p.converge_translation, p.converge_rotation_d = 0.0, 0.0
    pair = dict(small_pair, params=p)
    o, ot = oracle_mod.icp_run(pair["tgt"], pair["src"], pair["params"], pair["init_guess"])
    assert o["iters"] == 20
    for use_graph in (1, 0):
        ctx.set_tunable("use_graph", use_graph)
        g, gt = ctx.run_batch([pair], want_trace=True)
        assert_parity(g[0], gt[0], o, ot)
    ctx.set_tunable("use_graph", 1)
    # and with a wrong first guess: big early corrections, matches change for several iterations before they settle
    init = np.array(small_pair["init_guess"], np.float64).copy()
    init[0, 3] += 0.6
    init[1, 3] -= 0.4
    pair2 = dict(pair, init_guess=init)
    assert_parity(*run_both(ctx, oracle_mod, pair2))
