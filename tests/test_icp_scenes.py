"""Each adversarial scene of icp_scenes.py reaches the edge it is named after, in the oracle's own run (no GPU).

The numpy restatement of the loop records what determine_corres saw and returned; icp_scenes.probe requires it to equal
the oracle's counts in every iteration, so an edge seen in the record is an edge of the oracle's run."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

import icp_scenes as S
import test_oracle_fullloop_crosscheck as fl

F32, F64 = np.float32, np.float64


@pytest.fixture(scope="module")
def probed(oracle_mod):
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = S.probe(oracle_mod, S.scenes_by_name(oracle_mod, name), min_iters=1)
        return cache[name]

    return get


def ties_in(rec, it, c):
    """sources whose nearest target has an exact float-distance twin at another index"""
    r = rec[(it, c)]
    src, tgt = r["src"], r["tgt"]
    k = min(4, len(tgt))
    _, cand = cKDTree(tgt[:, 0:3].astype(F64)).query(src[:, 0:3].astype(F64), k=k)
    d2 = np.stack([fl.l2_simple(src[:, 0:3], tgt[cand[:, j], 0:3]) for j in range(k)], axis=1)
    j, best = r["nn"]
    twins = (d2 == best[:, None]) & (cand != j[:, None])
    return np.flatnonzero(twins.any(1) & (best.astype(F64) <= (2.5 * float(r["thre"])) ** 2))


def test_contention_decided_across_chunks_and_shrinks_below_500(probed):
    rec = probed("contention")
    p = S.contention()
    j, _ = rec[(0, S.B)]["nn"]
    cluster = np.arange(len(p["tgt"][S.B]) - 4, len(p["tgt"][S.B]))
    on_cluster = np.isin(j[p["contenders"]], cluster)
    assert on_cluster.sum() >= 3 * 128  # several chunks' worth of sources claim four targets
    assert np.isin(cluster, j).all()
    n_src = rec["trace"]["n_src"][:, S.B]
    assert n_src[0] >= S.DEDUP_MIN_SRC and (n_src[1:] < S.DEDUP_MIN_SRC).any()
    # the survivors on the cluster are the lowest source index claiming each target
    shrunk = rec[(0, S.B)]["out"][0]
    src0 = rec[(0, S.B)]["src"]
    for t in cluster:
        first = np.flatnonzero(j == t).min()
        assert (shrunk[:, 0:3] == src0[first, 0:3]).all(1).any()


@pytest.mark.parametrize("name,sizes", [("sizes_a", [501, 129, 500, 3, 127, 0]), ("sizes_b", [499, 128, 2, 0, 3, 0])])
def test_class_sizes_reach_the_rules(probed, name, sizes):
    rec = probed(name)
    seen = [len(rec[(0, c)]["src"]) if (0, c) in rec else 0 for c in range(6)]
    assert seen == sizes
    n_src = rec["trace"]["n_src"]
    if name == "sizes_a":  # exactly 500 is checked for duplicates and shrinks; 501 as well
        assert n_src[0][S.F] < 500 and n_src[0][S.G] < 501
        assert (n_src[:, S.PL] == 129).all() and (n_src[:, S.R] == 127).all()
    else:  # below 500 nothing shrinks; < 3 points on either side: no correspondences
        assert (n_src[:, S.G] == 499).all() and (rec["trace"]["n_corr"][:, S.F] == 0).all()
        assert (rec["trace"]["n_corr"][:, S.R] == 0).all()
    assert rec["result"]["code"] == 1 and rec["result"]["iters"] >= 4


def test_ties_occur_among_the_matches(probed):
    rec = probed("ties")
    assert len(ties_in(rec, 0, S.F)) >= 20  # duplicated facade targets
    sym = ties_in(rec, 0, S.B)
    assert len(sym) >= 8  # the symmetric pairs
    # a tie goes to the lower target index
    r = rec[(0, S.B)]
    j, d2 = r["nn"]
    for s in sym:
        same = np.flatnonzero(fl.l2_simple(r["src"][s:s + 1, 0:3], r["tgt"][:, 0:3]) == d2[s])
        assert j[s] == same.min()
    assert rec["result"]["code"] == 1 and rec["result"]["iters"] >= 4


def test_threshold_edges_are_exact(probed):
    rec = probed("thresholds")
    r = rec[(0, S.F)]
    thre = F32(r["thre"])
    j, d2 = r["nn"]
    on_rejector = np.flatnonzero(d2 == thre * thre)
    on_bound = np.flatnonzero(d2.astype(F64) == float(F32(2.5) * thre) ** 2)
    assert len(on_rejector) >= 4 and len(on_bound) >= 4
    shrunk, s_i, t_i, dd = r["out"]
    # rejector: '<' drops the exact ones; bound: '<=' keeps them through the shrink, the rejector then drops them
    assert not (dd == thre * thre).any()
    src = r["src"]
    kept_rows = {tuple(x) for x in shrunk[:, 0:3]}
    assert all(tuple(src[s, 0:3]) in kept_rows for s in on_bound)
    assert rec["result"]["code"] == 1 and rec["result"]["iters"] >= 4


def test_normal_cosine_exactly_on_the_threshold(probed):
    rec = probed("cos_edge")
    r = rec[(0, S.F)]
    assert r["cos_thre"] == 1.0
    n, m = np.array(S.COS_PASS_SRC, F32).astype(F64), np.array(S.COS_TGT, F32).astype(F64)
    dot = n[0] * m[0] + (n[1] * m[1] + n[2] * m[2])
    assert dot < 1.0 and F32(abs(dot)) == F32(1.0)
    n = np.array(S.COS_FAIL_SRC, F32).astype(F64)
    assert F32(abs(n[0] * m[0] + (n[1] * m[1] + n[2] * m[2]))) < F32(1.0)
    _, s_i, _, _ = r["out"]
    shrunk = r["out"][0]
    nrm = shrunk[s_i, 4:7]
    assert (nrm == np.array(S.COS_PASS_SRC, F32)).all(1).sum() == 4
    assert (nrm == np.array(S.COS_FAIL_SRC, F32)).all(1).sum() == 0
    assert rec["result"]["code"] == -2 and rec["result"]["iters"] == 2


def test_keep_mode_second_targets_take_over_in_iteration_three(probed):
    rec = probed("keep_mode")
    assert rec["result"]["iters"] == 20
    n = S.KEEP_N
    j2, j3 = rec[(2, S.R)]["nn"][0][-n:], rec[(3, S.R)]["nn"][0][-n:]
    changed = np.flatnonzero(j2 != j3)
    assert len(changed) >= S.KEEP_N // 2
    # the new match is a second target (appended after the first ones), KEEP_EPS closer than the first
    assert (j3[changed] > j2[changed]).all()
    # and every later iteration still matches: correspondences in all 20 iterations
    assert (rec["trace"]["n_corr"][:, S.R] > 0).all()


def test_bound_faces_are_exact(probed):
    rec = probed("bound_faces")
    p = S.bound_faces()
    moved = fl.rigid(p["src"][S.G][-len(p["face_points"]):], p["init_guess"])
    np.testing.assert_array_equal(moved[:, 0:3], p["face_points"])  # the initial guess puts them exactly on the faces
    lo, hi = p["faces"]
    inside = ((p["face_points"][:, :2].astype(F64) > lo) & (p["face_points"][:, :2].astype(F64) < hi)).all(1)
    assert inside.sum() == len(inside) // 2  # one float step inside: in; on a face: out
    for c in (S.G, S.PL, S.F):
        seen = {tuple(x) for x in rec[(0, c)]["src"][:, 0:3]}
        got = np.array([tuple(x) in seen for x in p["face_points"]])
        np.testing.assert_array_equal(got, inside)
    assert rec["result"]["code"] == 1 and rec["result"]["iters"] >= 4


def test_deep_grid_class_is_wider_than_the_morton_range(probed):
    rec = probed("deep_grid")
    tgt = rec[(0, S.F)]["tgt"]
    assert np.ptp(tgt[:, 0]) > 4096 * 0.125 * 2  # the finest cell doubles at least twice
    assert rec["result"]["code"] == 1 and rec["result"]["iters"] >= 4
