"""Host-side mirror of the reference's registration interface over the C-ABI.

`CRegistration.mm_lls_icp` has the argument list, defaults, outputs and return codes of
lo::CRegistration<PointT>::mm_lls_icp (include/common/cregistration.hpp:1114-1123, :1131-1136,
:1405, :1418-1420); `CloudBlock` / `Constraint` carry the members of cloudblock_t / constraint_t
that the function touches (include/common/utility.hpp:233-553, :561-590). Clouds are (n,7)
[x y z nx ny nz intensity] or (n,12) pcl::PointXYZINormal-row float32 arrays.

Everything here runs on the GPU through libmulls_b200.so; there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import abi

_FEATURES = ("ground", "pillar", "facade", "beam", "roof", "vertex")  # used_feature_type order


def _empty() -> np.ndarray:
    return np.zeros((0, 12), dtype=np.float32)


@dataclass
class CloudBlock:
    """cloudblock_t: per feature class a dense cloud (pc_*) and a down-sampled one (pc_*_down)."""

    pc_ground: np.ndarray = field(default_factory=_empty)
    pc_pillar: np.ndarray = field(default_factory=_empty)
    pc_facade: np.ndarray = field(default_factory=_empty)
    pc_beam: np.ndarray = field(default_factory=_empty)
    pc_roof: np.ndarray = field(default_factory=_empty)
    pc_vertex: np.ndarray = field(default_factory=_empty)
    pc_ground_down: np.ndarray = field(default_factory=_empty)
    pc_pillar_down: np.ndarray = field(default_factory=_empty)
    pc_facade_down: np.ndarray = field(default_factory=_empty)
    pc_beam_down: np.ndarray = field(default_factory=_empty)
    pc_roof_down: np.ndarray = field(default_factory=_empty)
    # bounds_t local_bound: min_x min_y min_z max_x max_y max_z (utility.hpp:101-136)
    local_bound: tuple = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0)
    # centerpoint_t local_station (utility.hpp:92-99): the scanner position, pivot of the 4-DoF global search
    local_station: tuple = (0.0, 0.0, 0.0)
    # pc_down: the down-sampled cloud the baseline registrations (omp_ndt) work on
    pc_down: np.ndarray = field(default_factory=_empty)

    def clone_feature(self, get_feature_down: bool):
        """cloudblock_t::clone_feature (utility.hpp:524-550): the six clouds mm_lls_icp works on."""
        if get_feature_down:
            src = (self.pc_ground_down, self.pc_pillar_down, self.pc_facade_down, self.pc_beam_down,
                   self.pc_roof_down, self.pc_vertex)
        else:
            src = (self.pc_ground, self.pc_pillar, self.pc_facade, self.pc_beam, self.pc_roof, self.pc_vertex)
        return [abi.as_aos48(c) for c in src]

    @staticmethod
    def from_class_list(clouds, down=None, local_bound=None) -> "CloudBlock":
        """clouds/down: six arrays in used_feature_type order (ground, pillar, facade, beam, roof, vertex)."""
        b = CloudBlock()
        for name, arr in zip(_FEATURES, clouds):
            setattr(b, f"pc_{name}", abi.as_aos48(arr))
        for name, arr in zip(_FEATURES[:5], (down if down is not None else clouds)[:5]):
            setattr(b, f"pc_{name}_down", abi.as_aos48(arr))
        if local_bound is None:
            pts = [abi.as_aos48(c)[:, :3] for c in clouds if len(c)]
            if pts:
                allp = np.concatenate(pts, axis=0).astype(np.float64)
                local_bound = tuple(allp.min(0)) + tuple(allp.max(0))
            else:
                local_bound = (0.0,) * 6
        b.local_bound = tuple(float(v) for v in local_bound)
        return b


@dataclass
class Constraint:
    """constraint_t: block1 = target, block2 = source; outputs of mm_lls_icp."""

    block1: CloudBlock = field(default_factory=CloudBlock)
    block2: CloudBlock = field(default_factory=CloudBlock)
    Trans1_2: np.ndarray = field(default_factory=lambda: np.eye(4))
    information_matrix: np.ndarray = field(default_factory=lambda: np.eye(6))
    sigma: float = float(np.finfo(np.float32).max)
    confidence: float = 0.0


def _xyz_rows(c):
    """(n, 3) xyz rows are accepted too where only positions are read (NDT)"""
    c = np.asarray(c, np.float32)
    if c.ndim == 2 and c.shape[1] == 3:
        c = np.concatenate([c, np.zeros((len(c), 9), np.float32)], axis=1)
    return abi.as_aos48(c)


def _ndt_out(res, tr, first, trace_cap):
    """the dict omp_ndt returns, from a mulls_ndt_result and its trace rows tr[first:first + trace_cap]"""
    out = dict(code=res.code, trans=np.array(res.trans[:], np.float64).reshape(4, 4), iterations=res.iterations,
               converged=bool(res.converged), fitness=res.fitness, n_target=res.n_target, n_source=res.n_source)
    if trace_cap > 0:
        k = min(res.iterations, int(trace_cap))
        rows = [tr[first + i] for i in range(k)]
        out["trace"] = dict(p=np.array([r.p[:] for r in rows], np.float64).reshape(k, 6),
                            step=np.array([r.step for r in rows], np.float64),
                            score=np.array([r.score for r in rows], np.float64),
                            reversed=np.array([r.reversed for r in rows], np.int32))
    return out



def _gicp_pcl_trace(tr, k):
    """the first k rows of a mulls_gicp_pcl_iter array as numpy arrays"""
    return dict(x=np.array([tr[i].x[:] for i in range(k)], np.float64).reshape(k, 6),
                delta=np.array([tr[i].delta for i in range(k)], np.float64),
                n_corr=np.array([tr[i].n_corr for i in range(k)], np.int32),
                inner_iterations=np.array([tr[i].inner_iterations for i in range(k)], np.int32),
                status=np.array([tr[i].status for i in range(k)], np.int32),
                evaluations=np.array([tr[i].evaluations for i in range(k)], np.int32))

class Context:
    """Thin RAII wrapper of a mulls_ctx (one CUDA device, one stream)."""

    def __init__(self, device: int = 0, max_pairs: int = 1, max_src_pts: int = 150000, max_tgt_pts: int = 150000):
        self.lib = abi.load_library()
        self.handle = self.lib.mulls_create(device, max_pairs, max_src_pts, max_tgt_pts)
        if not self.handle:
            raise RuntimeError(self.lib.mulls_last_error(None).decode())
        self.max_pairs = max_pairs
        self._keep = None
        self._n = 0

    def close(self):
        if getattr(self, "handle", None):
            self.lib.mulls_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != 0:
            raise RuntimeError(f"mulls_b200 error {rc}: {self.lib.mulls_last_error(self.handle).decode()}")

    def set_tunable(self, name: str, value: int):
        self._check(self.lib.mulls_set_tunable(self.handle, name.encode(), int(value)))

    @staticmethod
    def _pack(pairs):
        n = len(pairs)
        tv = (abi.CloudView * (6 * n))()
        sv = (abi.CloudView * (6 * n))()
        pa = (abi.IcpParams * n)()
        init = np.zeros((n, 16), dtype=np.float64)
        keep = []
        for i, pr in enumerate(pairs):
            for c in range(6):
                t = abi.as_aos48(pr["tgt"][c])
                s = abi.as_aos48(pr["src"][c])
                keep += [t, s]
                tv[6 * i + c] = abi.cloud_view(t)
                sv[6 * i + c] = abi.cloud_view(s)
            pa[i] = pr["params"]
            init[i] = np.asarray(pr["init_guess"], dtype=np.float64).reshape(16)
        return tv, sv, pa, init, keep

    def upload(self, pairs):
        """pairs: list of dict(tgt=[6 arrays], src=[6 arrays], params=IcpParams, init_guess=4x4)."""
        tv, sv, pa, init, keep = self._pack(pairs)
        self._keep = (tv, sv, pa, init, keep)
        self._n = len(pairs)
        self._check(self.lib.mulls_batch_upload(self.handle, len(pairs), tv, sv, pa,
                                                init.ctypes.data_as(C.POINTER(C.c_double))))

    def run_resident(self, want_trace: bool = False):
        n = self._n
        res = (abi.IcpResult * max(n, 1))()
        tr = (abi.IcpTrace * max(n, 1))() if want_trace else None
        self._check(self.lib.mulls_batch_run_resident(self.handle, res, tr))
        res, tr = res[:n], (tr[:n] if tr is not None else None)
        out = [abi.result_to_dict(r) for r in res]
        return (out, [abi.trace_to_dict(t) for t in tr]) if want_trace else (out, None)

    def run_batch(self, pairs, want_trace: bool = False):
        """Host buffers in, results out: H2D + ingest + iterations + D2H in one call."""
        tv, sv, pa, init, keep = self._pack(pairs)
        n = len(pairs)
        res = (abi.IcpResult * n)()
        tr = (abi.IcpTrace * n)() if want_trace else None
        self._check(self.lib.mulls_icp_run_batch(self.handle, n, tv, sv, pa,
                                                 init.ctypes.data_as(C.POINTER(C.c_double)), res, tr))
        out = [abi.result_to_dict(r) for r in res]
        return (out, [abi.trace_to_dict(t) for t in tr]) if want_trace else (out, None)

    def run_sharded(self, pair, src_index_base, src_global_n, allreduce, want_trace: bool = False):
        """mulls_icp_run_sharded: `pair["src"]` holds this rank's contiguous slice of every source class
        (global start index src_index_base[c] of src_global_n[c] points); `allreduce(ptr, count, dtype, op,
        stream) -> int` performs the in-place all-reduce on a device buffer (dtype 0 = f64, 1 = i32; op 0 = sum,
        1 = min), e.g. mulls_b200.dist.torch_allreduce()."""
        tv, sv, pa, init, keep = self._pack([pair])
        base = (C.c_uint32 * 6)(*[int(v) for v in src_index_base])
        glob = (C.c_uint32 * 6)(*[int(v) for v in src_global_n])
        res = abi.IcpResult()
        tr = abi.IcpTrace() if want_trace else None

        def _cb(user, ptr, count, dtype, op, stream):
            try:
                return int(allreduce(ptr, count, dtype, op, stream))
            except Exception as exc:  # surface Python errors as a communication failure
                print("all-reduce callback raised:", exc)
                return 1

        cb = abi.ALLREDUCE_FN(_cb)
        self._check(self.lib.mulls_icp_run_sharded(self.handle, tv, sv, base, glob, pa, init.ctypes.data_as(
            C.POINTER(C.c_double)), cb, None, C.byref(res), C.byref(tr) if tr is not None else None))
        return abi.result_to_dict(res), (abi.trace_to_dict(tr) if tr is not None else None)

    def nccl_init(self, rank: int, world: int, unique_id: bytes):
        """mulls_nccl_init: collective; `unique_id` = the 128 bytes rank 0 got from mulls_b200.dist.nccl_unique_id()."""
        self._check(self.lib.mulls_nccl_init(self.handle, int(rank), int(world), C.c_char_p(bytes(unique_id))))

    def run_sharded_nccl(self, pair, src_index_base, src_global_n, want_trace: bool = False):
        """mulls_icp_run_sharded_nccl on the context's own communicator (nccl_init): the per-iteration exchanges are
        ncclAllReduce calls inside the library — nothing interpreted in the loop."""
        tv, sv, pa, init, keep = self._pack([pair])
        base = (C.c_uint32 * 6)(*[int(v) for v in src_index_base])
        glob = (C.c_uint32 * 6)(*[int(v) for v in src_global_n])
        res = abi.IcpResult()
        tr = abi.IcpTrace() if want_trace else None
        self._check(self.lib.mulls_icp_run_sharded_nccl(self.handle, None, tv, sv, base, glob, pa,
                                                        init.ctypes.data_as(C.POINTER(C.c_double)), C.byref(res),
                                                        C.byref(tr) if tr is not None else None))
        return abi.result_to_dict(res), (abi.trace_to_dict(tr) if tr is not None else None)

    def nn_query(self, cls: int, xyz: np.ndarray):
        """mulls_nn_query: what block1->tree_*->nearestKSearch(point, 1) answers in the reference, on the sorted target
        slices the last registration left in HBM. Returns (index into the caller's class cloud or -1, squared distance)."""
        q = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        idx = np.empty(len(q), np.int32)
        d2 = np.empty(len(q), np.float32)
        self._check(self.lib.mulls_nn_query(self.handle, int(cls), q.ctypes.data_as(C.POINTER(C.c_float)), len(q),
                                            idx.ctypes.data_as(C.POINTER(C.c_int32)), d2.ctypes.data_as(C.POINTER(C.c_float))))
        return idx, d2

    def pca_features(self, cloud: np.ndarray, radius: float, k: int, stride: int = 1, unit_dist=None) -> dict:
        """PrincipleComponentAnalysis::get_pc_pca_feature (pca.hpp:294-354) on the GPU. With `unit_dist`,
        distance_adaptive_on = true: points farther than unit_dist from the origin search sqrt(dist / unit_dist) * radius."""
        c = abi.as_aos48(cloud)
        n = c.shape[0]
        ev = np.zeros((n, 3), np.float32)
        pr = np.zeros((n, 3), np.float32)
        nr = np.zeros((n, 3), np.float32)
        cnt = np.zeros(n, np.int32)
        out = abi.PcaOut(ev.ctypes.data_as(C.POINTER(C.c_float)), pr.ctypes.data_as(C.POINTER(C.c_float)),
                         nr.ctypes.data_as(C.POINTER(C.c_float)), cnt.ctypes.data_as(C.POINTER(C.c_int32)))
        if unit_dist is None:
            rc = self.lib.mulls_pca_features(self.handle, abi.cloud_view(c), float(radius), int(k), int(stride), C.byref(out))
        else:
            rc = self.lib.mulls_pca_features_adaptive(self.handle, abi.cloud_view(c), float(radius), int(k), int(stride),
                                                      float(unit_dist), C.byref(out))
        self._check(rc)
        return {"eigenvalues": ev, "principal": pr, "normal": nr, "pt_num": cnt}

    def classify_nground(self, cloud_in: np.ndarray, params: abi.ClassifyParams) -> dict:
        """CFilter::classify_nground_pts (cfilter.hpp:2058-2290) on the GPU: {"pillar": (n,12) rows, "beam", "facade",
        "roof", "pillar_down", ..., "vertex" (the new keypoints), "unground" (cloud_in as the call leaves it)}."""
        res = abi.classify_call(self.lib.mulls_classify_nground, self.handle, cloud_in, params)
        if "rc" in res:
            self._check(res["rc"])
        return res

    def fast_ground_filter(self, cloud_in: np.ndarray, params: abi.GroundParams) -> dict:
        """CFilter::fast_ground_filter (cfilter.hpp:1658-2036) on the GPU: {"ground", "ground_down", "unground"} rows."""
        res = abi.ground_call(self.lib.mulls_fast_ground_filter, self.handle, cloud_in, params)
        if "rc" in res:
            self._check(res["rc"])
        return res

    def voxel_downsample(self, cloud_in: np.ndarray, voxel_size: float) -> np.ndarray:
        """CFilter::voxel_downsample (cfilter.hpp:83-165) on the GPU: one row per occupied voxel, voxel-index order."""
        cloud = abi.as_aos48(cloud_in)
        out = np.zeros((max(len(cloud), 1), 12), np.float32)
        n = C.c_size_t(0)
        self._check(self.lib.mulls_voxel_downsample(self.handle, abi.cloud_view(cloud), float(voxel_size),
                                                    out.ctypes.data_as(C.POINTER(C.c_float)), len(out), C.byref(n)))
        return np.ascontiguousarray(out[: n.value])

    def extract_semantic_pts(self, pc_raw: np.ndarray, vf_downsample_resolution: float, ground: abi.GroundParams,
                             classify: abi.ClassifyParams) -> dict:
        """CFilter::extract_semantic_pts (cfilter.hpp:2295-2413) on the GPU, stages chained in HBM: {"down", "ground",
        "ground_down", "pillar", ..., "vertex", "unground"} as (n,12) rows."""
        raw = abi.as_aos48(pc_raw)
        n = max(len(raw), 1)
        fp = C.POINTER(C.c_float)
        bufs = {k: np.zeros((n, 12), np.float32) for k in ("down", "ground", "ground_down")}
        cbufs = [np.zeros((n, 12), np.float32) for _ in range(abi.OUT_COUNT)]
        P = abi.ExtractParams(float(vf_downsample_resolution), ground, classify)
        out = abi.ExtractOut()
        out.pc_down, out.pc_ground = bufs["down"].ctypes.data_as(fp), bufs["ground"].ctypes.data_as(fp)
        out.pc_ground_down = bufs["ground_down"].ctypes.data_as(fp)
        out.cap = n
        for k in range(abi.OUT_COUNT):
            out.cls.rows[k] = cbufs[k].ctypes.data_as(fp)
        out.cls.cap = n
        self._check(self.lib.mulls_extract_semantic_pts(self.handle, abi.cloud_view(raw), C.byref(P), C.byref(out)))
        res = {"down": bufs["down"][: out.n_down].copy(), "ground": bufs["ground"][: out.n_ground].copy(),
               "ground_down": bufs["ground_down"][: out.n_ground_down].copy()}
        for k in range(abi.OUT_COUNT):
            res[abi.OUT_NAMES[k]] = np.ascontiguousarray(cbufs[k][: out.cls.n[k]])
        return res

    def sor_filter(self, cloud: np.ndarray, mean_k: int, n_std: float):
        """CFilter::sor_filter (cfilter.hpp:203-247, pcl::StatisticalOutlierRemoval) on the GPU. Returns (keep: bool[n],
        the kept points being cloud[keep]; mean_dist: float32[n], 0 for non-finite points; stats: dict of mean, stddev,
        threshold, n_valid, n_kept)."""
        c = abi.as_aos48(cloud)
        n = c.shape[0]
        bits = np.zeros(max((n + 7) // 8, 1), np.uint8)
        dist = np.zeros(max(n, 1), np.float32)
        st = abi.SorStats()
        self._check(self.lib.mulls_sor_filter(self.handle, abi.cloud_view(c), int(mean_k), float(n_std),
                                              bits.ctypes.data_as(C.POINTER(C.c_uint8)),
                                              dist.ctypes.data_as(C.POINTER(C.c_float)), C.byref(st)))
        keep = np.unpackbits(bits, bitorder="little")[:n].astype(bool)
        return keep, dist[:n], {k: getattr(st, k) for k, _ in abi.SorStats._fields_}

    def vertical_intrinsic_calibration(self, cloud: np.ndarray, var_vertical_ang_d: float, inverse_z: bool = False):
        """CFilter::vertical_intrinsic_calibration (cfilter.hpp:250-291) on the GPU. Returns (xyz: float32[n, 3], the
        member's return value)."""
        c = abi.as_aos48(cloud)
        xyz = np.zeros((max(len(c), 1), 3), np.float32)
        applied = C.c_int(0)
        self._check(self.lib.mulls_vertical_intrinsic_calibration(self.handle, abi.cloud_view(c), float(var_vertical_ang_d),
                                                                  int(bool(inverse_z)), xyz.ctypes.data_as(C.POINTER(C.c_float)),
                                                                  C.byref(applied)))
        return xyz[: len(c)], bool(applied.value)

    def timestamp_ratio(self, cloud: np.ndarray, timestamp_available: bool = True, scan_begin_ang_deg: float = 180.0,
                        scan_duration_ms: float = 100.0) -> np.ndarray:
        """CFilter::get_pts_timestamp_ratio_in_frame (cfilter.hpp:412-467) on the GPU: the new curvature column, float32[n]."""
        c = abi.as_aos48(cloud)
        ratio = np.zeros(max(len(c), 1), np.float32)
        self._check(self.lib.mulls_timestamp_ratio(self.handle, abi.cloud_view(c), int(bool(timestamp_available)),
                                                   float(scan_begin_ang_deg), float(scan_duration_ms),
                                                   ratio.ctypes.data_as(C.POINTER(C.c_float))))
        return ratio[: len(c)]

    def motion_compensation(self, clouds, T, s_ambiguous_thre: float = 0.0):
        """CFilter::apply_motion_compensation (cfilter.hpp:470-516) on the GPU for 1..6 clouds in one call (as
        batch_apply_motion_compensation :519-549). `clouds`: one (n, 12) array or a list of them; T: 4x4. Returns the new
        xyz (float32[n, 3]) of each cloud, in the same form."""
        single = isinstance(clouds, np.ndarray)
        cl = [abi.as_aos48(c) for c in ([clouds] if single else clouds)]
        views = (abi.CloudView * max(len(cl), 1))(*[abi.cloud_view(c) for c in cl])
        outs = [np.zeros((max(len(c), 1), 3), np.float32) for c in cl]
        fp = C.POINTER(C.c_float)
        ptrs = (fp * max(len(cl), 1))(*[o.ctypes.data_as(fp) for o in outs])
        Td = np.ascontiguousarray(np.asarray(T, np.float64).reshape(16))
        self._check(self.lib.mulls_motion_compensation(self.handle, views, len(cl), Td.ctypes.data_as(C.POINTER(C.c_double)),
                                                       float(s_ambiguous_thre), ptrs))
        res = [o[: len(c)] for o, c in zip(outs, cl)]
        return res[0] if single else res

    def ncc_correspondences(self, target_kpts: np.ndarray, source_kpts: np.ndarray, fixed_num_corr: bool = False,
                            corr_num: int = 2000, reciprocal_on: bool = True):
        """CRegistration::find_feature_correspondence_ncc (cregistration.hpp:409-601) on the GPU, as index pairs: returns
        None where the reference returns false (fewer than 10 keypoints in a cloud), else (tgt_idx, src_idx), int32 arrays
        of the rows the reference appends to target_corrs / source_corrs, in its order. The resident batch is untouched."""
        t, s = abi.as_aos48(target_kpts), abi.as_aos48(source_kpts)
        cap = 7 * min(len(t), len(s)) if fixed_num_corr else len(t)  # at most 7 pairs per keypoint / one per target row
        ti = np.zeros(max(cap, 1), np.int32)
        si = np.zeros(max(cap, 1), np.int32)
        n = C.c_size_t(0)
        performed = C.c_int(0)
        ip = C.POINTER(C.c_int32)
        self._check(self.lib.mulls_ncc_correspondences(self.handle, abi.cloud_view(t), abi.cloud_view(s), int(bool(fixed_num_corr)),
                                                       int(corr_num), int(bool(reciprocal_on)), ti.ctypes.data_as(ip),
                                                       si.ctypes.data_as(ip), cap, C.byref(n), C.byref(performed)))
        if not performed.value:
            return None
        return ti[: n.value].copy(), si[: n.value].copy()

    def coarse_reg_ransac(self, target_pts: np.ndarray, source_pts: np.ndarray, noise_bound: float = 0.2,
                          min_inlier_num: int = 8, max_iter_num: int = 20000, tran_mat=None):
        """CRegistration::coarse_reg_ransac (cregistration.hpp:604-661) on the GPU over the correspondences i <-> i,
        i < len(target_pts). Returns (status, tran_mat, n_inliers, n_hypotheses): status 1 (reliable), 0 (need check) or
        -1 (failed); tran_mat is a (4, 4) float64 copy of the given one (identity when None), replaced by the estimate
        when status >= 0. The resident batch is untouched."""
        t, s = abi.as_aos48(target_pts), abi.as_aos48(source_pts)
        T = np.array(np.eye(4) if tran_mat is None else tran_mat, np.float64).reshape(4, 4).copy()
        buf = np.ascontiguousarray(T.ravel())
        st, ni, nh = C.c_int(0), C.c_int(0), C.c_int(0)
        self._check(self.lib.mulls_coarse_reg_ransac(self.handle, abi.cloud_view(t), abi.cloud_view(s), float(noise_bound),
                                                     int(min_inlier_num), int(max_iter_num),
                                                     buf.ctypes.data_as(C.POINTER(C.c_double)), C.byref(st), C.byref(ni),
                                                     C.byref(nh)))
        return st.value, buf.reshape(4, 4), ni.value, nh.value

    def coarse_reg_teaser(self, target_pts: np.ndarray, source_pts: np.ndarray, noise_bound: float = 0.2,
                          min_inlier_num: int = 8, tran_mat=None):
        """CRegistration::coarse_reg_teaser (cregistration.hpp:664-759) on the GPU over the correspondences i <-> i.
        Returns (status, tran_mat, info): status 1 (reliable), 0 (need check) or -1 (failed); tran_mat is a (4, 4)
        float64 copy of the given one (identity when None), replaced by the estimate when status >= 0; info a dict of
        mulls_teaser_info (n_edges, max_core, clique_size, rotation_inliers, gnc_iterations, search_launches). The
        resident batch is untouched."""
        t, s = abi.as_aos48(target_pts), abi.as_aos48(source_pts)
        T = np.array(np.eye(4) if tran_mat is None else tran_mat, np.float64).reshape(4, 4).copy()
        buf = np.ascontiguousarray(T.ravel())
        st, info = C.c_int(0), abi.TeaserInfo()
        self._check(self.lib.mulls_coarse_reg_teaser(self.handle, abi.cloud_view(t), abi.cloud_view(s), float(noise_bound),
                                                     int(min_inlier_num), buf.ctypes.data_as(C.POINTER(C.c_double)),
                                                     C.byref(st), C.byref(info)))
        return st.value, buf.reshape(4, 4), {k: getattr(info, k) for k, _ in abi.TeaserInfo._fields_ if k != "pad"}

    def omp_ndt(self, target: np.ndarray, source: np.ndarray, target_bound, source_bound, ndt_resolution: float = 1.0,
                use_direct_search: bool = True, initial_guess=None, apply_intersection_filter: bool = True,
                fitness_score_thre: float = 10.0, trace_cap: int = 0):
        """CRegistration::omp_ndt (cregistration.hpp:945-1021, DIRECT7) on the GPU: target / source are block1 / block2
        ->pc_down ((n, 3), (n, 7) or (n, 12) rows), the bounds their local_bound (min_x min_y min_z max_x max_y max_z). Returns a dict: code (1, or -3 when
        the fitness exceeds fitness_score_thre), trans (Trans1_2, (4, 4) float64), iterations, converged, fitness,
        n_target / n_source after the intersection filter, and with trace_cap > 0 `trace`: per iteration the pose vector
        p (6), the step length, the score and whether the direction was reversed. use_direct_search=False (KDTREE) raises:
        omp_ndt_kdtree runs that mode. Replaces the resident batch."""
        t, s = _xyz_rows(target), _xyz_rows(source)
        g = np.ascontiguousarray(np.eye(4) if initial_guess is None else initial_guess, np.float64).reshape(16).copy()
        tb = np.ascontiguousarray(target_bound, np.float64).reshape(6).copy()
        sb = np.ascontiguousarray(source_bound, np.float64).reshape(6).copy()
        res = abi.NdtResult()
        tr = (abi.NdtIter * max(int(trace_cap), 1))()
        dp = C.POINTER(C.c_double)
        self._check(self.lib.mulls_omp_ndt(self.handle, abi.cloud_view(t), abi.cloud_view(s), float(ndt_resolution),
                                           int(bool(use_direct_search)), g.ctypes.data_as(dp), int(bool(apply_intersection_filter)),
                                           float(fitness_score_thre), tb.ctypes.data_as(dp), sb.ctypes.data_as(dp), C.byref(res),
                                           tr, int(trace_cap)))
        return _ndt_out(res, tr, 0, trace_cap)

    def omp_ndt_kdtree(self, target: np.ndarray, source: np.ndarray, target_bound, source_bound, ndt_resolution: float = 1.0,
                       initial_guess=None, apply_intersection_filter: bool = True, fitness_score_thre: float = 10.0,
                       trace_cap: int = 0):
        """CRegistration::omp_ndt with use_direct_search=False (KDTREE, mulls_omp_ndt_kdtree) on the GPU: every leaf
        centroid within ndt_resolution of a moved source point is its neighbour, as PCL's radius search finds them.
        omp_ndt's arguments without use_direct_search; returns the dict omp_ndt returns. Replaces the resident batch."""
        t, s = _xyz_rows(target), _xyz_rows(source)
        g = np.ascontiguousarray(np.eye(4) if initial_guess is None else initial_guess, np.float64).reshape(16).copy()
        tb = np.ascontiguousarray(target_bound, np.float64).reshape(6).copy()
        sb = np.ascontiguousarray(source_bound, np.float64).reshape(6).copy()
        res = abi.NdtResult()
        tr = (abi.NdtIter * max(int(trace_cap), 1))()
        dp = C.POINTER(C.c_double)
        self._check(self.lib.mulls_omp_ndt_kdtree(self.handle, abi.cloud_view(t), abi.cloud_view(s), float(ndt_resolution),
                                                  g.ctypes.data_as(dp), int(bool(apply_intersection_filter)),
                                                  float(fitness_score_thre), tb.ctypes.data_as(dp), sb.ctypes.data_as(dp),
                                                  C.byref(res), tr, int(trace_cap)))
        return _ndt_out(res, tr, 0, trace_cap)

    def omp_ndt_batch(self, targets, sources, target_bounds, source_bounds, ndt_resolution: float = 1.0,
                      use_direct_search: bool = True, initial_guesses=None, apply_intersection_filter: bool = True,
                      fitness_score_thre: float = 10.0, trace_cap: int = 0):
        """omp_ndt for P pairs in one call (mulls_omp_ndt_batch): targets / sources / target_bounds / source_bounds are
        sequences of P clouds and bounds, initial_guesses None or P (4, 4) matrices; the other parameters are shared.
        Returns one dict per pair, equal bit for bit to what omp_ndt returns for that pair alone. Needs a context made
        for at least P pairs. Replaces the resident batch."""
        ts, ss = [_xyz_rows(t) for t in targets], [_xyz_rows(s) for s in sources]
        n = len(ts)
        if len(ss) != n or len(target_bounds) != n or len(source_bounds) != n or (initial_guesses is not None and len(initial_guesses) != n):
            raise ValueError("omp_ndt_batch: targets, sources, bounds and initial guesses must have one entry per pair")
        g = np.ascontiguousarray([np.eye(4)] * n if initial_guesses is None else initial_guesses, np.float64).reshape(16 * n).copy()
        tb = np.ascontiguousarray(target_bounds, np.float64).reshape(6 * n).copy()
        sb = np.ascontiguousarray(source_bounds, np.float64).reshape(6 * n).copy()
        tv = (abi.CloudView * max(n, 1))(*[abi.cloud_view(t) for t in ts])
        sv = (abi.CloudView * max(n, 1))(*[abi.cloud_view(s) for s in ss])
        res = (abi.NdtResult * max(n, 1))()
        cap = int(trace_cap)
        tr = (abi.NdtIter * max(n * cap, 1))()
        dp = C.POINTER(C.c_double)
        self._check(self.lib.mulls_omp_ndt_batch(self.handle, n, tv, sv, float(ndt_resolution), int(bool(use_direct_search)),
                                                 g.ctypes.data_as(dp), int(bool(apply_intersection_filter)),
                                                 float(fitness_score_thre), tb.ctypes.data_as(dp), sb.ctypes.data_as(dp), res,
                                                 tr, cap))
        return [_ndt_out(res[i], tr, i * cap, cap) for i in range(n)]

    def omp_gicp(self, target: np.ndarray, source: np.ndarray, target_bound, source_bound, max_iter_num: int = 20,
                 dis_thre_unit: float = 1.5, using_voxel_gicp: bool = True, voxel_size: float = 1.0, initial_guess=None,
                 apply_intersection_filter: bool = False, fitness_score_thre: float = 10.0, trace_cap: int = 0):
        """CRegistration::omp_gicp (cregistration.hpp:1024-1098, FastVGICP) on the GPU: target / source are block1 /
        block2 ->pc_down ((n, 3), (n, 7) or (n, 12) rows), the bounds their local_bound. max_iter_num and dis_thre_unit
        are accepted and ignored, as the reference ignores them. The walk draws from the process's rand() where the
        reference does. Returns a dict: code (1, or -3 when the fitness exceeds fitness_score_thre), trans (Trans1_2,
        (4, 4) float64), iterations, converged, fitness, n_target / n_source after the prologue, x0 (the start point),
        and with trace_cap > 0 `trace`: per step the point x (6), the step delta (6), the correspondence count and
        whether the step was the random fallback. using_voxel_gicp=False raises. Replaces the resident batch."""
        del max_iter_num, dis_thre_unit  # not read by FastVGICP

        def aos48(c):  # (n, 3) xyz rows are accepted too: GICP reads positions only
            c = np.asarray(c, np.float32)
            if c.ndim == 2 and c.shape[1] == 3:
                c = np.concatenate([c, np.zeros((len(c), 9), np.float32)], axis=1)
            return abi.as_aos48(c)

        t, s = aos48(target), aos48(source)
        g = np.ascontiguousarray(np.eye(4) if initial_guess is None else initial_guess, np.float64).reshape(16).copy()
        tb = np.ascontiguousarray(target_bound, np.float64).reshape(6).copy()
        sb = np.ascontiguousarray(source_bound, np.float64).reshape(6).copy()
        res = abi.GicpResult()
        tr = (abi.GicpIter * max(int(trace_cap), 1))()
        dp = C.POINTER(C.c_double)
        self._check(self.lib.mulls_omp_gicp(self.handle, abi.cloud_view(t), abi.cloud_view(s), int(bool(using_voxel_gicp)),
                                            float(voxel_size), g.ctypes.data_as(dp), int(bool(apply_intersection_filter)),
                                            float(fitness_score_thre), tb.ctypes.data_as(dp), sb.ctypes.data_as(dp),
                                            C.byref(res), tr, int(trace_cap)))
        out = dict(code=res.code, trans=np.array(res.trans[:], np.float64).reshape(4, 4), iterations=res.iterations,
                   converged=bool(res.converged), fitness=res.fitness, n_target=res.n_target, n_source=res.n_source,
                   x0=np.array(res.x0[:], np.float32))
        if trace_cap > 0:
            k = min(res.iterations, int(trace_cap))
            out["trace"] = dict(x=np.array([tr[i].x[:] for i in range(k)], np.float32).reshape(k, 6),
                                delta=np.array([tr[i].delta[:] for i in range(k)], np.float32).reshape(k, 6),
                                n_corr=np.array([tr[i].n_corr for i in range(k)], np.int32),
                                random_step=np.array([tr[i].random_step for i in range(k)], np.int32))
        return out

    def omp_gicp_pcl(self, target: np.ndarray, source: np.ndarray, target_bound, source_bound, max_iter_num: int = 20,
                     dis_thre_unit: float = 1.5, initial_guess=None, apply_intersection_filter: bool = False,
                     fitness_score_thre: float = 10.0, trace_cap: int = 0):
        """CRegistration::omp_gicp with using_voxel_gicp=False (cregistration.hpp:1024-1098, point-wise GICP with PCL's
        BFGS) on the GPU: target / source are block1 / block2 ->pc_down ((n, 3), (n, 7) or (n, 12) rows), the bounds
        their local_bound. max_iter_num caps the BFGS steps of each outer iteration, as setMaximumOptimizerIterations
        does; dis_thre_unit is accepted and ignored, as the reference ignores it. Returns a dict: code (1, or -3 when
        the fitness exceeds fitness_score_thre), trans (Trans1_2, (4, 4) float64), iterations, converged, fitness,
        n_target / n_source after the prologue, and with trace_cap > 0 `trace`: per outer iteration the solver's state
        x (6: tx ty tz, X Y Z angles), delta, the correspondence count, the BFGS steps, the BFGS status and the functor
        calls. Replaces the resident batch."""
        del dis_thre_unit  # not read by GeneralizedIterativeClosestPoint

        def aos48(c):  # (n, 3) xyz rows are accepted too: GICP reads positions only
            c = np.asarray(c, np.float32)
            if c.ndim == 2 and c.shape[1] == 3:
                c = np.concatenate([c, np.zeros((len(c), 9), np.float32)], axis=1)
            return abi.as_aos48(c)

        t, s = aos48(target), aos48(source)
        g = np.ascontiguousarray(np.eye(4) if initial_guess is None else initial_guess, np.float64).reshape(16).copy()
        tb = np.ascontiguousarray(target_bound, np.float64).reshape(6).copy()
        sb = np.ascontiguousarray(source_bound, np.float64).reshape(6).copy()
        res = abi.GicpPclResult()
        tr = (abi.GicpPclIter * max(int(trace_cap), 1))()
        dp = C.POINTER(C.c_double)
        self._check(self.lib.mulls_omp_gicp_pcl(self.handle, abi.cloud_view(t), abi.cloud_view(s), int(max_iter_num),
                                                g.ctypes.data_as(dp), int(bool(apply_intersection_filter)),
                                                float(fitness_score_thre), tb.ctypes.data_as(dp), sb.ctypes.data_as(dp),
                                                C.byref(res), tr, int(trace_cap)))
        out = dict(code=res.code, trans=np.array(res.trans[:], np.float64).reshape(4, 4), iterations=res.iterations,
                   converged=bool(res.converged), fitness=res.fitness, n_target=res.n_target, n_source=res.n_source)
        if trace_cap > 0:
            out["trace"] = _gicp_pcl_trace(tr, min(res.iterations, int(trace_cap)))
        return out

    def non_max_suppress(self, cloud: np.ndarray, non_max_radius: float):
        """CFilter::non_max_suppress(cloud_in_out, non_max_radius) (cfilter.hpp:1183-1240) on the GPU. Returns
        (kept_idx, performed): kept_idx is an int32 array of the input rows the reference leaves in the cloud, in its
        order (cloud[kept_idx] is that cloud); performed is False, with kept_idx empty, where the reference returns false
        and leaves the cloud as it was (fewer than 10 points). The resident batch is untouched."""
        c = abi.as_aos48(cloud)
        idx = np.zeros(max(len(c), 1), np.int32)
        n = C.c_size_t(0)
        performed = C.c_int(0)
        self._check(self.lib.mulls_non_max_suppress(self.handle, abi.cloud_view(c), float(non_max_radius),
                                                    idx.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(n), C.byref(performed)))
        return idx[: n.value].copy(), bool(performed.value)

    def stats(self) -> dict:
        s = abi.RunStats()
        self._check(self.lib.mulls_get_stats(self.handle, C.byref(s)))
        d = {k: getattr(s, k) for k, _ in abi.RunStats._fields_}
        d["ms_search_iter"] = [float(v) for v in s.ms_search_iter]
        return d


class PipelinedContext:
    """N independent contexts (own CUDA stream each) on one device, driven from N host threads: while one
    slice of a batch is being registered, the next slice's clouds are already crossing PCIe, and small
    kernels of different slices fill each other's tails. Same results as one Context (pairs are independent)."""

    def __init__(self, device: int, n_lanes: int, max_pairs_per_lane: int, max_src_pts: int, max_tgt_pts: int):
        from concurrent.futures import ThreadPoolExecutor

        self.lanes = [Context(device, max_pairs_per_lane, max_src_pts, max_tgt_pts) for _ in range(n_lanes)]
        self.pool = ThreadPoolExecutor(n_lanes)
        self._slices = None

    def close(self):
        for c in self.lanes:
            c.close()
        self.pool.shutdown()

    def set_tunable(self, name: str, value: int):
        for c in self.lanes:
            c.set_tunable(name, value)

    def _split(self, pairs):
        n, k = len(pairs), len(self.lanes)
        bounds = [(n * i) // k for i in range(k + 1)]
        return [pairs[bounds[i]:bounds[i + 1]] for i in range(k)]

    @staticmethod
    def _join(futs, want_trace: bool):
        out, traces = [], []
        for f in futs:
            o, t = f.result()
            out += o
            traces += t or []
        return out, (traces if want_trace else None)

    def run_batch(self, pairs, want_trace: bool = False):
        """Host buffers in, results out; slices are uploaded and registered concurrently. Returns (results, traces)
        in the order of `pairs`, as Context.run_batch does."""
        parts = self._split(pairs)
        futs = [self.pool.submit(lambda c=c, p=p: c.run_batch(p, want_trace) if p else ([], None))
                for c, p in zip(self.lanes, parts)]
        return self._join(futs, want_trace)

    def upload(self, pairs):
        self._slices = self._split(pairs)
        for c, p in zip(self.lanes, self._slices):
            if p:
                c.upload(p)

    def run_resident(self, want_trace: bool = False):
        """One pass over the resident batch, the slices registered concurrently. Returns (results, traces) as
        Context.run_resident does."""
        futs = [self.pool.submit(lambda c=c, p=p: c.run_resident(want_trace) if p else ([], None))
                for c, p in zip(self.lanes, self._slices)]
        return self._join(futs, want_trace)

    def run_resident_steps(self, k: int):
        """k passes over the resident batch; every lane runs its k passes back to back (no per-step barrier
        between lanes). Returns (results of the last pass, per-lane summed kernel launches)."""

        def work(c, p):
            if not p:
                return [], 0
            launches, out = 0, []
            for _ in range(k):
                out = c.run_resident()[0]
                launches += c.stats()["kernel_launches"]
            return out, launches

        futs = [self.pool.submit(work, c, p) for c, p in zip(self.lanes, self._slices)]
        out, launches = [], 0
        for f in futs:
            o, n = f.result()
            out += o
            launches += n
        return out, launches

    def run_batch_steps(self, pairs, k: int):
        """k end-to-end passes (host buffers -> results) over `pairs`, lanes free-running as above."""
        parts = self._split(pairs)

        def work(c, p):
            out = []
            for _ in range(k):
                out = c.run_batch(p)[0] if p else []
            return out

        futs = [self.pool.submit(work, c, p) for c, p in zip(self.lanes, parts)]
        out = []
        for f in futs:
            out += f.result()
        return out

    def stats(self):
        return [c.stats() for c, p in zip(self.lanes, self._slices or [[]] * len(self.lanes)) if p]


def heading_trial_guesses(local_station, heading_step_d: float):
    """The initial guesses mm_lls_icp_4dof_global tries (cregistration.hpp:1607-1641): a rotation about z by
    heading_d = 0, step, 2*step, ... < 360 (accumulated in float as the reference does), about the source
    block's station. Returns (list of heading_d, list of 4x4)."""
    heads, mats = [], []
    heading_d = np.float32(0.0)
    step = np.float32(heading_step_d)
    sx, sy, sz = (float(v) for v in local_station)
    while float(heading_d) < 360.0:
        heading_rad = np.float32(float(heading_d) * np.pi / 180.0)
        rot = np.eye(4)
        rot[0, 0] = np.cos(float(heading_rad))
        rot[0, 1] = np.sin(float(heading_rad))
        rot[1, 0] = -np.sin(float(heading_rad))
        rot[1, 1] = np.cos(float(heading_rad))
        g2s, s2g = np.eye(4), np.eye(4)
        g2s[:3, 3] = (-sx, -sy, -sz)
        s2g[:3, 3] = (sx, sy, sz)
        mats.append(s2g @ rot @ g2s)
        heads.append(float(heading_d))
        heading_d = np.float32(heading_d + step)
    return heads, mats


class CRegistration:
    """lo::CRegistration<PointT> — the part of its public surface on the hot path."""

    def __init__(self, device: int = 0, max_src_pts: int = 700000, max_tgt_pts: int = 700000):
        self._device, self._max_src, self._max_tgt = device, max_src_pts, max_tgt_pts
        self._ctx = Context(device, 1, max_src_pts, max_tgt_pts)
        self._batch_ctx = None
        self.last_trace = None

    def find_feature_correspondence_ncc(self, target_kpts: np.ndarray, source_kpts: np.ndarray, target_corrs=None,
                                        source_corrs=None, fixed_num_corr: bool = False, corr_num: int = 2000,
                                        reciprocal_on: bool = True):
        """lo::CRegistration::find_feature_correspondence_ncc (cregistration.hpp:409-601): returns (ok, target_corrs,
        source_corrs). The matched keypoint rows are appended to the given (n, 12) clouds (empty when None), which come
        back unchanged when ok is False (fewer than 10 keypoints in a cloud)."""
        t, s = abi.as_aos48(target_kpts), abi.as_aos48(source_kpts)
        tc = _empty() if target_corrs is None else abi.as_aos48(target_corrs)
        sc = _empty() if source_corrs is None else abi.as_aos48(source_corrs)
        got = self._ctx.ncc_correspondences(t, s, fixed_num_corr, corr_num, reciprocal_on)
        if got is None:
            return False, tc, sc
        ti, si = got
        return True, np.concatenate([tc, t[ti]]), np.concatenate([sc, s[si]])

    def coarse_reg_ransac(self, target_pts: np.ndarray, source_pts: np.ndarray, tran_mat=None, noise_bound: float = 0.2,
                          min_inlier_num: int = 8, max_iter_num: int = 20000):
        """lo::CRegistration::coarse_reg_ransac (cregistration.hpp:604-661): returns (status, tran_mat). tran_mat is the
        given (4, 4) matrix (identity when None), replaced by the estimate when status >= 0 and left as it was on -1."""
        status, T, _, _ = self._ctx.coarse_reg_ransac(target_pts, source_pts, noise_bound, min_inlier_num, max_iter_num, tran_mat)
        return status, T

    def coarse_reg_teaser(self, target_pts: np.ndarray, source_pts: np.ndarray, tran_mat=None, noise_bound: float = 0.2,
                          min_inlier_num: int = 8):
        """lo::CRegistration::coarse_reg_teaser (cregistration.hpp:664-759): returns (status, tran_mat). tran_mat is the
        given (4, 4) matrix (identity when None), replaced by the estimate when status >= 0 and left as it was on -1."""
        status, T, _ = self._ctx.coarse_reg_teaser(target_pts, source_pts, noise_bound, min_inlier_num, tran_mat)
        return status, T

    def omp_ndt(self, target: np.ndarray, source: np.ndarray, target_bound, source_bound, ndt_resolution: float = 1.0,
                use_direct_search: bool = True, initial_guess=None, apply_intersection_filter: bool = True,
                fitness_score_thre: float = 10.0):
        """lo::CRegistration::omp_ndt (cregistration.hpp:945-1021): returns (code, Trans1_2) for block1 = target and
        block2 = source with their local_bounds. Only the DIRECT7 search (use_direct_search=True) runs here; omp_ndt_kdtree
        runs KDTREE."""
        r = self._ctx.omp_ndt(target, source, target_bound, source_bound, ndt_resolution, use_direct_search, initial_guess,
                              apply_intersection_filter, fitness_score_thre)
        return r["code"], r["trans"]

    def omp_ndt_kdtree(self, target: np.ndarray, source: np.ndarray, target_bound, source_bound, ndt_resolution: float = 1.0,
                       initial_guess=None, apply_intersection_filter: bool = True, fitness_score_thre: float = 10.0):
        """lo::CRegistration::omp_ndt with use_direct_search=False (KDTREE): returns (code, Trans1_2) for block1 = target
        and block2 = source with their local_bounds."""
        r = self._ctx.omp_ndt_kdtree(target, source, target_bound, source_bound, ndt_resolution, initial_guess,
                                     apply_intersection_filter, fitness_score_thre)
        return r["code"], r["trans"]

    def omp_ndt_batch(self, registration_cons, ndt_resolution: float = 1.0, use_direct_search: bool = True,
                      initial_guesses=None, apply_intersection_filter: bool = True, fitness_score_thre: float = 10.0):
        """omp_ndt for every Constraint of registration_cons in one call (block1 = target, block2 = source, their pc_down
        and local_bounds; initial_guesses None or one (4, 4) per constraint): each one's Trans1_2 is written as
        omp_ndt writes it. Returns the codes, one per constraint."""
        n = len(registration_cons)
        if self._batch_ctx is None or self._batch_ctx.max_pairs < n or self._batch_cap < (self._max_src, self._max_tgt):
            if self._batch_ctx is not None:
                self._batch_ctx.close()
            self._batch_ctx = Context(self._device, max(n, 1), self._max_src, self._max_tgt)
            self._batch_cap = (self._max_src, self._max_tgt)
        res = self._batch_ctx.omp_ndt_batch([c.block1.pc_down for c in registration_cons],
                                            [c.block2.pc_down for c in registration_cons],
                                            [c.block1.local_bound for c in registration_cons],
                                            [c.block2.local_bound for c in registration_cons], ndt_resolution,
                                            use_direct_search, initial_guesses, apply_intersection_filter, fitness_score_thre)
        for c, r in zip(registration_cons, res):
            c.Trans1_2 = r["trans"]
        return [r["code"] for r in res]

    def omp_gicp(self, target: np.ndarray, source: np.ndarray, target_bound, source_bound, max_iter_num: int = 20,
                 dis_thre_unit: float = 1.5, using_voxel_gicp: bool = True, voxel_size: float = 1.0, initial_guess=None,
                 apply_intersection_filter: bool = False, fitness_score_thre: float = 10.0):
        """lo::CRegistration::omp_gicp (cregistration.hpp:1024-1098): returns (code, Trans1_2) for block1 = target and
        block2 = source with their local_bounds. Only the voxelized GICP (using_voxel_gicp=True) runs here."""
        r = self._ctx.omp_gicp(target, source, target_bound, source_bound, max_iter_num, dis_thre_unit, using_voxel_gicp,
                               voxel_size, initial_guess, apply_intersection_filter, fitness_score_thre)
        return r["code"], r["trans"]

    def omp_gicp_pcl(self, target: np.ndarray, source: np.ndarray, target_bound, source_bound, max_iter_num: int = 20,
                     dis_thre_unit: float = 1.5, initial_guess=None, apply_intersection_filter: bool = False,
                     fitness_score_thre: float = 10.0):
        """lo::CRegistration::omp_gicp with using_voxel_gicp=False (cregistration.hpp:1024-1098): returns
        (code, Trans1_2) for block1 = target and block2 = source with their local_bounds."""
        r = self._ctx.omp_gicp_pcl(target, source, target_bound, source_bound, max_iter_num, dis_thre_unit, initial_guess,
                                   apply_intersection_filter, fitness_score_thre)
        return r["code"], r["trans"]

    def mm_lls_icp_4dof_global(self, registration_con: Constraint, heading_step_d: float, max_iter_num: int = 20,
                               dis_thre_unit: float = 1.5, converge_translation: float = 0.005,
                               converge_rotation_d: float = 0.05, dis_thre_min: float = 0.5,
                               dis_thre_update_rate: float = 1.05, max_bearable_rotation_d: float = 15.0) -> bool:
        """lo::CRegistration::mm_lls_icp_4dof_global (cregistration.hpp:1584-1681): try every heading and keep the
        registration with the best confidence / sigma. The reference runs the trials one after the other; here
        they are ONE batched call — the trials are independent registrations of the same clouds.
        As in the reference, converge_translation is also passed as converge_rotation_d (:1636-1637) and
        converge_rotation_d / max_bearable_rotation_d are not forwarded."""
        heads, mats = heading_trial_guesses(registration_con.block2.local_station, heading_step_d)
        p = abi.default_params()
        p.max_iter_num = max_iter_num
        p.dis_thre_unit = dis_thre_unit
        p.converge_translation = converge_translation
        p.converge_rotation_d = converge_translation
        p.dis_thre_min = dis_thre_min
        p.dis_thre_update_rate = dis_thre_update_rate
        p.used_feature_type = b"111110"
        p.weight_strategy = b"1001"
        p.target_bound[:] = list(registration_con.block1.local_bound)
        tgt = registration_con.block1.clone_feature(False)
        src = registration_con.block2.clone_feature(True)
        pairs = [{"tgt": tgt, "src": src, "params": p, "init_guess": m} for m in mats]
        ns, nt = sum(len(s) for s in src), sum(len(t) for t in tgt)
        if self._batch_ctx is None or self._batch_ctx.max_pairs < len(pairs) or self._batch_cap < (ns, nt):
            if self._batch_ctx is not None:
                self._batch_ctx.close()
            self._batch_ctx = Context(self._device, len(pairs), max(ns, 1), max(nt, 1))
            self._batch_cap = (ns, nt)
        res, _ = self._batch_ctx.run_batch(pairs)
        best_score, ok = 0.0, False
        self.best_heading_d = None
        for h, r in zip(heads, res):
            if r["code"] > 0:
                score = np.float32(r["confidence"]) / np.float32(r["sigma"])
                if score > best_score:
                    registration_con.Trans1_2 = r["T"]
                    registration_con.sigma = r["sigma"]
                    registration_con.information_matrix = r["info"]
                    registration_con.confidence = r["confidence"]
                    best_score, self.best_heading_d = float(score), h
                ok = True
        return ok

    def mm_lls_icp(self, registration_cons: Constraint, max_iter_num: int = 20, dis_thre_unit: float = 1.5,
                   converge_translation: float = 0.002, converge_rotation_d: float = 0.01, dis_thre_min: float = 0.4,
                   dis_thre_update_rate: float = 1.1, used_feature_type: str = "111110", weight_strategy: str = "1101",
                   z_xy_balanced_ratio: float = 1.0, pt2pt_residual_window: float = 0.1,
                   pt2pl_residual_window: float = 0.1, pt2li_residual_window: float = 0.1, initial_guess=None,
                   apply_intersection_filter: bool = True, apply_motion_undistortion_while_registration: bool = False,
                   normal_shooting_on: bool = False, normal_bearing: float = 45.0, use_more_points: bool = False,
                   keep_less_source_points: bool = False, sigma_thre: float = 0.5,
                   min_neccessary_corr_ratio: float = 0.03, max_bearable_rotation_d: float = 45.0) -> int:
        p = abi.default_params()
        p.max_iter_num = max_iter_num
        p.dis_thre_unit = dis_thre_unit
        p.converge_translation = converge_translation
        p.converge_rotation_d = converge_rotation_d
        p.dis_thre_min = dis_thre_min
        p.dis_thre_update_rate = dis_thre_update_rate
        p.used_feature_type = used_feature_type.encode()[:7]
        p.weight_strategy = weight_strategy.encode()[:7]
        p.z_xy_balanced_ratio = z_xy_balanced_ratio
        p.pt2pt_residual_window = pt2pt_residual_window
        p.pt2pl_residual_window = pt2pl_residual_window
        p.pt2li_residual_window = pt2li_residual_window
        p.apply_intersection_filter = int(apply_intersection_filter)
        p.apply_motion_undistortion_while_registration = int(apply_motion_undistortion_while_registration)
        p.normal_shooting_on = int(normal_shooting_on)
        p.normal_bearing = normal_bearing
        p.use_more_points = int(use_more_points)
        p.keep_less_source_points = int(keep_less_source_points)
        p.sigma_thre = sigma_thre
        p.min_neccessary_corr_ratio = min_neccessary_corr_ratio
        p.max_bearable_rotation_d = max_bearable_rotation_d
        p.target_bound[:] = list(registration_cons.block1.local_bound)
        init = np.eye(4) if initial_guess is None else np.asarray(initial_guess, dtype=np.float64)
        pair = {
            "tgt": registration_cons.block1.clone_feature(False),               # :1180
            "src": registration_cons.block2.clone_feature(not use_more_points),  # :1181
            "params": p,
            "init_guess": init,
        }
        res, tr = self._ctx.run_batch([pair], want_trace=True)
        r = res[0]
        self.last_trace = tr[0]
        registration_cons.Trans1_2 = r["T"]
        registration_cons.information_matrix = r["info"]
        registration_cons.sigma = r["sigma"]
        registration_cons.confidence = r["confidence"]
        return r["code"]
