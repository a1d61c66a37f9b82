/*
 * mulls_b200 C-ABI — the drop-in boundary of the MULLS registration hot path on H100.
 *
 * Every entry point below is what a reference-side binding for this path would call. The
 * reference interface each one replaces is cited as file:line relative to the MULLS tree
 * (YuePanEdward/MULLS @ b275607):
 *
 *   mulls_icp_run            <- lo::CRegistration<PointT>::mm_lls_icp
 *                               include/common/cregistration.hpp:1114-1440
 *                               (determine_corres :1701-1835, multi_metrics_lls_tran_estimation
 *                                :1869-1967, pt2pl/pt2li/pt2pt_lls_summation :1976-2275,
 *                                get_multi_metrics_lls_residual :2518-2677, the per-class PCL kd-tree
 *                                build :1209-1232, intersection_filter :2894-2922)
 *   mulls_icp_run_batch      <- the same call made for N independent scan pairs (BASELINE config 4)
 *   mulls_batch_upload /
 *   mulls_batch_run_resident <- same, split so that inputs can stay resident in HBM between runs
 *   mulls_icp_run_sharded    <- the same call with the source clouds sharded over ranks
 *                               (BASELINE config 5); the per-iteration exchange is delegated to a
 *                               caller-supplied all-reduce; mulls_icp_run_sharded_nccl: the same over NCCL inside the
 *                               library (mulls_nccl_unique_id, mulls_nccl_init)
 *   mulls_nn_query           <- block1->tree_*->nearestKSearch(pt, 1, ...): the kd-trees mm_lls_icp leaves behind
 *                               (cregistration.hpp:1213-1232), read at src/map_manager.cpp:197-205
 *   mulls_scan_read / _probe <- DataIo::read_pc_cloud_block, include/common/dataio.hpp:1732-1756 (read_pcd_file :279-287,
 *                               read_bin_file :357-377); mulls_pose_write <- write_lo_pose_overwrite / _append :1896-1926
 *   mulls_pca_features       <- lo::PrincipleComponentAnalysis<PointT>::get_pc_pca_feature
 *                               include/common/pca.hpp:294-354 (+ get_pca_feature :390-434)
 *   mulls_pca_features_adaptive <- the same with distance_adaptive_on (pca.hpp:310-326)
 *   mulls_map_update        <- lo::MapManager::update_local_map, src/map_manager.cpp:17-145
 *   mulls_classify_nground   <- lo::CFilter<PointT>::classify_nground_pts, include/common/cfilter.hpp:2058-2290
 *   mulls_icp_run_to_map     <- mm_lls_icp with block1 = the device-resident local map
 *   mulls_fast_ground_filter <- lo::CFilter<PointT>::fast_ground_filter, include/common/cfilter.hpp:1658-2036
 *   mulls_voxel_downsample   <- lo::CFilter<PointT>::voxel_downsample, include/common/cfilter.hpp:83-165
 *   mulls_extract_semantic_pts <- lo::CFilter<PointT>::extract_semantic_pts, include/common/cfilter.hpp:2295-2413
 *   mulls_sor_filter         <- lo::CFilter<PointT>::sor_filter, include/common/cfilter.hpp:203-247
 *   mulls_vertical_intrinsic_calibration <- lo::CFilter<PointT>::vertical_intrinsic_calibration, cfilter.hpp:250-291
 *   mulls_timestamp_ratio    <- lo::CFilter<PointT>::get_pts_timestamp_ratio_in_frame, cfilter.hpp:412-467
 *   mulls_motion_compensation <- lo::CFilter<PointT>::apply_motion_compensation / batch_apply_motion_compensation,
 *                               cfilter.hpp:470-549
 *   mulls_ncc_correspondences <- lo::CRegistration<PointT>::find_feature_correspondence_ncc, cregistration.hpp:409-601
 *   mulls_coarse_reg_ransac  <- lo::CRegistration<PointT>::coarse_reg_ransac, cregistration.hpp:604-661
 *   mulls_coarse_reg_teaser  <- lo::CRegistration<PointT>::coarse_reg_teaser, cregistration.hpp:664-759
 *   mulls_non_max_suppress   <- lo::CFilter<PointT>::non_max_suppress(cloud_in_out, non_max_radius), cfilter.hpp:1183-1240
 *   mulls_omp_ndt            <- lo::CRegistration<PointT>::omp_ndt with use_direct_search (DIRECT7), cregistration.hpp:945-1021
 *   mulls_omp_ndt_kdtree     <- lo::CRegistration<PointT>::omp_ndt without use_direct_search (KDTREE), cregistration.hpp:945-1021
 *   mulls_omp_ndt_batch      <- P independent omp_ndt calls with shared parameters, in one call
 *   mulls_omp_gicp           <- lo::CRegistration<PointT>::omp_gicp with using_voxel_gicp (FastVGICP), cregistration.hpp:1024-1098
 *   mulls_omp_gicp_pcl       <- lo::CRegistration<PointT>::omp_gicp without using_voxel_gicp (point-wise GICP with PCL's BFGS),
 *                               cregistration.hpp:1024-1098
 *                               (mulls_voxel_downsample, mulls_fast_ground_filter and mulls_classify_nground also accept
 *                                device pointers for their input rows and output buffers)
 *
 * Plain C, plain pointers and sizes. No torch / Eigen / PCL types cross this boundary; the C++ shim
 * in include/common/cregistration.hpp converts Eigen/PCL objects to these PODs.
 *
 * Return convention: every function returns 0 on success or a negative MULLS_E_* code for
 * *infrastructure* errors (CUDA failure, bad argument, unsupported option). The *algorithmic* status
 * of a registration (1, -1, -2, -3 exactly as cregistration.hpp:1131-1136) is in mulls_icp_result.code.
 * There is no CPU fallback: without a CUDA device mulls_create fails with MULLS_E_CUDA.
 */
#ifndef MULLS_B200_ABI_H
#define MULLS_B200_ABI_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MULLS_NUM_CLASSES 6
/* Order of the feature classes everywhere in this ABI == the index order of `used_feature_type`
 * inside mm_lls_icp (cregistration.hpp:1196-1232): ground, pillar, facade, beam, roof, vertex. */
enum {
    MULLS_GROUND = 0,
    MULLS_PILLAR = 1,
    MULLS_FACADE = 2,
    MULLS_BEAM = 3,
    MULLS_ROOF = 4,
    MULLS_VERTEX = 5
};

/* infrastructure error codes */
enum {
    MULLS_OK = 0,
    MULLS_E_CUDA = -100,        /* CUDA runtime error, see mulls_last_error */
    MULLS_E_ARG = -101,         /* invalid argument */
    MULLS_E_CAPACITY = -102,    /* more points / pairs than the context was created for */
    MULLS_E_UNSUPPORTED = -103, /* option of mm_lls_icp that this build does not implement */
    MULLS_E_COMM = -104,        /* the caller's all-reduce callback failed */
    MULLS_E_IO = -105           /* a scan / pose file could not be opened or parsed */
};

#define MULLS_MAX_TRACE_ITERS 64

/* Zero-copy view of pcl::PointCloud<pcl::PointXYZINormal>::points (utility.hpp:40):
 * 12 floats (48 bytes) per point: x y z _ | normal_x normal_y normal_z _ | intensity curvature _ _ .
 * For pillar/beam clouds normal_* holds the principal direction (pca.hpp:437-454). Host pointer. */
typedef struct mulls_cloud_view {
    const float *aos48;
    size_t n;
} mulls_cloud_view;

/* The 21 scalar/string arguments of mm_lls_icp (cregistration.hpp:1114-1123), same names, same
 * defaults (see mulls_icp_default_params), plus the target block's bounding box that the function
 * reads from registration_cons.block1->local_bound (cregistration.hpp:2916). */
typedef struct mulls_icp_params {
    int32_t max_iter_num;
    float dis_thre_unit;
    float converge_translation;
    float converge_rotation_d;
    float dis_thre_min;
    float dis_thre_update_rate;
    char used_feature_type[8]; /* "111110" + NUL; order ground,pillar,facade,beam,roof,vertex */
    char weight_strategy[8];   /* "1101" + NUL; balance,residual,distance,intensity */
    float z_xy_balanced_ratio;
    float pt2pt_residual_window;
    float pt2pl_residual_window;
    float pt2li_residual_window;
    int32_t apply_intersection_filter;
    int32_t apply_motion_undistortion_while_registration; /* sources carry the timestamp ratio in `curvature` */
    int32_t normal_shooting_on;                           /* k = 10 normal-shooting candidates for ground/facade/roof */
    float normal_bearing;
    int32_t use_more_points; /* informational: the caller already chose pc_* vs pc_*_down */
    int32_t keep_less_source_points; /* random down-sampling of :2866-2892, deterministic in random_seed */
    float sigma_thre;
    float min_neccessary_corr_ratio;
    float max_bearable_rotation_d;
    double target_bound[6]; /* block1->local_bound: min_x min_y min_z max_x max_y max_z */
    /* Seed of the random down-sampling used by keep_less_source_points. The reference seeds pcl::RandomSample
     * with time(NULL) (cfilter.hpp:620, SURVEY Q11), i.e. its result is not reproducible; here the kept subset is
     * a deterministic uniform sample: the k points with the smallest splitmix64(seed, cloud, index) keys. */
    uint32_t random_seed;
    uint32_t _pad;
} mulls_icp_params;

/* Outputs of mm_lls_icp: constraint_t::Trans1_2 / information_matrix / sigma / confidence
 * (cregistration.hpp:1405, :1418-1420) and the return code (:1439). Matrices are ROW-major. */
typedef struct mulls_icp_result {
    double T[16];
    double info[36];
    float sigma;
    float confidence;
    int32_t code;  /* 1 ok, -1 step too large, -2 too few correspondences, -3 sigma too large, 0 no iteration */
    int32_t iters; /* number of loop bodies entered (the failing / converging one included) */
    uint32_t n_corr[MULLS_NUM_CLASSES]; /* |Corr_f| per class in the last executed iteration */
    uint32_t n_src[MULLS_NUM_CLASSES];  /* source points per class left after the last executed iteration */
} mulls_icp_result;

/* Optional per-iteration trace (parity tests): what the reference would LOG(INFO) per iteration. */
typedef struct mulls_icp_trace {
    int32_t n_iter;
    int32_t _pad;
    double atpa[MULLS_MAX_TRACE_ITERS][36]; /* row-major, symmetrised as at cregistration.hpp:1924-1938 */
    double atpb[MULLS_MAX_TRACE_ITERS][6];
    double x[MULLS_MAX_TRACE_ITERS][6];
    uint32_t n_corr[MULLS_MAX_TRACE_ITERS][MULLS_NUM_CLASSES];
    uint32_t n_src[MULLS_MAX_TRACE_ITERS][MULLS_NUM_CLASSES]; /* source sizes after determine_corres */
} mulls_icp_trace;

typedef struct mulls_ctx mulls_ctx;

/* Create a context on CUDA device `device` able to hold `max_pairs` scan pairs of at most
 * `max_src_pts` source and `max_tgt_pts` target points each (sum over the six classes). */
mulls_ctx *mulls_create(int device, size_t max_pairs, size_t max_src_pts, size_t max_tgt_pts);
void mulls_destroy(mulls_ctx *ctx);
const char *mulls_last_error(const mulls_ctx *ctx); /* ctx may be NULL: error of the failed create */

/* Fill `p` with the default arguments of mm_lls_icp (cregistration.hpp:1115-1123). */
void mulls_icp_default_params(mulls_icp_params *p);

/* One registration: host clouds in, host result out (H2D + all iterations + D2H inside). */
int mulls_icp_run(mulls_ctx *ctx, const mulls_cloud_view tgt[MULLS_NUM_CLASSES],
                  const mulls_cloud_view src[MULLS_NUM_CLASSES], const mulls_icp_params *params,
                  const double init_guess[16] /* row-major 4x4 */, mulls_icp_result *out,
                  mulls_icp_trace *trace /* may be NULL */);

/* n_pairs independent registrations in one call. tgt/src are [n_pairs][6]. */
int mulls_icp_run_batch(mulls_ctx *ctx, size_t n_pairs, const mulls_cloud_view *tgt,
                        const mulls_cloud_view *src, const mulls_icp_params *params /* [n_pairs] */,
                        const double *init_guess /* [n_pairs][16] */, mulls_icp_result *out /* [n_pairs] */,
                        mulls_icp_trace *trace /* [n_pairs] or NULL */);

/* Split form: copy the inputs to HBM once, then run the whole path (ingest: filter, spatial sort,
 * grid build; all iterations; posterior) any number of times from the resident copies. */
int mulls_batch_upload(mulls_ctx *ctx, size_t n_pairs, const mulls_cloud_view *tgt,
                       const mulls_cloud_view *src, const mulls_icp_params *params,
                       const double *init_guess);
int mulls_batch_run_resident(mulls_ctx *ctx, mulls_icp_result *out /* [n_pairs] or NULL */,
                             mulls_icp_trace *trace /* [n_pairs] or NULL */);

/* Statistics of the last call on this context (for bench.py). A registration fills every field; a front-end call
 * (PCA, SOR, raw-scan corrections, NCC, RANSAC, voxel / ground filter, classification, extract_semantic_pts) fills
 * kernel_launches and ms_total and zeroes the rest, so a call that launches nothing reports zero launches. */
typedef struct mulls_run_stats {
    uint64_t kernel_launches;   /* kernels of this library launched by the last call (library sorts and scans are not counted) */
    uint64_t algorithmic_bytes; /* sum over pairs and executed iterations of 28*(N_s,active + N_t) */
    uint64_t iterations;        /* sum over pairs of executed iterations */
    uint64_t search_launches;   /* launches of the search kernel (one per ICP iteration of the batch) */
    float ms_ingest;            /* device time of the ingest phase (CUDA events) */
    float ms_iterate;           /* device time of the iteration kernels */
    float ms_search;            /* device time of the fused transform+NN+claim kernel only */
    float ms_total;
    float ms_search_iter[MULLS_MAX_TRACE_ITERS]; /* per-iteration device time of the search kernel */
    /* one-shot calls with host buffers (mulls_icp_run_batch): where the call's wall time went */
    float ms_host_pack; /* host: repacking the clouds into the pinned staging (0 when they are shipped as rows) */
    float ms_h2d;       /* device: first cloud copy enqueued -> last cloud copy done */
    float ms_host_call; /* host: wall time of the whole call */
    float ms_host_upload; /* host: wall time of the upload part (tables, packing, enqueueing the copies) */
} mulls_run_stats;
int mulls_get_stats(const mulls_ctx *ctx, mulls_run_stats *out);

/* Source-sharded single registration (BASELINE config 5): every rank holds the full target and a
 * contiguous slice of every source class starting at global index src_index_base[c]. The caller
 * supplies the all-reduce used once (sum, doubles) or twice (+ min, int32 claim table) per
 * iteration on device buffers; with NCCL: ncclAllReduce(buf, buf, count, type, op, comm, stream). */
typedef int (*mulls_allreduce_fn)(void *user, void *device_buf, size_t count,
                                  int dtype /* 0 = float64, 1 = int32 */, int op /* 0 = sum, 1 = min */,
                                  void *cuda_stream);
int mulls_icp_run_sharded(mulls_ctx *ctx, const mulls_cloud_view tgt[MULLS_NUM_CLASSES],
                          const mulls_cloud_view src_shard[MULLS_NUM_CLASSES],
                          const uint32_t src_index_base[MULLS_NUM_CLASSES],
                          const uint32_t src_global_n[MULLS_NUM_CLASSES],
                          const mulls_icp_params *params, const double init_guess[16],
                          mulls_allreduce_fn allreduce, void *user, mulls_icp_result *out,
                          mulls_icp_trace *trace);

/* The same over NCCL, entirely inside the library (no callback, nothing interpreted in the loop): the three
 * exchanges of an iteration are ncclAllReduce calls enqueued on the context's stream between its kernels.
 * libnccl.so.2 is resolved at run time with dlopen (inside a PyTorch process: the NCCL PyTorch has loaded), so the
 * library has no link-time dependency on NCCL.
 *   mulls_nccl_unique_id   rank 0 creates an id (ncclGetUniqueId) and ships the 128 bytes to the other ranks by any
 *                          means (MPI, a file, torch.distributed.broadcast)
 *   mulls_nccl_init        collective: ncclCommInitRank on the context's device; the communicator belongs to the
 *                          context and is destroyed with it
 *   mulls_icp_run_sharded_nccl   `comm` = an ncclComm_t of the SAME libnccl (e.g. one the application already has
 *                          for these ranks), or NULL for the context's own (mulls_nccl_init) */
#define MULLS_NCCL_ID_BYTES 128
int mulls_nccl_unique_id(char id[MULLS_NCCL_ID_BYTES]);
int mulls_nccl_init(mulls_ctx *ctx, int rank, int world, const char id[MULLS_NCCL_ID_BYTES]);
int mulls_icp_run_sharded_nccl(mulls_ctx *ctx, void *comm /* ncclComm_t or NULL */,
                               const mulls_cloud_view tgt[MULLS_NUM_CLASSES],
                               const mulls_cloud_view src_shard[MULLS_NUM_CLASSES],
                               const uint32_t src_index_base[MULLS_NUM_CLASSES],
                               const uint32_t src_global_n[MULLS_NUM_CLASSES], const mulls_icp_params *params,
                               const double init_guess[16], mulls_icp_result *out, mulls_icp_trace *trace);

/* Stand-in for block1->tree_* (cregistration.hpp:1213-1232): mm_lls_icp leaves a kd-tree per target class in
 * registration_cons.block1, and MapManager::map_scan_feature_pts_distance_removal (src/map_manager.cpp:221-258, called
 * from :197-205) runs nearestKSearch(point, 1, ...) on them. Here the last mulls_icp_run / mulls_icp_run_batch (pair 0)
 * on `ctx` leaves its sorted target slices and their grid in HBM, and this call answers the same query on them:
 * for every query point the exact nearest target of class `cls` (FLANN float distance, ties to the lower index)
 * within the radius the registration searched (2.5 * dis_thre_unit, which covers dynamic_dist_thre_max of
 * map_manager.h:28). idx[i] = index of that target in the caller's ORIGINAL class cloud (the reference's index is
 * into its bbox-filtered private clone), d2[i] = squared distance; nothing within the radius: idx -1, d2 +inf.
 * Targets removed by the intersection filter are not candidates (as in the reference: the trees are built after
 * the filter, :1186-1232). Returns MULLS_E_ARG if no registration has run on the context since its last upload. */
int mulls_nn_query(mulls_ctx *ctx, int cls, const float *xyz /* [n][3], host */, size_t n, int32_t *idx /* [n] */,
                   float *d2 /* [n] */);

/* PCA neighbourhood features (pca.hpp:294-354): for every `stride`-th point of `cloud` take the
 * at most `k` nearest neighbours within `radius` (the point itself included), and return
 * eigenvalues (descending), principal direction, normal direction, and the neighbour count.
 * k <= 0 or k > 1024 is treated as 1024 (the reference uses 25..50). */
typedef struct mulls_pca_out {
    float *eigenvalues; /* [n][3] lambda1 >= lambda2 >= lambda3 (pcl::PCA convention) */
    float *principal;   /* [n][3] unit principal direction (eigenvector of lambda1) */
    float *normal;      /* [n][3] unit normal direction (col0 x col1, pcl::PCA convention) */
    int32_t *pt_num;    /* [n] neighbours used (0 for points skipped by the stride) */
} mulls_pca_out;
int mulls_pca_features(mulls_ctx *ctx, mulls_cloud_view cloud, float radius, int k, int stride,
                       mulls_pca_out *out);
/* The same with distance_adaptive_on = true (pca.hpp:310-326): a point at range dist = |xyz| > unit_dist (float norm,
 * strict) searches the radius (float)(sqrt(dist / unit_dist) * radius); nearer points search `radius`. unit_dist <= 0:
 * MULLS_E_ARG (classify_nground_pts passes 30, the function's own default is 35). */
int mulls_pca_features_adaptive(mulls_ctx *ctx, mulls_cloud_view cloud, float radius, int k, int stride, float unit_dist,
                                mulls_pca_out *out);

/* ---- Device-resident local map (SURVEY §8(f) rank 1) -------------------------------------------------------
 * lo::MapManager::update_local_map, src/map_manager.cpp:17-145 (+ map_based_dynamic_close_removal :149-217,
 * map_scan_feature_pts_distance_removal :221-258; cloudblock_t::append_feature / transform_feature
 * utility.hpp:438-470, :495-516; CFilter::dist_filter cfilter.hpp:838-873; random_downsample_pcl :606-628;
 * get_cloud_bbx utility.hpp:817-847). The six target clouds of the scan-to-map registration stay in HBM between
 * frames: per frame only the new scan's down-sampled feature clouds cross PCIe, and mulls_icp_run_to_map reads the
 * target straight from the map. */
typedef struct mulls_map mulls_map;

/* Arguments of update_local_map (include/pgo/map_manager.h:22-32), same names and defaults. */
typedef struct mulls_map_params {
    float local_map_radius;              /* 80 */
    int32_t max_num_pts;                 /* 20000 */
    int32_t kept_vertex_num;             /* 800 */
    float last_frame_reliable_radius;    /* 60; accepted and unused, as in the reference body */
    int32_t map_based_dynamic_removal_on; /* 0; needs the preceding mulls_icp_run_to_map on the same context: the
                                            reference queries the kd-trees that registration left in block1 */
    char used_feature_type[8];           /* "111110" */
    float dynamic_removal_center_radius; /* 30 */
    float dynamic_dist_thre_min;         /* 0.3 */
    float dynamic_dist_thre_max;         /* 3.0 */
    float near_dist_thre;                /* 0.03 */
    int32_t recalculate_feature_on;      /* 0; 1: update_cloud_vectors (:95-115, :260-295) on the map's pillars and beams */
    uint32_t random_seed;                /* seed of the budgeted down-sampling (pcl::RandomSample in the reference) */
} mulls_map_params;

typedef struct mulls_map_info {
    double pose_lo[16];     /* local_map->pose_lo after the update (= the scan's pose), row-major */
    double local_bound[6];  /* local_map->local_bound: min_x min_y min_z max_x max_y max_z (map frame) */
    double bound[6];        /* local_map->bound (world frame, points transformed by pose_lo) */
    uint32_t n[MULLS_NUM_CLASSES];          /* points per class after the update */
    uint32_t n_appended[MULLS_NUM_CLASSES]; /* scan points appended per class (after dynamic removal) */
    int32_t feature_point_num;              /* ground + pillar + facade + beam + roof */
    float ms_update;                        /* device time of the update (CUDA events) */
} mulls_map_info;

void mulls_map_default_params(mulls_map_params *p);
/* A map whose six class clouds hold at most `max_pts_per_class` points each (map + appended scan). */
mulls_map *mulls_map_create(mulls_ctx *ctx, size_t max_pts_per_class);
void mulls_map_destroy(mulls_map *map);
/* Replace the content of the map by host clouds (e.g. a map built elsewhere) and set its pose. */
int mulls_map_set(mulls_map *map, const mulls_cloud_view cls[MULLS_NUM_CLASSES], const double pose_lo[16]);
/* update_local_map(local_map, last_target_cblock, ...): `scan_down` are last_target_cblock->pc_*_down (index 5:
 * pc_vertex), `scan_pose_lo` its pose_lo. The scan block itself is not modified (the reference leaves its down
 * clouds transformed into the old map frame and thinned by the dynamic removal). */
int mulls_map_update(mulls_map *map, const mulls_cloud_view scan_down[MULLS_NUM_CLASSES], const double scan_pose_lo[16],
                     const mulls_map_params *params, mulls_map_info *info /* may be NULL */);
int mulls_map_get_info(const mulls_map *map, mulls_map_info *info);
/* Copy class `cls` of the map to the host (48-byte rows); *n receives the point count, `cap` is the room in rows. */
int mulls_map_download(mulls_map *map, int cls, float *out_aos48, size_t cap, size_t *n);
/* mm_lls_icp with block1 = the resident map: the target views and block1->local_bound come from the map
 * (params->target_bound is ignored), only the source clouds are copied to the device. */
int mulls_icp_run_to_map(mulls_ctx *ctx, mulls_map *map, const mulls_cloud_view src[MULLS_NUM_CLASSES],
                         const mulls_icp_params *params, const double init_guess[16], mulls_icp_result *out,
                         mulls_icp_trace *trace /* may be NULL */);

/* ---- Non-ground feature classification (SURVEY §8(f) rank 2) -------------------------------------------------
 * lo::CFilter<PointT>::classify_nground_pts, include/common/cfilter.hpp:2058-2290: PCA of every pca_down_rate-th point
 * (pca.hpp:294-354, a16), linearity / planarity / direction thresholds -> pillar, beam, facade, roof (:2103-2166),
 * vertex-neighbourhood promotion (:2169-2210), keypoints with the neighbourhood-category descriptor
 * (encode_stable_points, :1071-1181), non-maximum suppression (non_max_suppress, :1243-1312) and the fixed-number
 * down-sampling (random_downsample_pcl :606-628, xy_normal_balanced_downsample :551-602). */
enum {
    MULLS_OUT_PILLAR = 0,
    MULLS_OUT_BEAM = 1,
    MULLS_OUT_FACADE = 2,
    MULLS_OUT_ROOF = 3,
    MULLS_OUT_PILLAR_DOWN = 4,
    MULLS_OUT_BEAM_DOWN = 5,
    MULLS_OUT_FACADE_DOWN = 6,
    MULLS_OUT_ROOF_DOWN = 7,
    MULLS_OUT_VERTEX = 8,   /* the keypoints this call appends to cloud_vertex */
    MULLS_OUT_UNGROUND = 9, /* cloud_in as the call leaves it (sampled, normals assigned) */
    MULLS_OUT_COUNT = 10
};

/* Arguments of classify_nground_pts (cfilter.hpp:2070-2081), same names; defaults where the reference has them,
 * otherwise the values extract_semantic_pts / test/mulls_slam.cpp pass by default. */
typedef struct mulls_classify_params {
    float neighbor_searching_radius;      /* 1.0 */
    int32_t neighbor_k;                   /* 50; 1..64 */
    int32_t neigh_k_min;                  /* 8 */
    int32_t pca_down_rate;                /* 1 */
    float edge_thre;                      /* 0.65 */
    float planar_thre;                    /* 0.65 */
    float edge_thre_down;                 /* 0.75 */
    float planar_thre_down;               /* 0.75 */
    int32_t extract_vertex_points_method; /* 2 */
    float curvature_thre;                 /* 0.12 */
    float vertex_curvature_non_max_radius; /* 1.5 * radius; unused by the reference body */
    float linear_vertical_sin_high_thre;  /* 0.94 */
    float linear_vertical_sin_low_thre;   /* 0.17 */
    float planar_vertical_sin_high_thre;  /* 0.98 */
    float planar_vertical_sin_low_thre;   /* 0.34 */
    int32_t fixed_num_downsampling;       /* 0 */
    int32_t pillar_down_fixed_num;        /* 200 */
    int32_t facade_down_fixed_num;        /* 800 */
    int32_t beam_down_fixed_num;          /* 200 */
    int32_t roof_down_fixed_num;          /* 100 */
    int32_t unground_down_fixed_num;      /* 20000 */
    float beam_height_max;                /* FLT_MAX */
    float roof_height_min;                /* -FLT_MAX */
    float feature_pts_ratio_guess;        /* 0.3 */
    int32_t sharpen_with_nms;             /* 1 */
    int32_t use_distance_adaptive_pca;    /* 0; != 0: every query farther than pca_unit_distance from the origin searches
                                             sqrt(dist / pca_unit_distance) * neighbor_searching_radius (pca.hpp:310-326);
                                             needs pca_unit_distance > 0, else MULLS_E_UNSUPPORTED */
    uint32_t random_seed;                 /* seed of every random_downsample_pcl inside */
    float pca_unit_distance;              /* 0 (unset); classify_nground_pts passes 30 (cfilter.hpp:2093) */
} mulls_classify_params;

typedef struct mulls_classify_out {
    float *rows[MULLS_OUT_COUNT]; /* caller buffers of `cap` 48-byte rows each (NULL: not wanted) */
    size_t cap;                   /* cloud_in.n rows are always enough */
    size_t n[MULLS_OUT_COUNT];    /* rows written */
} mulls_classify_out;

void mulls_classify_default_params(mulls_classify_params *p);
int mulls_classify_nground(mulls_ctx *ctx, mulls_cloud_view cloud_in, const mulls_classify_params *params,
                           mulls_classify_out *out);

/* ---- Ground segmentation (SURVEY §8(f) rank 2, first half) ---------------------------------------------------
 * lo::CFilter<PointT>::fast_ground_filter, include/common/cfilter.hpp:1658-2036: 2-D grid over the cloud, lowest point
 * per cell and per 3x3 neighbourhood, two height thresholds -> ground / non-ground, rate-based down-sampling by the
 * position inside the cell, and (estimate_ground_normal_method 3, the default) a RANSAC plane per ground cell
 * (estimate_ground_normal_by_ransac :2038-2054 -> CProceesing::plane_seg_ransac cprocessing.hpp:67-105 ->
 * pcl::SACSegmentation, SACMODEL_PLANE / SAC_RANSAC, optimize coefficients; PCL 1.10 semantics restated). The first
 * stage of extract_semantic_pts (:2355-2361); its `cloud_unground` is the input of mulls_classify_nground. */
typedef struct mulls_ground_params { /* argument names of :1658-1672; defaults = extract_semantic_pts / mulls_slam gflags */
    int32_t min_grid_pt_num;                     /* 10  (gf_grid_min_pt_num) */
    float grid_resolution;                       /* 3.0 (gf_grid_size) */
    float max_height_difference;                 /* 0.3 (gf_in_grid_h_thre) */
    float neighbor_height_diff;                  /* 1.5 (gf_neigh_grid_h_thre) */
    float max_ground_height;                     /* 5.0 (gf_max_h) */
    int32_t ground_random_down_rate;             /* 15  (gf_ground_down_rate) */
    int32_t ground_random_down_down_rate;        /* 2   (gf_down_down_rate) */
    int32_t nonground_random_down_rate;          /* 3   (gf_nonground_down_rate) */
    int32_t reliable_neighbor_grid_num_thre;     /* 0 */
    int32_t estimate_ground_normal_method;       /* 3; 0 = (0,0,1), 3 = RANSAC per cell; 1 and 2: MULLS_E_UNSUPPORTED */
    float normal_estimation_radius;              /* 2.0; only read by method 1 */
    int32_t distance_weight_downsampling_method; /* 2 (dist_inverse_sampling_method): 0 off, 1 linear, 2 quadratic */
    float standard_distance;                     /* 15.0 (unit_dist) */
    int32_t fixed_num_downsampling;              /* 0 */
    int32_t down_ground_fixed_num;               /* 300 (ground_down_fixed_num) */
    float intensity_thre;                        /* FLT_MAX */
    int32_t apply_grid_wise_outlier_filter;      /* 0 (extract_semantic_pts passes apply_scanner_filter here, :2361) */
    float outlier_std_scale;                     /* 3.0 */
    uint32_t random_seed; /* seed of random_downsample_pcl (fixed_num_downsampling); pcl::RandomSample is time-seeded */
} mulls_ground_params;

typedef struct mulls_ground_out {
    float *ground;      /* cloud_ground: caller buffers of `cap` 48-byte rows each (NULL: not wanted) */
    float *ground_down; /* cloud_ground_down */
    float *unground;    /* cloud_unground; row[3] = approximate height above ground (:1752, :1880, :1894) */
    size_t cap;         /* cloud_in.n rows are always enough */
    size_t n_ground, n_ground_down, n_unground;
} mulls_ground_out;

void mulls_ground_default_params(mulls_ground_params *p);
int mulls_fast_ground_filter(mulls_ctx *ctx, mulls_cloud_view cloud_in, const mulls_ground_params *params,
                             mulls_ground_out *out);

/* lo::CFilter<PointT>::voxel_downsample, include/common/cfilter.hpp:83-165: one point per occupied voxel, in voxel-index
 * order (voxel_size < 0.001 copies the cloud, :89-97). `out` receives at most cloud_in.n rows. The reference's
 * std::sort leaves open WHICH point of a voxel survives; here it is the one with the lowest index. */
int mulls_voxel_downsample(mulls_ctx *ctx, mulls_cloud_view cloud_in, float voxel_size, float *out, size_t cap, size_t *n_out);

/* lo::CFilter<PointT>::extract_semantic_pts, include/common/cfilter.hpp:2295-2413, the per-frame feature extraction:
 * voxel_downsample(pc_raw -> pc_down) (:2346), fast_ground_filter(pc_down) (:2355-2361), classify_nground_pts(pc_unground)
 * (:2378-2391) — chained in HBM: only the raw scan goes up and the feature clouds come down. Not produced: pc_sketch
 * (:2348), the scanner / semantic-mask pre-filters (:2328-2342) and update_parameters_self_adaptive (:2406-2410). */
typedef struct mulls_extract_params {
    float vf_downsample_resolution; /* cloud_down_res */
    mulls_ground_params ground;     /* the gf_* arguments */
    mulls_classify_params classify; /* the pca_* / *_thre / *_fixed_num arguments */
} mulls_extract_params;

typedef struct mulls_extract_out {
    float *pc_down;        /* in_block->pc_down; caller buffers of `cap` 48-byte rows (NULL: not wanted) */
    float *pc_ground;      /* in_block->pc_ground */
    float *pc_ground_down; /* in_block->pc_ground_down */
    size_t cap;            /* pc_raw.n rows are always enough */
    size_t n_down, n_ground, n_ground_down;
    mulls_classify_out cls; /* pc_pillar .. pc_roof_down, pc_vertex, pc_unground (MULLS_OUT_*) */
} mulls_extract_out;

int mulls_extract_semantic_pts(mulls_ctx *ctx, mulls_cloud_view pc_raw, const mulls_extract_params *params,
                               mulls_extract_out *out);

/* lo::CFilter<PointT>::sor_filter, include/common/cfilter.hpp:203-247 (both overloads; test/mulls_slam.cpp:1008-1009 runs it
 * with mean_k 20, n_std 2.0 on the merged map): pcl::StatisticalOutlierRemoval, PCL 1.10 applyFilterIndices (SURVEY
 * Appendix B item 10). For every point with finite x, y, z: the mean of the square roots of the squared (FLANN float)
 * distances to its mean_k nearest other points, summed in double in ascending order, stored as float (mean_dist[i]; 0 for
 * the other points). Then, in input order and in double, sum and sum of squares (the float square widened), mean =
 * sum / n_valid, stddev = sqrt((sq_sum - sum * sum / n_valid) / (n_valid - 1)), threshold = mean + n_std * stddev, and
 * point i is kept iff NOT (mean_dist[i] > threshold) — a NaN threshold keeps every point. keep_bits: bit i % 8 of byte
 * i / 8 (LSB first) set for a kept point; stats->n_kept counts them. Kept rows are meant to be gathered in input order.
 * Defined where the reference is not:
 *   - points with a non-finite coordinate never enter the neighbour search (PCL would hand them to FLANN, as the merged
 *     map claims is_dense); they get distance 0 and count towards neither n_valid nor the neighbours of others
 *   - at most mean_k finite points: MULLS_E_ARG (PCL would read past its neighbour vector)
 *   - mean_k < 1 or mean_k > 63: MULLS_E_ARG
 * A cloud of more than the context's max_tgt_pts points: MULLS_E_CAPACITY. The call replaces the batch resident on the
 * context (as mulls_pca_features does). */
typedef struct mulls_sor_stats {
    double mean, stddev, threshold;
    uint64_t n_valid, n_kept;
} mulls_sor_stats;
int mulls_sor_filter(mulls_ctx *ctx, mulls_cloud_view cloud, int mean_k, double n_std,
                     uint8_t *keep_bits /* [(n+7)/8] */, float *mean_dist /* [n] or NULL */,
                     mulls_sor_stats *stats /* or NULL */);

/* ---- Raw-scan corrections: the CFilter members test/mulls_slam.cpp runs on every raw scan (:406-412, :707-711,
 * :967-980). Each call is stateless: the rows go to the device, the column the member changes comes back, nothing stays
 * resident and the batch resident on the context is left alone. No multiply-add is contracted. A cloud (or, for
 * mulls_motion_compensation, the clouds together) of more than the context's max_tgt_pts points: MULLS_E_CAPACITY. A NULL
 * pointer where points are to be read or written: MULLS_E_ARG. An empty cloud does no device work. */

/* vertical_intrinsic_calibration(cloud, var_vertical_ang_d, inverse_z), cfilter.hpp:250-291. xyz_out [n][3] receives the
 * coordinates the member leaves, *applied what it returns:
 *   - var_vertical_ang_d == 0: the input's coordinates, *applied = 0 (no device work)
 *   - var_vertical_ang_d >= 180 or inverse_z: z negated, *applied = 0
 *   - otherwise dist = (double)sqrtf(x*x + y*y + z*z) (float products and sum), v = asin(z / dist), v_c = v + var
 *     (radians), x and y times cos(v_c) / cos(v), z = dist * sin(v_c), all in double, stored as float; *applied = 1.
 *     A point at the origin becomes NaN, as in the reference.
 * asin / cos / sin are CUDA's double functions, not the host's libm: a coordinate can differ from the host's in its
 * last float bit. */
int mulls_vertical_intrinsic_calibration(mulls_ctx *ctx, mulls_cloud_view cloud, double var_vertical_ang_d, int inverse_z,
                                         float *xyz_out /* [n][3] */, int *applied);

/* get_pts_timestamp_ratio_in_frame(cloud, timestamp_available, scan_begin_ang_deg, scan_duration_ms), cfilter.hpp:412-467:
 * ratio_out [n] receives the new curvature column (the member always returns true).
 *   - timestamp_available: last / first = the running max_ / min_ macros (utility.hpp:31-32) over the curvature column
 *     in input order — a NaN timestamp resets both, so they are the extremes of the points after the last NaN (NaN when
 *     the last point is NaN); if last - first < 0.75 * scan_duration_ms it becomes the (float) duration; ratio =
 *     min_(1.0, max_(0.0, (last - curvature) / duration)) in double. Equal timestamps give 0 / 0 = NaN, as in the
 *     reference. Bit-exact.
 *   - otherwise: the float atan2(y, x), widened; + 2 pi when negative; + the begin angle; - 2 pi when >= 2 pi; ratio =
 *     (2 pi - angle) / (2 pi), in double. The float atan2 is computed as the double one rounded to float. */
int mulls_timestamp_ratio(mulls_ctx *ctx, mulls_cloud_view cloud, int timestamp_available, double scan_begin_ang_deg,
                          float scan_duration_ms, float *ratio_out /* [n] */);

/* apply_motion_compensation(cloud, T, s_ambiguous_thre), cfilter.hpp:470-516, over n_clouds (1..6) clouds in one upload
 * and one launch: one cloud for apply_motion_compensation, five or six for batch_apply_motion_compensation (:519-549).
 * q = Eigen::Quaterniond(T's rotation), computed once on the host; a point whose curvature s (the timestamp ratio) is
 * < s_ambiguous_thre or > 1.0 - s_ambiguous_thre keeps its coordinates, every other point becomes
 * Identity().slerp(s, q) * p + s * t in double, stored as float. xyz_out[c] [clouds[c].n][3] receives cloud c's
 * coordinates. n_clouds outside 1..6: MULLS_E_ARG. */
int mulls_motion_compensation(mulls_ctx *ctx, const mulls_cloud_view *clouds, int n_clouds, const double T[16] /* row-major */,
                              float s_ambiguous_thre, float *const *xyz_out);

/* lo::CRegistration<PointT>::find_feature_correspondence_ncc(target_kpts, source_kpts, target_corrs, source_corrs,
 * fixed_num_corr, corr_num, reciprocal_on), cregistration.hpp:409-601: the keypoint matching in front of the global
 * registration (test/mulls_reg.cpp:173-174, test/mulls_slam.cpp:534-535). Stateless like the raw-scan corrections: the
 * batch resident on the context and its grid are left alone. The keypoints are 48-byte pcl::PointXYZINormal rows
 * (x y z data[3] | normal_x normal_y normal_z normal[3] | intensity curvature _ _). tgt_idx[k] / src_idx[k] (k < *n_out)
 * receive the row indices of the k-th correspondence in the order the reference appends them; the caller appends
 * target_kpts[tgt_idx[k]] to target_corrs and source_kpts[src_idx[k]] to source_corrs.
 *   - fewer than 10 keypoints in either cloud (:421-425): *performed = 0, *n_out = 0 (the reference returns false and
 *     leaves both output clouds as they are); otherwise *performed = 1 (it returns true)
 *   - intensity range over the target only, with max_ / min_ (utility.hpp:31-32) started from 0 and FLT_MAX (not
 *     -FLT_MAX); a NaN intensity becomes the running value and the next point replaces it
 *   - descriptor (11 floats): the decimal digit pairs of (int)normal[0] and (int)normal[1] (/1000000, %1000000/10000,
 *     %10000/100, %100, C++ integer semantics), (i - min) / (max - min) in float times the double 255.0,
 *     normal[3] * 100 and data[3] * 30 in float; (int) of a NaN or out-of-range float is INT_MIN, the x86-64 result. A
 *     constant target intensity gives NaN / infinite components, as in the reference
 *   - distance: the float L1 sum over the 11 components, in component order, no contraction
 *   - plain mode (!fixed_num_corr, !reciprocal_on): per target i in order, the first j with d < best from (FLT_MAX, 0);
 *     NaN never wins, a row without a finite value below FLT_MAX pairs with source 0
 *   - reciprocal mode: the same, target i dropped when best_i > d[r][j_i] for some target r (the non-NaN column minimum)
 *   - fixed-number mode (reciprocal_on ignored): K = min_(corr_num, n_t * n_s) compared as size_t (negative corr_num:
 *     every pair, 0: none); the first K pairs in ascending distance, ties in pair-index order (i * n_s + j), NaN after
 *     every number (std::sort leaves that order open); walked in order, a pair is skipped when its target or its source
 *     already holds 7 kept pairs. n_t * n_s > INT_MAX (the reference's int pair index): MULLS_E_ARG
 * A cloud of more than the context's max_tgt_pts keypoints: MULLS_E_CAPACITY. More correspondences than cap: MULLS_E_ARG,
 * with nothing written. Indices are int32_t like the reference's int keypoint counts; NULL index arrays need cap == 0. */
int mulls_ncc_correspondences(mulls_ctx *ctx, mulls_cloud_view target_kpts, mulls_cloud_view source_kpts, int fixed_num_corr,
                              int corr_num, int reciprocal_on, int32_t *tgt_idx, int32_t *src_idx, size_t cap, size_t *n_out,
                              int *performed);

/* lo::CRegistration<PointT>::coarse_reg_ransac(target_pts, source_pts, tran_mat, noise_bound, min_inlier_num,
 * max_iter_num), cregistration.hpp:604-661: the coarse transform of the global registration (test/mulls_reg.cpp:170-195,
 * test/mulls_slam.cpp:532-560), PCL 1.10's CorrespondenceRejectorSampleConsensus over the correspondences i <-> i,
 * i < N = target_pts.n, with the inlier threshold noise_bound, max_iter_num iterations and the refinement on. Stateless
 * like mulls_ncc_correspondences: the batch resident on the context and its grid are left alone. 48-byte rows as for
 * the NCC matching; only x y z are read. Readings (ransac_core.cuh R1-R6 and C1-C2 state them in full):
 *   - the sample stream is boost::mt19937(12345) with rnd() = mt() >> 1 on the model's persistent shuffle, a sample is
 *     good when its three pairwise float squared source distances exceed the sample distance threshold (float
 *     covariance of the N source points, pcl::eigen33); 1000 attempts per selection, an empty selection ends the search
 *   - each hypothesis is pcl::umeyama in double (3x3 Jacobi SVD, sums in a fixed order) cast to float; a correspondence
 *     is an inlier when the float squared error of T [s, 1] against t is < noise_bound^2 in double
 *   - the adaptive k of RandomSampleConsensus (p = 0.99), at most max_iter_num + 1 hypotheses (max_iter_num == 0: none)
 *   - refineModel(3, 1000): re-fit, re-select, threshold sqrt(min(noise_bound^2, 9 * 2.1981 * median)), stopping when
 *     the inlier set repeats, the sizes oscillate, or after 1000 rounds
 *   - the search finds no model (N < 3, no good sample, max_iter_num == 0), or fewer than 3 inliers survive: all N
 *     correspondences remain, with the identity; a failed refinement leaves none and the identity (PCL's matrix would
 *     be uninitialised; it is read only when min_inlier_num is 0)
 * Outputs: *status is 1 when the remaining count is >= 2 * min_inlier_num, 0 when it is >= min_inlier_num, -1 otherwise
 * (the comparisons are against size_t, so a negative min_inlier_num always gives -1); tran_mat (row-major) is written
 * only when *status >= 0, with the float model widened; *n_inliers is the remaining count and *n_hypotheses the
 * hypotheses scored. source_pts shorter than target_pts, or a NULL output: MULLS_E_ARG (nothing written). N above the
 * context's max_tgt_pts: MULLS_E_CAPACITY. */
int mulls_coarse_reg_ransac(mulls_ctx *ctx, mulls_cloud_view target_pts, mulls_cloud_view source_pts, float noise_bound,
                            int min_inlier_num, int max_iter_num, double tran_mat[16] /* row-major, written only when status >= 0 */,
                            int *status, int *n_inliers, int *n_hypotheses);

/* lo::CRegistration<PointT>::coarse_reg_teaser(target_pts, source_pts, tran_mat, noise_bound, min_inlier_num),
 * cregistration.hpp:664-759: the coarse transform of the global registration with --teaser_on / the default
 * --teaser_based_global_registration_on (test/mulls_reg.cpp:170-186, test/mulls_slam.cpp:532-559): TEASER++'s
 * RobustRegistrationSolver over the correspondences i <-> i with cbar2 = 1, fixed scale, GNC-TLS rotation (100
 * iterations, factor 1.4, cost threshold 0.005) and the maximum clique. Stateless like mulls_coarse_reg_ransac: the
 * batch resident on the context and its grid are left alone. 48-byte rows; only x y z are read, widened to double.
 * Readings of TEASER++ as published (teaser_core.cuh T1-T9 state them in full; none is confirmed against a checkout):
 *   - T1/T2 a pair i < j of correspondences is an edge of the consistency graph when the lengths of its source and
 *     target TIMs (v_j - v_i) differ by at most 2 * noise_bound, each sqrt((x^2 + y^2) + z^2) in double; NaN: no edge
 *   - T3 a maximum clique of that graph (PMC_EXACT), ascending; a clique of at most one vertex is an invalid solution
 *   - T4-T6 GNC-TLS over the chain TIMs of the clique with the noise bound 2 * noise_bound; the rotation inliers are the
 *     chain TIMs with weight >= 0.5, and their count is what min_inlier_num is compared with
 *   - T7 the translation per axis by TLS adaptive voting over the clique's correspondences, ranges noise_bound
 *   - T8 every sum in one fixed order (Eigen's depends on the machine), so the last bits can differ from a TEASER++ build
 *   - T9 among several maximum cliques, the lexicographically smallest ascending index list (PMC leaves the choice to
 *     its threads); equal voting boundaries in ascending signed key order
 * Outputs: *status is -1 when the clouds differ in size or N <= 3 (the reference's refusals: not an error, nothing
 * else written), when the solution is invalid or when the rotation-inlier count is below min_inlier_num; else 1 when
 * the count is >= 2 * min_inlier_num and 0 otherwise (the comparisons are against size_t, so a negative min_inlier_num
 * always gives -1). tran_mat (row-major) is written only when *status >= 0. info (may be NULL) reports the graph's
 * edge count, its largest core number, the clique size, the rotation-inlier count, the GNC iterations (svdRot calls)
 * and the number of search launches.
 * A NULL tran_mat or status, or NULL rows with n > 0: MULLS_E_ARG. N above MULLS_TEASER_MAX_CORR or the context's
 * max_tgt_pts: MULLS_E_CAPACITY. The clique search runs in launches in which each warp processes at most 2^18 64-bit
 * words of the pruned graph; after MULLS_TEASER_SEARCH_LAUNCHES launches without an answer (about 30 s at most on an
 * H100, sized to cover graphs one CPU thread solves in that time) it stops with MULLS_E_CAPACITY: a pathological graph ends with an error, never with a different clique. (TEASER++
 * would keep searching for up to PMC's time limit of 3 600 s.) The context stays usable after any of these. */
#define MULLS_TEASER_MAX_CORR 32768                    /* correspondences: 128 MiB of adjacency */
#define MULLS_TEASER_SEARCH_LAUNCHES 4096              /* the clique search's budget */
typedef struct mulls_teaser_info {
    int64_t n_edges;      /* edges of the consistency graph */
    int max_core;         /* its largest core number (the clique has at most max_core + 1 vertices) */
    int clique_size;      /* the maximum clique's size */
    int rotation_inliers; /* the count compared with min_inlier_num */
    int gnc_iterations;   /* svdRot calls of the GNC-TLS loop */
    int search_launches;  /* launches of the clique search */
    int pad;
} mulls_teaser_info;
int mulls_coarse_reg_teaser(mulls_ctx *ctx, mulls_cloud_view target_pts, mulls_cloud_view source_pts, float noise_bound,
                            int min_inlier_num, double tran_mat[16] /* row-major, written only when status >= 0 */,
                            int *status, mulls_teaser_info *info);

/* lo::CFilter<PointT>::non_max_suppress(cloud_in_out, non_max_radius, kd_tree_already_built = false), cfilter.hpp:1183-1240:
 * the keypoint suppression in front of the NCC matching (test/mulls_reg.cpp:145-149, test/mulls_slam.cpp:462). Stateless
 * like mulls_ncc_correspondences: the batch resident on the context and its grid are left alone. 48-byte rows as for the
 * NCC matching; x y z and the score normal[3] (float 7 of the row) are read. The reference sorts the cloud by score,
 * descending, then walks it: the first point not yet visited is kept and every point within the radius of it is
 * visited; the cloud becomes the kept points in that order. kept_idx[k] (k < *n_kept) receives the input row index of
 * the k-th kept point; the entries past *n_kept are unspecified. Readings:
 *   - fewer than 10 points (:1189-1191): *performed = 0, *n_kept = 0, kept_idx untouched (the reference returns false
 *     and leaves the cloud unsorted); otherwise *performed = 1 (it returns true)
 *   - order: descending score; equal scores keep input order (std::sort leaves it open), +0 and -0 are equal, NaN scores
 *     come after every number, in input order (std::sort with > is undefined on NaN)
 *   - neighbour test: FLANN's float L2_Simple distance flann_l2(kept, p) < r2, r2 = (float)((double)r * r): a negative
 *     radius acts as its absolute value, a zero or NaN radius suppresses nothing
 *   - a point with a non-finite coordinate is within the radius of no point (its FLANN distances are NaN or inf): it is
 *     kept when the walk reaches it and suppresses nothing, as PCL does on a cloud that is not dense
 *   - kd_tree_already_built = true (a tree built on the cloud before the sort) is not served here; the drop-in forwards
 *     it to the reference member
 * A cloud of more than the context's max_tgt_pts points: MULLS_E_CAPACITY. A NULL output, or NULL rows with n > 0:
 * MULLS_E_ARG. */
int mulls_non_max_suppress(mulls_ctx *ctx, mulls_cloud_view cloud, float non_max_radius, int32_t *kept_idx /* [cloud.n] */,
                           size_t *n_kept, int *performed);

/* NDT registration: lo::CRegistration<PointT>::omp_ndt(reg_con, ndt_resolution, use_direct_search, initial_guess,
 * apply_intersection_filter, fitness_score_thre) (cregistration.hpp:945-1021), i.e. koide_reg::NormalDistributionsTransform
 * (include/baseline_reg/ndt_omp_impl.hpp) over koide_reg::VoxelGridCovariance with the DIRECT7 neighbourhood.
 * target = block1->pc_down, source = block2->pc_down, target_bound / source_bound = block1 / block2 ->local_bound
 * (min_x min_y min_z max_x max_y max_z). The readings of the reference are listed in mulls_b200/csrc/ndt_core.cuh
 * (N1-N6, C1-C2); in short:
 *   - prologue: a non-identity initial guess (isIdentity(1e-6)) moves the source in double with a float store and the
 *     intersection box is target_bound with the moved source's bbox, else the two bounds; padded by 2.0; with
 *     apply_intersection_filter both clouds keep the points strictly inside it;
 *   - target leaves of edge ndt_resolution: sums in input order in double, covariance finalised, eigenvalues checked and
 *     inflated to 0.01 of the largest, inverse cast to float; a leaf needs 6 points to be a neighbour; more than
 *     INT32_MAX cells: no leaves;
 *   - the Newton walk with the constants omp_ndt leaves at their defaults (step_size 0.1, transformation_epsilon 0.1,
 *     max_iterations 35, outlier_ratio 0.55): every step is clamp(|newton step|, 0.05, 0.1) along the normalised
 *     direction, so even a converged run may end up to 0.05 (mixed m / rad) past the Newton point;
 *   - fitness = getFitnessScore(): the mean squared distance of the moved (filtered) source to its nearest target,
 *     DBL_MAX when no point counts (empty source or target); code -3 when fitness > fitness_score_thre, else 1;
 *   - Trans1_2 = (double)final_transformation * initial_guess when the guess moved the source, else the former;
 *   - an empty target (for instance after the intersection filter) has no leaves: no point finds a neighbour, the
 *     gradient is zero and the walk ends at once with the identity (the reference is undefined there);
 *   - points with a non-finite coordinate take part in nothing.
 * The walk runs on the host: one evaluation (a few kernels and one 344-byte download) per iteration. The call replaces
 * the resident batch (the fitness search uses the ingest's grid). iterations = nr_iterations_ (at most 37), converged
 * = converged_. trace (may be NULL with trace_cap 0) receives up to trace_cap iterations: the pose vector after the step,
 * the step length, the score at it and whether the direction was reversed. use_direct_search = 0 (KDTREE): MULLS_E_UNSUPPORTED (mulls_omp_ndt_kdtree runs that
 * mode; the drop-in calls the reference member). A NULL output or matrix, NULL rows with n > 0, or ndt_resolution <= 0: MULLS_E_ARG. A target above
 * max_tgt_pts or a source above max_src_pts: MULLS_E_CAPACITY. */
typedef struct mulls_ndt_result {
    double trans[16];  /* Trans1_2, row-major */
    int code;          /* 1, or -3 when fitness > fitness_score_thre */
    int iterations;
    int converged;
    int n_target;      /* points after the intersection filter (finite) */
    int n_source;      /* points after the intersection filter */
    double fitness;
} mulls_ndt_result;
typedef struct mulls_ndt_iter {
    double p[6];  /* x y z roll pitch yaw after the step */
    double step;  /* step length: 0, or in [0.05, 0.1] */
    double score; /* the score at p */
    int reversed; /* 1: the Newton direction pointed downhill and was turned around */
} mulls_ndt_iter;
int mulls_omp_ndt(mulls_ctx *ctx, mulls_cloud_view target, mulls_cloud_view source, float ndt_resolution, int use_direct_search,
                  const double initial_guess[16] /* row-major */, int apply_intersection_filter, float fitness_score_thre,
                  const double target_bound[6], const double source_bound[6], mulls_ndt_result *out, mulls_ndt_iter *trace,
                  int trace_cap);

/* NDT registration with the KDTREE neighbourhood: omp_ndt with use_direct_search = false (test/mulls_slam.cpp with
 * --ndt_searching_method=false), koide_reg::KDTREE, PCL's original NDT neighbourhood. Everything but the neighbourhood
 * is mulls_omp_ndt's: the arguments (without use_direct_search), the prologue, the leaves, the walk, the fitness,
 * Trans1_2, the result and trace types, the codes, the capacities, the refusals and the replaced resident batch. The
 * readings are K1-K5 in mulls_b200/csrc/ndt_core.cuh; in short:
 *   - the searchable cloud holds the float centroid (float sum in input order / nr_points) of every leaf with at least
 *     6 points, in ascending leaf index, including leaves that the eigenvalue check rejects;
 *   - a source point's neighbours are the centroids at float squared distance d2 < (float)(resolution^2) from its float
 *     moved position, in (d2, index) order; each contributes with its leaf's double mean and float inverse covariance,
 *     which is zero for a rejected leaf (it adds -gauss_d1 to the score only);
 *   - no searchable leaf (empty target, every leaf under 6 points, more than INT32_MAX cells): no neighbours.
 * Each evaluation runs a radius search kernel per source point before the derivatives. */
int mulls_omp_ndt_kdtree(mulls_ctx *ctx, mulls_cloud_view target, mulls_cloud_view source, float ndt_resolution,
                         const double initial_guess[16] /* row-major */, int apply_intersection_filter, float fitness_score_thre,
                         const double target_bound[6], const double source_bound[6], mulls_ndt_result *out,
                         mulls_ndt_iter *trace, int trace_cap);

/* A batch of NDT registrations: n_pairs independent mulls_omp_ndt calls in one. ndt_resolution, use_direct_search,
 * apply_intersection_filter and fitness_score_thre are shared by the batch (as the driver's flags are); pair i has its
 * target and source views, initial_guesses[16 i .. 16 i + 15] (row-major), target_bounds[6 i ..] and source_bounds[6 i ..].
 * out[i] and trace[i * trace_cap ..] (up to trace_cap iterations; may be NULL with trace_cap 0) receive what
 * mulls_omp_ndt returns for pair i alone with the same parameters, bit for bit: code, iterations, converged, n_target,
 * n_source, every bit of trans and fitness, every trace row. The pairs' walks run in lockstep on the host: each
 * iteration evaluates every pair whose walk has not ended in one launch and downloads their terms at once.
 * Refusals, with the pair named in mulls_last_error where one pair is the cause; a refused batch writes no result:
 * use_direct_search = 0: MULLS_E_UNSUPPORTED. n_pairs above the context's max_pairs, or a pair whose target exceeds
 * max_tgt_pts or whose source exceeds max_src_pts: MULLS_E_CAPACITY. n_pairs = 0, a NULL array, NULL rows with n > 0
 * or ndt_resolution <= 0: MULLS_E_ARG. The call replaces the resident batch, as mulls_omp_ndt does. */
int mulls_omp_ndt_batch(mulls_ctx *ctx, size_t n_pairs, const mulls_cloud_view *targets, const mulls_cloud_view *sources,
                        float ndt_resolution, int use_direct_search, const double *initial_guesses /* [16 n_pairs] */,
                        int apply_intersection_filter, float fitness_score_thre, const double *target_bounds /* [6 n_pairs] */,
                        const double *source_bounds /* [6 n_pairs] */, mulls_ndt_result *out /* [n_pairs] */,
                        mulls_ndt_iter *trace /* [n_pairs * trace_cap] */, int trace_cap);

/* Voxelized GICP registration: lo::CRegistration<PointT>::omp_gicp(reg_con, max_iter_num, dis_thre_unit, using_voxel_gicp,
 * voxel_size, initial_guess, apply_intersection_filter, fitness_score_thre) (cregistration.hpp:1024-1098) with
 * using_voxel_gicp, i.e. koide_reg::FastVGICP (include/baseline_reg/fast_vgicp_impl.hpp) in its Sophus build.
 * target = block1->pc_down, source = block2->pc_down, target_bound / source_bound = block1 / block2 ->local_bound. The
 * readings of the reference are listed in mulls_b200/csrc/gicp_core.cuh (G1-G7, C1-C3); in short:
 *   - prologue: omp_ndt's (see mulls_omp_ndt), with apply_intersection_filter defaulting to false in omp_gicp; points
 *     with a non-finite coordinate are dropped from both clouds;
 *   - each cloud's covariances from its 20 nearest neighbours (the point itself included), PLANE-regularised; target
 *     voxels of edge voxel_size (coord floor(x / res - 0.5)) with the ADDITIVE means and covariances;
 *   - the Gauss-Newton walk with FastVGICP's defaults (64 iterations, rotation / translation epsilons 2e-3 / 5e-4,
 *     DIRECT1): max_iter_num and dis_thre_unit have no effect in the reference and are not parameters here;
 *   - the walk draws from the process's rand() where the reference does: 3 draws for its start point, 6 more for every
 *     step the LLT solve leaves non-finite (for instance when no source point hits a voxel);
 *   - fitness = getFitnessScore() as mulls_omp_ndt; code -3 when fitness > fitness_score_thre, else 1;
 *     Trans1_2 = (double)final_transformation * initial_guess when the guess moved the source, else the former.
 * The walk runs on the host: one evaluation (two kernels and one 224-byte download) per iteration. The call replaces
 * the resident batch (both clouds go through the ingest). iterations = the Gauss-Newton steps taken (at most 64; the
 * reference's nr_iterations_ + 1), converged = converged_, x0 = the start point (so3, translation). trace (may be NULL
 * with trace_cap 0) receives up to trace_cap iterations: the point after the step, the step, the correspondence count
 * and whether the step was the random fallback. Refused with MULLS_E_UNSUPPORTED: using_voxel_gicp = 0 (the drop-in
 * calls the reference member), fewer than 20 points in either cloud after the prologue (the reference reads
 * uninitialised memory there), a target whose voxel coordinates do not fit 21 bits. A NULL output or matrix, NULL rows
 * with n > 0, or voxel_size <= 0: MULLS_E_ARG. Either cloud above max_tgt_pts: MULLS_E_CAPACITY. */
typedef struct mulls_gicp_result {
    double trans[16];  /* Trans1_2, row-major */
    int code;          /* 1, or -3 when fitness > fitness_score_thre */
    int iterations;
    int converged;
    int n_target;      /* points after the prologue (finite) */
    int n_source;
    double fitness;
    float x0[6];       /* the walk's start point: so3 then translation */
} mulls_gicp_result;
typedef struct mulls_gicp_iter {
    float x[6];        /* so3 then translation after the step */
    float delta[6];    /* the Gauss-Newton step */
    int n_corr;        /* correspondences (source points in a voxel) of the evaluation */
    int random_step;   /* 1: the solve was not finite and the step is Random() * 1e-2 */
} mulls_gicp_iter;
int mulls_omp_gicp(mulls_ctx *ctx, mulls_cloud_view target, mulls_cloud_view source, int using_voxel_gicp, float voxel_size,
                   const double initial_guess[16] /* row-major */, int apply_intersection_filter, float fitness_score_thre,
                   const double target_bound[6], const double source_bound[6], mulls_gicp_result *out, mulls_gicp_iter *trace,
                   int trace_cap);

/* Point-wise GICP registration: lo::CRegistration<PointT>::omp_gicp(reg_con, max_iter_num, dis_thre_unit,
 * using_voxel_gicp = false, voxel_size, initial_guess, apply_intersection_filter, fitness_score_thre)
 * (cregistration.hpp:1024-1098), i.e. koide_reg::GeneralizedIterativeClosestPoint (include/baseline_reg/gicp_omp.h,
 * gicp_omp_impl.hpp) with PCL's BFGS solver: the mode mulls_slam runs with --voxel_gicp_on=false. target = block1->pc_down,
 * source = block2->pc_down, target_bound / source_bound = block1 / block2 ->local_bound. The readings of the reference
 * and of PCL's bfgs.h are listed in mulls_b200/csrc/gicp_pcl_core.cuh (P1-P8, B1-B7, C1-C3); in short:
 *   - prologue, fitness and epilogue: mulls_omp_gicp's; points with a non-finite coordinate are dropped from both clouds;
 *   - each cloud's covariances from its 20 nearest neighbours (the point itself included), summed in double and
 *     rebuilt from the SVD's U with (1, 1, 1e-3);
 *   - up to 200 outer iterations: every source point's exact nearest target, kept within 5 m, with
 *     M = (R C_src R^T + C_tgt)^-1; then PCL's BFGS over (tx ty tz, X Y Z angles) for at most max_iter_num steps
 *     (setMaximumOptimizerIterations(max_iter_num), the one argument of omp_gicp this class reads; with
 *     max_iter_num <= 0 one step is still taken, and a walk that has not finished then ends the loop);
 *   - the loop stops when the transformation changes by less than rotation / translation epsilons 2e-3 / 5e-4, or
 *     ends early, unconverged, when fewer than 4 correspondences are found or the solver did not finish;
 *   - fitness = getFitnessScore(); code -3 when fitness > fitness_score_thre, else 1; Trans1_2 = final * initial_guess
 *     when the guess moved the source, else final.
 * Each outer iteration runs one match kernel, an order-preserving compaction and one 4-byte download; each functor call
 * of the solver runs one evaluation and one tile-sum kernel and downloads 8, 96 or 104 bytes. The solver runs on the
 * host. The call replaces the resident batch (both clouds go through the ingest). The result has mulls_ndt_result's
 * fields: iterations = nr_iterations_, converged = converged_. trace (may be NULL with trace_cap 0) receives up to
 * trace_cap outer iterations. dis_thre_unit and voxel_size have no effect on this class and are not parameters.
 * Refusals: fewer than 20 points in either cloud after the prologue: MULLS_E_UNSUPPORTED (the reference reads
 * covariances it never computed there). A NULL output or matrix, NULL rows with n > 0, or trace_cap > 0 without a
 * trace: MULLS_E_ARG. Either cloud above max_tgt_pts: MULLS_E_CAPACITY. */
typedef mulls_ndt_result mulls_gicp_pcl_result;
typedef struct mulls_gicp_pcl_iter {
    double x[6];       /* the solver's state after the outer iteration: tx ty tz, then the X Y Z angles */
    double delta;      /* the largest epsilon-scaled change of a transformation entry (converged when < 1) */
    int n_corr;        /* correspondences of the iteration */
    int inner_iterations; /* BFGS steps taken (at most max_iter_num, at least 1) */
    int status;        /* the BFGS status the steps ended on: 0 success, 1 no progress, -1 still running (step cap) */
    int evaluations;   /* functor calls of the iteration (operator(), df and fdf together) */
} mulls_gicp_pcl_iter;
int mulls_omp_gicp_pcl(mulls_ctx *ctx, mulls_cloud_view target, mulls_cloud_view source, int max_iter_num,
                       const double initial_guess[16] /* row-major */, int apply_intersection_filter, float fitness_score_thre,
                       const double target_bound[6], const double source_bound[6], mulls_gicp_pcl_result *out,
                       mulls_gicp_pcl_iter *trace, int trace_cap);

/* The wire format the library ships host clouds in when the "host_pack" tunable is on (csrc/host_pack.h): the 28 of the
 * 48 bytes of a pcl::PointXYZINormal row (utility.hpp:40) that the path reads, repacked on the host cores into pinned
 * staging before the DMA. format 1: [n x (x y z intensity)] [n x (nx ny nz)]; format 2 (motion undistortion, which also
 * reads `curvature`): [n x (x y z intensity)] [n x (nx ny nz curvature)]. `out` (16-byte aligned) receives
 * 4n + 3n floats (format 1) or 8n floats (format 2). Exposed for callers that keep their clouds packed, and for tests. */
int mulls_pack_rows(const float *aos48, size_t n, int format, float *out);

/* Scans in, poses out — the reference's DataIo on the two sides of the hot path (SURVEY 8f rank 3; csrc/scan_io.h, host
 * code only). A scan is read straight into pcl::PointXYZINormal rows (48 bytes), i.e. into the buffer every registration
 * and front-end entry point above takes; with mulls_host_alloc that buffer is pinned and crosses PCIe as it is.
 *   mulls_scan_probe   rows the file holds (KITTI .bin: one more than its records — the reference's read loop appends a
 *                      default point at end-of-file, include/common/dataio.hpp:366-373)
 *   mulls_scan_read    DataIo::read_pc_cloud_block (dataio.hpp:1732-1756) over read_pcd_file (:279-287; PCD v0.7, DATA
 *                      ascii | binary, float32 fields x y z intensity normal_x normal_y normal_z curvature, others are
 *                      ignored; binary_compressed: MULLS_E_UNSUPPORTED) and read_bin_file (:357-377; by the .bin
 *                      extension); local_bound (may be NULL) = CloudUtility::get_cloud_bbx (utility.hpp:817-848);
 *                      normalize_intensity != 0: intensity rescaled to 0..255 in float (:1738-1750)
 *   mulls_pose_write   DataIo::write_lo_pose_overwrite / write_lo_pose_append (dataio.hpp:1896-1926): the upper 3 x 4 of a
 *                      row-major 4 x 4 pose, setprecision(8), one line
 *   mulls_host_alloc / mulls_host_free   pinned host memory (cudaHostAlloc); NULL without a CUDA device */
int mulls_scan_probe(const char *path, size_t *n_points);
int mulls_scan_read(const char *path, float *rows48, size_t capacity_points, size_t *n_points, double local_bound[6],
                    int normalize_intensity);
int mulls_pose_write(const char *path, const double pose[16], int overwrite);
void *mulls_host_alloc(size_t bytes);
void mulls_host_free(void *p);

/* Runtime tunables (integers). Returns MULLS_E_ARG for any other name.
 *   "use_graph"     1 (default): the iteration loop as one CUDA graph launch, or as one cooperative kernel for batches
 *                   whose chunks all find a co-resident block; 0: the host launch loop (per-kernel timing events)
 *   "host_pack"     repack host clouds to the packed wire format on the host cores before the copy:
 *                   0 never, 1 always, 2 (default) when a call ships at least 2^18 points
 *   "pack_threads"  the process-wide packing pool has at least n workers (n <= 0: MULLS_PACK_THREADS or cores/16, 2..8) */
int mulls_set_tunable(mulls_ctx *ctx, const char *name, int value);

#ifdef __cplusplus
}
#endif
#endif /* MULLS_B200_ABI_H */
