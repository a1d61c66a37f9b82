// Device-resident local map: lo::MapManager::update_local_map (src/map_manager.cpp:17-145).
// The map is a few 10^4 points (max_num_pts 8000-20000 + one scan's features), so the update is latency work, not
// bandwidth work: one 1024-thread block per feature class walks its cloud in order (order-preserving block
// compaction, no atomics on the data path, bit-reproducible), and two launches cover the whole function. The only
// cross-class dependency — the sampling budget, which needs the five class sizes after the radius crop — sits
// between the two launches.
#pragma once
#include "device_math.cuh"
#include "device_types.cuh"
#include "kernels_ingest.cuh"
#include "kernels_pca.cuh"

namespace mulls {

constexpr int kMapBlock = 1024;
constexpr uint32_t kMapCloudId = 12; // sampling-key cloud ids 12..17 (0..11 are the registration's clouds)

struct MapState {
    uint32_t n_mid[kNumClasses];      // after append + transform + radius crop
    uint32_t n_out[kNumClasses];      // after the budgeted sampling
    uint32_t n_appended[kNumClasses]; // scan points appended (dynamic removal applied)
    float lb[kNumClasses][6];         // per-class bbox in the map frame (min xyz, max xyz)
    float gb[kNumClasses][6];         // per-class bbox in the world frame
};

struct MapArgs {
    const float4 *old_pts[kNumClasses];
    const float4 *scan_pts[kNumClasses];
    const uint8_t *scan_drop[kNumClasses]; // 1 = removed by the map-based dynamic filter (may be null)
    float4 *mid[kNumClasses];
    float4 *out[kNumClasses];
    uint32_t n_old[kNumClasses];
    uint32_t n_scan[kNumClasses];
    int used[kNumClasses];
    double T[16];    // tran_target_map: old map frame -> new (scan) frame
    double Tinv[16]; // its inverse: scan frame -> old map frame
    double pose[16]; // the scan's pose_lo (world frame)
    double radius;   // (double)local_map_radius
    int max_num_pts;
    int kept_vertex_num;
    uint32_t seed;
    MapState *state;
};

struct MapRow {
    float4 a, b, c; // x y z 1 | nx ny nz 0 | intensity curvature 0 0
};

// pcl::transformPointCloudWithNormals (double math, float store), as load_input_point (kernels_ingest.cuh)
__device__ __forceinline__ void map_transform(MapRow &r, const double *t) {
    const double px = r.a.x, py = r.a.y, pz = r.a.z, qx = r.b.x, qy = r.b.y, qz = r.b.z;
    r.a.x = (float)(t[0] * px + t[1] * py + t[2] * pz + t[3]);
    r.a.y = (float)(t[4] * px + t[5] * py + t[6] * pz + t[7]);
    r.a.z = (float)(t[8] * px + t[9] * py + t[10] * pz + t[11]);
    r.b.x = (float)(t[0] * qx + t[1] * qy + t[2] * qz);
    r.b.y = (float)(t[4] * qx + t[5] * qy + t[6] * qz);
    r.b.z = (float)(t[8] * qx + t[9] * qy + t[10] * qz);
}

// Order-preserving compaction step of one 1024-point tile: returns the output slot of this thread's row (valid only
// when `keep`) and advances the block's running total. All threads of the block must call it.
__device__ __forceinline__ uint32_t map_tile_slot(bool keep, uint32_t *s_warp, uint32_t *s_total) {
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[warp] = (uint32_t)__popc(ballot);
    __syncthreads();
    uint32_t before = 0, all = 0;
    for (unsigned w = 0; w < (unsigned)(kMapBlock / 32); ++w) {
        const uint32_t v = s_warp[w];
        if (w < warp) before += v;
        all += v;
    }
    const uint32_t slot = *s_total + before + (uint32_t)__popc(ballot & ((1u << lane) - 1u));
    __syncthreads();
    if (threadIdx.x == 0) *s_total += all;
    __syncthreads();
    return slot;
}

// ---- k_map_dynamic: map_scan_feature_pts_distance_removal (map_manager.cpp:221-258) for pillar, beam, facade.
//      One warp per scan point; the reference's kd-tree query is an exact unbounded 1-NN in the cloud the preceding
//      registration built block1's tree on (the intersection-filtered target clone, cregistration.hpp:1209-1232) —
//      still resident as the Morton-sorted target slices of that run. These clouds are a few thousand points:
//      a flat scan by the warp beats any tree walk.
struct MapDynArgs {
    const float4 *scan_pts[3];
    uint8_t *drop[3];
    uint32_t n_scan[3];
    int cls[3];
    double Tinv[16];
    float center_radius, dist_min, dist_max, near_thre;
};

__global__ void __launch_bounds__(256) k_map_dynamic(DeviceArrays A, MapDynArgs D) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31;
    uint32_t q = w;
    int k = 0;
    while (k < 3 && q >= D.n_scan[k]) {
        q -= D.n_scan[k];
        ++k;
    }
    if (k >= 3) return;
    if (D.n_scan[k] <= 10) return; // :224
    const int c = D.cls[k];
    const PairConst &pc = A.pc[0];
    const uint32_t n_tree = pc.used[c] ? (uint32_t)A.ps[0].n_tgt[c] : 0u;
    if (n_tree == 0) return; // no tree was built for this class: the cloud stays as it is
    MapRow r;
    r.a = D.scan_pts[k][3 * (size_t)q];
    r.b = make_float4(0.f, 0.f, 0.f, 0.f);
    map_transform(r, D.Tinv);
    const float px = r.a.x, py = r.a.y, pz = r.a.z;
    if (px * px + py * py > D.center_radius * D.center_radius) return; // kept without a query
    const float4 *tp = A.tgt_pos + pc.tgt_base[c];
    float best = INFINITY;
    for (uint32_t j = lane; j < n_tree; j += 32) {
        const float4 t = __ldg(&tp[j]);
        best = fminf(best, flann_l2(px, py, pz, t.x, t.y, t.z));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = fminf(best, __shfl_xor_sync(0xffffffffu, best, o));
    const bool keep = (best > D.near_thre * D.near_thre && best < D.dist_min * D.dist_min) || best > D.dist_max * D.dist_max;
    if (lane == 0 && !keep) D.drop[k][q] = 1;
}

// ---- k_map_merge: one block per class. append_feature (utility.hpp:438-470) + transform_feature (:495-516) +
//      dist_filter (cfilter.hpp:838-873), in order: old map points, then the scan's.
__global__ void __launch_bounds__(kMapBlock) k_map_merge(MapArgs M) {
    const int c = blockIdx.x;
    __shared__ uint32_t s_warp[kMapBlock / 32];
    __shared__ uint32_t s_total;
    __shared__ uint32_t s_app;
    if (threadIdx.x == 0) s_total = 0, s_app = 0;
    __syncthreads();
    const uint32_t n_old = M.n_old[c];
    const uint32_t n_scan = (c == MULLS_VERTEX || M.used[c]) ? M.n_scan[c] : 0u;
    const uint32_t total = n_old + n_scan;
    for (uint32_t tile = 0; tile < total; tile += kMapBlock) {
        const uint32_t i = tile + threadIdx.x;
        bool keep = false;
        MapRow r;
        if (i < total) {
            bool present = true;
            if (i < n_old) {
                const float4 *p = M.old_pts[c] + 3 * (size_t)i;
                r.a = p[0], r.b = p[1], r.c = p[2];
            } else {
                const uint32_t k = i - n_old;
                const float4 *p = M.scan_pts[c] + 3 * (size_t)k;
                r.a = p[0], r.b = p[1], r.c = p[2];
                if (M.scan_drop[c] && M.scan_drop[c][k]) present = false;
                // the scan's down clouds were moved into the old map frame first (map_manager.cpp:32); pc_vertex
                // has no down cloud and is appended as it is
                if (present && c != MULLS_VERTEX) map_transform(r, M.Tinv);
                if (present) atomicAdd(&s_app, 1u);
            }
            if (present) {
                map_transform(r, M.T);
                const double dis_square = (double)(r.a.x * r.a.x + r.a.y * r.a.y);
                keep = dis_square < M.radius * M.radius && (double)r.a.z < 1.7976931348623157e308 &&
                       (double)r.a.z > -1.7976931348623157e308;
            }
        }
        const uint32_t slot = map_tile_slot(keep, s_warp, &s_total);
        if (keep) {
            float4 *o = M.mid[c] + 3 * (size_t)slot;
            o[0] = make_float4(r.a.x, r.a.y, r.a.z, 1.0f);
            o[1] = make_float4(r.b.x, r.b.y, r.b.z, 0.0f);
            o[2] = make_float4(r.c.x, r.c.y, 0.0f, 0.0f);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        M.state->n_mid[c] = s_total;
        M.state->n_appended[c] = s_app;
    }
}

// ---- k_map_sample: one block per class. Budget (map_manager.cpp:69-78), random_downsample_pcl (cfilter.hpp:606-628,
//      here: keep the k smallest splitmix64 keys, radix select in shared memory), bounding boxes (:88-93).
__global__ void __launch_bounds__(kMapBlock) k_map_sample(MapArgs M) {
    const int c = blockIdx.x;
    __shared__ uint32_t s_warp[kMapBlock / 32];
    __shared__ uint32_t s_total;
    __shared__ uint32_t s_hist[256];
    __shared__ uint64_t s_prefix;
    __shared__ uint32_t s_rank;
    __shared__ float s_red[kMapBlock / 32][12];
    const uint32_t n = M.state->n_mid[c];
    int current = 0;
    for (int k = 0; k < 5; ++k) current += (int)M.state->n_mid[k];
    long long keep_num = -1; // < 0: cloud untouched
    if (c == MULLS_VERTEX)
        keep_num = M.kept_vertex_num;
    else if (current > 0)
        keep_num = (long long)(int)(1.0 * (double)M.max_num_pts / (double)current * (double)n + 1.0);
    const bool sample = keep_num >= 0 && (long long)n > keep_num; // size() <= keep_number: untouched
    const uint32_t cloud = kMapCloudId + (uint32_t)c;
    if (threadIdx.x == 0) s_total = 0, s_prefix = 0, s_rank = (uint32_t)(sample ? keep_num : 0);
    __syncthreads();
    if (sample && keep_num > 0) {
        for (int pass = 0; pass < 8; ++pass) {
            if (threadIdx.x < 256) s_hist[threadIdx.x] = 0;
            __syncthreads();
            const int shift = 56 - 8 * pass;
            const uint64_t prefix = s_prefix;
            for (uint32_t i = threadIdx.x; i < n; i += kMapBlock) {
                const uint64_t key = sample_key(M.seed, cloud, i);
                if (pass == 0 || (key >> (shift + 8)) == (prefix >> (shift + 8))) atomicAdd(&s_hist[(key >> shift) & 0xff], 1u);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                uint32_t cum = 0;
                const uint32_t rank = s_rank;
                int d = 0;
                for (; d < 256; ++d) {
                    if (cum + s_hist[d] >= rank) break;
                    cum += s_hist[d];
                }
                s_prefix = prefix | ((uint64_t)d << shift);
                s_rank = rank - cum;
            }
            __syncthreads();
        }
    }
    const uint64_t thr = s_prefix;
    float mn[6] = {FLT_MAX, FLT_MAX, FLT_MAX, FLT_MAX, FLT_MAX, FLT_MAX};    // local xyz, world xyz
    float mx[6] = {-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (uint32_t tile = 0; tile < n; tile += kMapBlock) {
        const uint32_t i = tile + threadIdx.x;
        bool keep = false;
        MapRow r;
        if (i < n) {
            keep = !sample || (keep_num > 0 && sample_key(M.seed, cloud, i) <= thr);
            if (keep) {
                const float4 *p = M.mid[c] + 3 * (size_t)i;
                r.a = p[0], r.b = p[1], r.c = p[2];
            }
        }
        const uint32_t slot = map_tile_slot(keep, s_warp, &s_total);
        if (keep) {
            float4 *o = M.out[c] + 3 * (size_t)slot;
            o[0] = r.a, o[1] = r.b, o[2] = r.c;
            const double px = r.a.x, py = r.a.y, pz = r.a.z;
            const double *t = M.pose;
            const float w[3] = {(float)(t[0] * px + t[1] * py + t[2] * pz + t[3]), (float)(t[4] * px + t[5] * py + t[6] * pz + t[7]),
                                (float)(t[8] * px + t[9] * py + t[10] * pz + t[11])};
            const float l[3] = {r.a.x, r.a.y, r.a.z};
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                mn[d] = fminf(mn[d], l[d]), mx[d] = fmaxf(mx[d], l[d]);
                mn[3 + d] = fminf(mn[3 + d], w[d]), mx[3 + d] = fmaxf(mx[3 + d], w[d]);
            }
        }
    }
#pragma unroll
    for (int d = 0; d < 6; ++d)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[d] = fminf(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
            mx[d] = fmaxf(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
        }
    if ((threadIdx.x & 31) == 0)
        for (int d = 0; d < 6; ++d) s_red[threadIdx.x >> 5][d] = mn[d], s_red[threadIdx.x >> 5][6 + d] = mx[d];
    __syncthreads();
    if (threadIdx.x < 12) {
        const int d = threadIdx.x;
        float v = s_red[0][d];
        for (int w = 1; w < kMapBlock / 32; ++w) v = (d < 6) ? fminf(v, s_red[w][d]) : fmaxf(v, s_red[w][d]);
        // s_red rows: [min local xyz, min world xyz, max local xyz, max world xyz]
        const int side = d / 6, comp = d % 6; // comp 0..2 local, 3..5 world
        if (comp < 3)
            M.state->lb[c][3 * side + comp] = v;
        else
            M.state->gb[c][3 * side + comp - 3] = v;
    }
    if (threadIdx.x == 0) M.state->n_out[c] = s_total;
}

// ---- k_map_revector: MapManager::update_cloud_vectors (map_manager.cpp:260-295) after the PCA pass. One block;
//      keeps, in order, the points with >= k_min neighbours and linearity (l1-l2)/l1 > min_linearity whose new
//      principal direction is steep (pillar: |z| > sin_high) or flat (beam: |z| < sin_low); the direction goes to
//      normal_*, the linearity to `curvature` (:283).
__global__ void __launch_bounds__(kMapBlock) k_map_revector(const float4 *in, uint32_t n, PcaArgs F, int k_min, float sin_low,
                                                            float sin_high, float min_linearity, float4 *out, uint32_t *n_out) {
    __shared__ uint32_t s_warp[kMapBlock / 32];
    __shared__ uint32_t s_total;
    if (threadIdx.x == 0) s_total = 0;
    __syncthreads();
    for (uint32_t tile = 0; tile < n; tile += kMapBlock) {
        const uint32_t i = tile + threadIdx.x;
        bool keep = false;
        MapRow r;
        if (i < n && F.pt_num[i] >= k_min) {
            // pca_feature_t keeps the eigenvalues and the ratios as double (pca.hpp:23-44, :425)
            const double l1 = F.eigenvalues[3 * (size_t)i], l2 = F.eigenvalues[3 * (size_t)i + 1];
            // identical neighbours give l1 == 0 and a NaN here whose bits differ from the x86 build's; it cannot reach
            // an output, because a NaN fails the `>` below (the classification writes its ratios: kernels_classify.cuh)
            const double linear_2 = (l1 - l2) / l1;
            const float pz = fabsf(F.principal[3 * (size_t)i + 2]);
            if (linear_2 > (double)min_linearity && (pz > sin_high || pz < sin_low)) {
                keep = true;
                const float4 *p = in + 3 * (size_t)i;
                r.a = p[0], r.c = p[2];
                r.b = make_float4(F.principal[3 * (size_t)i], F.principal[3 * (size_t)i + 1], F.principal[3 * (size_t)i + 2], 0.0f);
                r.c.y = (float)linear_2;
            }
        }
        const uint32_t slot = map_tile_slot(keep, s_warp, &s_total);
        if (keep) {
            float4 *o = out + 3 * (size_t)slot;
            o[0] = r.a, o[1] = r.b, o[2] = r.c;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) *n_out = s_total;
}

} // namespace mulls
