// Non-maximum suppression of keypoints: lo::CFilter<PointT>::non_max_suppress (include/common/cfilter.hpp:1183-1240 in
// place, :1243-1312 into cloud_out). One implementation for every caller: classify_nground_pts runs it on its four class
// clouds (k_cls_* in kernels_classify.cuh), mulls_non_max_suppress on one caller cloud. The reference is a greedy walk in
// score order: the first point not yet visited is kept and every point within the radius of it is visited. Here that
// walk runs 1024 points at a time in one block per cloud:
//   (1) a chunk point within the radius of a point kept in an earlier chunk is suppressed. The kept points are found
//       through a hash of cells whose edge is at least the radius (NmsArgs::hash): only the 27 cells around the point
//       are probed. A cloud of at most one chunk never gets here and has no index;
//   (2) every open chunk point builds the bit mask of the earlier chunk points within the radius;
//   (3) monotone rounds: a point is kept once every earlier near point is suppressed, suppressed once one is kept;
//   (4) the kept points of the chunk are appended in order and enter the hash.
// The neighbour test is FLANN's L2_Simple float distance, flann_l2(kept, p) < r2 with r2 = (float)((double)r * r).
#pragma once
#include "device_math.cuh"
#include "grid_key.cuh"
#include "kernels_map.cuh"

namespace mulls {

constexpr int kNmsBlock = kMapBlock; // 1024: map_tile_slot is written for this block size
constexpr int kNmsMaxClouds = 4;
constexpr int kNmsCellClamp = 1 << 20; // cell coordinates are clamped to [-2^20, 2^20): 21 bits per axis in the key
constexpr uint32_t kNmsMaxPoints = 1u << 29; // the position field of the sort key

// one slot of the cell hash: the packed cell coordinates (~0: empty) and the last kept point inserted in that cell
struct NmsSlot {
    unsigned long long key;
    int head;
    int pad;
};

struct NmsArgs {
    int n_clouds;            // 1..4, one block each in k_nms_select
    uint32_t on_mask;        // bit c: the caller asks for NMS on cloud c
    const uint32_t *n;       // [n_clouds] device: points of each cloud
    uint32_t *n_kept;        // [n_clouds] device: written for the clouds that ran
    uint32_t *ran;           // [n_clouds] device: 1 when the cloud had at least 10 points and was sorted, else 0
    float r2;                // squared radius
    double inv_cell;         // 1 / cell edge of the hash (used only with hash)
    const float4 *in[kNmsMaxClouds]; // 3 float4 per point; the score is row[1].w (normal[3])
    float4 *sorted[kNmsMaxClouds];   // the rows in score order
    float4 *kept_rows[kNmsMaxClouds]; // or null: the kept rows, in order
    int32_t *kept_idx[kNmsMaxClouds]; // or null: the input positions of the kept rows, in order
    float4 *sel[kNmsMaxClouds];       // positions of the kept points (as many as the cloud's points)
    NmsSlot *hash[kNmsMaxClouds];     // null when every cloud fits one chunk or r2 > 0 fails; else hash_mask + 1 slots
    int32_t *next[kNmsMaxClouds];     // the cell lists: kept point -> the one inserted before it in its cell
    uint32_t hash_mask;
    uint32_t total;                   // sort key slots, at least the points of the clouds together
    uint64_t *keys_a, *keys_b;        // [total]
    uint32_t *order;                  // [total] input position of each sorted point
};

__device__ __forceinline__ bool nms_active(const NmsArgs &A, int c) { return ((A.on_mask >> c) & 1u) && A.n[c] >= 10; }
__device__ __forceinline__ uint32_t nms_offset(const NmsArgs &A, int c) {
    uint32_t off = 0;
    for (int k = 0; k < c; ++k)
        if (nms_active(A, k)) off += A.n[k];
    return off;
}

// 32 bits that sort ascending as the score descends: +0 and -0 are one key, NaN comes after every number
__device__ __forceinline__ uint32_t nms_score_key(float s) {
    if (s != s) return 0xffffffffu;
    if (s == 0.f) s = 0.f;
    return ~((uint32_t)float_to_ordered(s) ^ 0x80000000u);
}

// cell of one coordinate. floor of a correctly rounded product is monotone in x, and the clamp is monotone and moves no
// two values further apart: two coordinates less than one cell edge apart get cells at most one apart (DESIGN §16).
__device__ __forceinline__ int nms_cell(float x, double inv_cell) {
    const double v = floor((double)x * inv_cell);
    return (int)fmin(fmax(v, (double)-kNmsCellClamp), (double)(kNmsCellClamp - 1));
}
__device__ __forceinline__ unsigned long long nms_cell_key(int cx, int cy, int cz) {
    return ((unsigned long long)(cx + kNmsCellClamp) << 42) | ((unsigned long long)(cy + kNmsCellClamp) << 21) |
           (unsigned long long)(cz + kNmsCellClamp);
}
__device__ __forceinline__ uint32_t nms_hash(unsigned long long k) { // splitmix64 finalizer
    k ^= k >> 30;
    k *= 0xbf58476d1ce4e5b9ull;
    k ^= k >> 27;
    k *= 0x94d049bb133111ebull;
    k ^= k >> 31;
    return (uint32_t)k;
}
__device__ __forceinline__ bool nms_finite(float4 p) { return isfinite(p.x) && isfinite(p.y) && isfinite(p.z); }

// sort key of a cloud entry: cloud | score key | position in the cloud. std::sort is not stable: equal scores keep
// their input order here and in the CPU restatement.
__global__ void __launch_bounds__(256) k_nms_keys(NmsArgs A) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const int c = blockIdx.y;
    if (!nms_active(A, c) || t >= A.n[c]) return;
    const float score = A.in[c][3 * (size_t)t + 1].w;
    A.keys_a[nms_offset(A, c) + t] = ((uint64_t)c << 61) | ((uint64_t)nms_score_key(score) << 29) | (uint64_t)t;
}

__global__ void __launch_bounds__(256) k_nms_gather(NmsArgs A) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= A.total) return;
    const uint64_t key = A.keys_b[r];
    if (key == ~0ull) return;
    const int c = (int)(key >> 61);
    const uint32_t slot = (uint32_t)(key & (kNmsMaxPoints - 1u));
    const float4 *in = A.in[c] + 3 * (size_t)slot;
    float4 *o = A.sorted[c] + 3 * (size_t)(r - nms_offset(A, c));
    o[0] = in[0], o[1] = in[1], o[2] = in[2];
    A.order[r] = slot;
}

// one block per cloud: the greedy walk in score order, 1024 points at a time (see the head of this file). The rounds of
// (3) are pure bit tests against two shared masks (selected / suppressed) that only ever gain bits.
__global__ void __launch_bounds__(kNmsBlock) k_nms_select(NmsArgs A) {
    const int c = blockIdx.x;
    __shared__ uint32_t s_warp[kNmsBlock / 32];
    __shared__ uint32_t s_total;
    __shared__ float s_x[kNmsBlock], s_y[kNmsBlock], s_z[kNmsBlock];
    __shared__ uint32_t s_sel[kNmsBlock / 32], s_sup[kNmsBlock / 32];
    if (!nms_active(A, c)) {
        if (threadIdx.x == 0) A.ran[c] = 0; // n_kept stays what the caller left
        return;
    }
    const uint32_t n = A.n[c];
    const float r2 = A.r2;
    const float4 *pts = A.sorted[c];
    const uint32_t *order = A.order + nms_offset(A, c);
    float4 *sel = A.sel[c];
    NmsSlot *hash = A.hash[c];
    int32_t *next = A.next[c];
    const uint32_t tid = threadIdx.x, myw = tid >> 5, mybit = 1u << (tid & 31);
    if (tid == 0) s_total = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += kNmsBlock) {
        const uint32_t i = base + tid;
        const bool valid = i < n;
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
        if (valid) p = pts[3 * (size_t)i];
        s_x[tid] = p.x, s_y[tid] = p.y, s_z[tid] = p.z;
        if (tid < kNmsBlock / 32) s_sel[tid] = 0, s_sup[tid] = 0;
        // (1) against the points kept in the earlier chunks, through the cells around p. A point with a non-finite
        //     coordinate is within the radius of no point.
        bool open = valid;
        if (valid && s_total > 0 && hash && nms_finite(p)) {
            const int cx = nms_cell(p.x, A.inv_cell), cy = nms_cell(p.y, A.inv_cell), cz = nms_cell(p.z, A.inv_cell);
            for (int dz = -1; dz <= 1 && open; ++dz)
                for (int dy = -1; dy <= 1 && open; ++dy)
                    for (int dx = -1; dx <= 1 && open; ++dx) {
                        const int x = cx + dx, y = cy + dy, z = cz + dz;
                        if (x < -kNmsCellClamp || y < -kNmsCellClamp || z < -kNmsCellClamp || x >= kNmsCellClamp ||
                            y >= kNmsCellClamp || z >= kNmsCellClamp)
                            continue;
                        const unsigned long long key = nms_cell_key(x, y, z);
                        uint32_t h = nms_hash(key) & A.hash_mask;
                        int t = -1;
                        while (true) {
                            const unsigned long long k = hash[h].key;
                            if (k == key) {
                                t = hash[h].head;
                                break;
                            }
                            if (k == ~0ull) break;
                            h = (h + 1) & A.hash_mask;
                        }
                        for (; t >= 0; t = next[t]) {
                            const float4 q = sel[t];
                            if (flann_l2(q.x, q.y, q.z, p.x, p.y, p.z) < r2) {
                                open = false;
                                break;
                            }
                        }
                    }
        }
        __syncthreads();
        if (!open) atomicOr(&s_sup[myw], mybit);
        // (2) near mask over the earlier points of the chunk
        uint32_t near[kNmsBlock / 32];
#pragma unroll
        for (int w = 0; w < kNmsBlock / 32; ++w) {
            uint32_t mk = 0;
            if (open && (uint32_t)(w * 32) < tid) {
                const uint32_t lim = min(32u, tid - (uint32_t)(w * 32));
                for (uint32_t b = 0; b < lim; ++b) {
                    const uint32_t t = (uint32_t)(w * 32) + b;
                    if (flann_l2(s_x[t], s_y[t], s_z[t], p.x, p.y, p.z) < r2) mk |= 1u << b;
                }
            }
            near[w] = mk;
        }
        __syncthreads();
        // (3) a point is selected once every earlier point within the radius is suppressed
        while (true) {
            int pending = 0;
            if (open) {
                bool hit = false, blocked = false;
#pragma unroll
                for (int w = 0; w < kNmsBlock / 32; ++w) {
                    const uint32_t nm = near[w];
                    if (nm) {
                        const uint32_t se = ((volatile uint32_t *)s_sel)[w];
                        const uint32_t su = ((volatile uint32_t *)s_sup)[w];
                        if (nm & se) hit = true;
                        if (nm & ~(se | su)) blocked = true;
                    }
                }
                if (hit) {
                    atomicOr(&s_sup[myw], mybit);
                    open = false;
                } else if (!blocked) {
                    atomicOr(&s_sel[myw], mybit);
                    open = false;
                } else {
                    pending = 1;
                }
            }
            if (!__syncthreads_or(pending)) break;
        }
        // (4) append the chunk's selected points, in order, and put them in the cell hash
        const bool keep = valid && (s_sel[myw] & mybit);
        const uint32_t slot = map_tile_slot(keep, s_warp, &s_total);
        if (keep) {
            if (A.kept_rows[c]) {
                const float4 *r = pts + 3 * (size_t)i;
                float4 *o = A.kept_rows[c] + 3 * (size_t)slot;
                o[0] = r[0], o[1] = r[1], o[2] = r[2];
            }
            if (A.kept_idx[c]) A.kept_idx[c][slot] = (int32_t)order[i];
            sel[slot] = p;
            if (hash && nms_finite(p)) {
                const unsigned long long key =
                    nms_cell_key(nms_cell(p.x, A.inv_cell), nms_cell(p.y, A.inv_cell), nms_cell(p.z, A.inv_cell));
                uint32_t h = nms_hash(key) & A.hash_mask;
                while (true) {
                    const unsigned long long old = atomicCAS(&hash[h].key, ~0ull, key);
                    if (old == ~0ull || old == key) break;
                    h = (h + 1) & A.hash_mask;
                }
                next[slot] = atomicExch(&hash[h].head, (int)slot);
            }
        }
        __syncthreads();
    }
    if (tid == 0) {
        A.n_kept[c] = s_total;
        A.ran[c] = 1;
    }
}

} // namespace mulls
