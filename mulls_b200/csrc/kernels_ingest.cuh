// Ingest phase: what mm_lls_icp does before its iteration loop (cregistration.hpp:1180-1232) —
// clone + apply initial guess, intersection filter, and (instead of six FLANN kd-trees) a spatial
// sort of every cloud plus a multi-level hashed grid over each target class.
#pragma once
#include "device_math.cuh"
#include "device_types.cuh"

namespace mulls {

// ---- load_input_point: input point `local` of segment `seg`, read from whichever of the three layouts is behind
//      in_ptr (block-uniform): the caller's 48-byte rows, or the host-packed wire formats (host_pack.h). A source point
//      gets the motion undistortion and the initial guess (double math, float store,
//      pcl::transformPointCloudWithNormals semantics). The bbox pass, k_make_keys and the last sort pass each recompute the point
//      here instead of reading a staged copy: one function, so every recomputation gives the same bits.
// kUndistort = false: the instantiation for batches in which no pair asks for motion undistortion (no slerp code).
// kNormals = false: position only (nrm untouched); the position does not depend on the normal, so its bits are the same.
template <bool kUndistort, bool kNormals>
__device__ __forceinline__ void load_input_point(const PairConst &pc, uint32_t seg, uint32_t local, float4 &pos, float4 &nrm) {
    const bool is_src = seg >= kNumClasses;
    const int cls = seg % kNumClasses;
    const bool undistort = kUndistort && is_src && pc.undistort && cls != MULLS_VERTEX;
    float x, y, z, intensity = 0.0f, curvature = 0.0f;
    float nx = 0.0f, ny = 0.0f, nz = 0.0f;
    const uint32_t fmt = pc.in_fmt[seg];
    if (fmt == 0u) {
        const float4 *in = pc.in_ptr[seg] + 3 * (size_t)local;
        const float4 a = in[0]; // x y z _
        x = a.x, y = a.y, z = a.z;
        if (kNormals) {
            const float4 b = in[1]; // nx ny nz _
            const float4 c = in[2]; // intensity curvature _ _
            nx = b.x, ny = b.y, nz = b.z;
            intensity = c.x, curvature = c.y;
        } else if (undistort) {
            curvature = reinterpret_cast<const float *>(in + 2)[1];
        }
    } else {
        const float4 *in = pc.in_ptr[seg];
        const float4 a = in[local]; // x y z intensity
        x = a.x, y = a.y, z = a.z, intensity = a.w;
        if (fmt == 1u) {
            if (kNormals) {
                const float *nr = reinterpret_cast<const float *>(in + pc.in_n[seg]) + 3 * (size_t)local;
                nx = nr[0], ny = nr[1], nz = nr[2];
            }
        } else if (kNormals) {
            const float4 b = in[(size_t)pc.in_n[seg] + local]; // nx ny nz curvature
            nx = b.x, ny = b.y, nz = b.z, curvature = b.w;
        } else if (undistort) {
            curvature = in[(size_t)pc.in_n[seg] + local].w;
        }
    }
    if (is_src) {
        const double *t = pc.init;
        int n_apply = 1;
        if (kUndistort && pc.undistort) {
            if (cls == MULLS_VERTEX) {
                n_apply = 2; // not undistorted and not re-cloned: the initial guess lands twice (reference behaviour)
            } else { // curvature: the timestamp ratio of the point inside its frame
                slerp_compensate(pc.ud_q, pc.ud_t, pc.ud_linear, pc.ud_neg, pc.ud_theta, pc.ud_sin_theta, 0.0f, curvature, x, y, z);
            }
        }
        for (int rep = 0; rep < n_apply; ++rep) {
            const double px = x, py = y, pz = z;
            x = (float)(t[0] * px + t[1] * py + t[2] * pz + t[3]);
            y = (float)(t[4] * px + t[5] * py + t[6] * pz + t[7]);
            z = (float)(t[8] * px + t[9] * py + t[10] * pz + t[11]);
            if (kNormals) {
                const double qx = nx, qy = ny, qz = nz;
                nx = (float)(t[0] * qx + t[1] * qy + t[2] * qz);
                ny = (float)(t[4] * qx + t[5] * qy + t[6] * qz);
                nz = (float)(t[8] * qx + t[9] * qy + t[10] * qz);
            }
        }
    }
    pos = make_float4(x, y, z, intensity);
    if (kNormals) nrm = make_float4(nx, ny, nz, __int_as_float((int)local));
}

// a point whose three coordinates are finite: kFiniteOnly ingests (mulls_sor_filter) leave every other point out of the
// grid's extent and out of the grid
__device__ __forceinline__ bool finite_xyz(const float4 &p) { return isfinite(p.x) && isfinite(p.y) && isfinite(p.z); }

// ---- k_ingest_bbox: bbox reductions for the intersection filter: source ground/pillar/facade
//      (cregistration.hpp:2912-2915) and all target points (grid extent). Reads positions only, writes nothing per point.
// kFiniteOnly: points with a non-finite coordinate do not enter the box (an infinite extent has no grid).
template <bool kUndistort, bool kFiniteOnly = false>
__global__ void __launch_bounds__(kIngestBlock) k_ingest_bbox(DeviceArrays A) {
    const ChunkDesc cd = A.in_chunks[blockIdx.x];
    const PairConst &pc = A.pc[cd.pair];
    const uint32_t seg = cd.seg;
    const bool is_src = seg >= kNumClasses;
    const int cls = seg % kNumClasses;
    const bool want = is_src ? (cls == MULLS_GROUND || cls == MULLS_PILLAR || cls == MULLS_FACADE) : true;
    if (!want) return; // block-uniform
    const uint32_t local = cd.first + threadIdx.x;
    bool valid = local < pc.in_n[seg];
    float4 p = make_float4(0.f, 0.f, 0.f, 0.f), unused;
    if (valid) load_input_point<kUndistort, false>(pc, seg, local, p, unused);
    if (kFiniteOnly) valid = valid && finite_xyz(p);
    float mn[3] = {valid ? p.x : FLT_MAX, valid ? p.y : FLT_MAX, valid ? p.z : FLT_MAX};
    float mx[3] = {valid ? p.x : -FLT_MAX, valid ? p.y : -FLT_MAX, valid ? p.z : -FLT_MAX};
#pragma unroll
    for (int d = 0; d < 3; ++d)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[d] = fminf(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
            mx[d] = fmaxf(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
        }
    __shared__ float s_mn[kIngestBlock / 32][3], s_mx[kIngestBlock / 32][3];
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int d = 0; d < 3; ++d) s_mn[threadIdx.x >> 5][d] = mn[d], s_mx[threadIdx.x >> 5][d] = mx[d];
    }
    __syncthreads();
    if (threadIdx.x < 6) { // one atomic per block and bound
        const int d = threadIdx.x % 3;
        const bool is_max = threadIdx.x >= 3;
        float v = is_max ? s_mx[0][d] : s_mn[0][d];
        for (int w = 1; w < kIngestBlock / 32; ++w) v = is_max ? fmaxf(v, s_mx[w][d]) : fminf(v, s_mn[w][d]);
        int *bb = is_src ? A.ps[cd.pair].bb_src : A.ps[cd.pair].bb_tgt;
        if (is_max) atomicMax(&bb[3 + d], float_to_ordered(v));
        else atomicMin(&bb[d], float_to_ordered(v));
    }
}

// ---- k_pair_setup: one thread per pair. Intersection bbox (utility.hpp:858-866, pad 1.0,
//      cregistration.hpp:2907-2916), grid geometry, initial state (:1144-1164).
constexpr float kH0Min = 0.125f; // smallest level-0 cell (m); doubled until the grid spans the pair
__global__ void k_pair_setup(DeviceArrays A, int n_pairs) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pairs) return;
    const PairConst &pc = A.pc[p];
    PairState &ps = A.ps[p];
    double smin[3], smax[3], tmin[3], tmax[3];
    for (int d = 0; d < 3; ++d) {
        smin[d] = (double)ordered_to_float(ps.bb_src[d]);
        smax[d] = (double)ordered_to_float(ps.bb_src[3 + d]);
        tmin[d] = (double)ordered_to_float(ps.bb_tgt[d]);
        tmax[d] = (double)ordered_to_float(ps.bb_tgt[3 + d]);
    }
    const double big = 1.7976931348623157e308;
    double gmin[3], gmax[3];
    if (pc.apply_filter) {
        const float pad = 1.0f;
        for (int d = 0; d < 3; ++d) {
            // an empty source bbox stays at +/-FLT_MAX here (DBL_MAX in the reference): either way
            // the intersection is empty and every point is filtered out.
            double lo = (pc.tbound[d] > smin[d]) ? pc.tbound[d] : smin[d];
            double hi = (pc.tbound[3 + d] < smax[d]) ? pc.tbound[3 + d] : smax[d];
            ps.ibb[d] = lo - (double)pad;
            ps.ibb[3 + d] = hi + (double)pad;
            gmin[d] = fmax(tmin[d], ps.ibb[d]);
            gmax[d] = fmin(tmax[d], ps.ibb[3 + d]);
        }
    } else {
        for (int d = 0; d < 3; ++d) {
            ps.ibb[d] = -big;
            ps.ibb[3 + d] = big;
            gmin[d] = tmin[d];
            gmax[d] = tmax[d];
        }
    }
    double ext = 0.0;
    for (int d = 0; d < 3; ++d) {
        if (!(gmax[d] >= gmin[d])) {
            gmin[d] = 0.0;
            gmax[d] = 0.0;
        }
        ext = fmax(ext, gmax[d] - gmin[d]);
    }
    const int ncell = 1 << kCoordBits;
    float h0 = kH0Min;
    while ((ext + 8.0 * h0) * 1.001 > (double)h0 * (ncell - 4)) h0 *= 2.0f;
    ps.h0 = h0;
    ps.inv_h0 = 1.0f / h0; // a power of two: exact
    for (int d = 0; d < 3; ++d) ps.origin[d] = (float)gmin[d] - 2.0f * h0;
    // number of levels: the top level's guaranteed coverage 0.999*h must reach the largest search
    // radius 2.5*dis_thre_unit (filter_dis_times, cregistration.hpp:1707)
    const float rmax = 2.5f * pc.thre_unit * 1.0001f;
    int L = 2; // level l's 2x2x2 block covers 0.999 * h0 * 2^(l-1) (see nn_search)
    while (L < kMaxLevels && 0.999f * 0.5f * h0 * (float)(1 << (L - 1)) < rmax) ++L;
    // normal shooting needs the exact 10 nearest targets with no distance bound: full pyramid, whose top 2x2x2
    // block (2 x 2048 level-0 cells per axis) spans the whole grid
    if (pc.normal_shooting) L = kMaxLevels;
    ps.n_levels = L;

    for (int i = 0; i < 16; ++i) {
        ps.T_total[i] = pc.init[i];
        ps.T_inc[i] = (i % 5 == 0) ? 1.0 : 0.0;
    }
    for (int i = 0; i < 36; ++i) ps.cofactor[i] = ps.info[i] = (i % 7 == 0) ? 1.0 : 0.0;
    for (int i = 0; i < 6; ++i) ps.x[i] = 0.0;
    ps.sigma2 = 1.0;
    ps.thre = pc.thre_unit;
    ps.confidence = 1.0f;
    ps.status = kRunning;
    ps.code = 0;
    ps.iter = 0;
    ps.iters_entered = 0;
    ps.final_buf = 0;
    ps.alg_bytes = 0;
    if (pc.max_iter <= 0) {
        ps.status = kDone;
        const int left = atomicSub(A.running, 1) - 1;
        *A.h_running = left;
        __threadfence_system();
    }
}

// Morton code of the level-0 cell of p. Targets are inside the grid by construction; sources may stick out (clamped:
// the source key only orders threads for locality, it never enters a distance decision).
__device__ __forceinline__ uint64_t cell_morton(const PairState &ps, const float4 &p) {
    const int hi = (1 << kCoordBits) - 1;
    const int cx = (int)floorf((p.x - ps.origin[0]) * ps.inv_h0);
    const int cy = (int)floorf((p.y - ps.origin[1]) * ps.inv_h0);
    const int cz = (int)floorf((p.z - ps.origin[2]) * ps.inv_h0);
    return morton36((uint32_t)min(max(cx, 0), hi), (uint32_t)min(max(cy, 0), hi), (uint32_t)min(max(cz, 0), hi));
}

// ---- digit histograms of the segment sort: a block counts into shared memory (one atomic per warp and distinct digit),
//      then adds its non-empty bins to the segment's global histogram. Every lane of the warp calls digit_hist_add.
__device__ __forceinline__ uint32_t *digit_hist_of(const DeviceArrays &A, uint32_t pair, uint32_t seg) {
    return A.digit_hist + (size_t)(pair * kNumSegs + seg) * (kSortPasses * kSortBins);
}
__device__ __forceinline__ void digit_hist_add(uint32_t (*s_hist)[kSortBins], bool on, uint64_t m) {
    const unsigned lt = (1u << (threadIdx.x & 31)) - 1u;
#pragma unroll
    for (int d = 0; d < kSortPasses; ++d) {
        const uint32_t b = on ? (uint32_t)(m >> (kSortDigitBits * d)) & (kSortBins - 1) : kSortBins;
        const unsigned peers = __match_any_sync(0xffffffffu, b);
        if (on && (peers & lt) == 0) atomicAdd(&s_hist[d][b], (unsigned)__popc(peers));
    }
}
__device__ __forceinline__ void digit_hist_flush(uint32_t (*s_hist)[kSortBins], uint32_t *g, bool subtract) {
    for (int i = threadIdx.x; i < kSortPasses * kSortBins; i += blockDim.x) {
        const uint32_t c = s_hist[i / kSortBins][i % kSortBins];
        if (c) atomicAdd(&g[i], subtract ? 0u - c : c);
    }
}

// ---- k_make_keys: one block per sort tile. Intersection filter (cfilter.hpp:950-981: strictly inside) + the point's
//      Morton code into keys_a (~0: filtered out, the point leaves the sort), and the digit histograms of the segment.
// kFiniteOnly: points with a non-finite coordinate are filtered out as well.
template <bool kUndistort, bool kFiniteOnly = false>
__global__ void __launch_bounds__(kIngestBlock) k_make_keys(DeviceArrays A) {
    const ChunkDesc td = A.sort_tiles[blockIdx.x];
    const PairConst &pc = A.pc[td.pair];
    PairState &ps = A.ps[td.pair];
    const uint32_t seg = td.seg;
    __shared__ uint32_t s_hist[kSortPasses][kSortBins];
    for (int i = threadIdx.x; i < kSortPasses * kSortBins; i += kIngestBlock) s_hist[i / kSortBins][i % kSortBins] = 0;
    __syncthreads();
    unsigned kept = 0;
#pragma unroll 1
    for (int k = 0; k < kSortItems; ++k) {
        const uint32_t local = td.first + k * kIngestBlock + threadIdx.x;
        bool inside = false;
        uint64_t m = 0;
        if (local < pc.in_n[seg]) {
            float4 p, unused;
            load_input_point<kUndistort, false>(pc, seg, local, p, unused);
            const double *b = ps.ibb;
            inside = (double)p.x > b[0] && (double)p.x < b[3] && (double)p.y > b[1] && (double)p.y < b[4] &&
                     (double)p.z > b[2] && (double)p.z < b[5];
            if (kFiniteOnly) inside = inside && finite_xyz(p);
            if (inside) m = cell_morton(ps, p);
            A.keys_a[(size_t)pc.in_off[seg] + local] = inside ? m : ~0ull;
        }
        digit_hist_add(s_hist, inside, m);
        kept += (unsigned)__popc(__ballot_sync(0xffffffffu, inside));
    }
    if ((threadIdx.x & 31) == 0 && kept) atomicAdd(&ps.seg_count[seg], kept);
    __syncthreads();
    digit_hist_flush(s_hist, digit_hist_of(A, td.pair, seg), false);
}

// ---- keep_less_source_pts (cregistration.hpp:2866-2892) -> random_downsample_pcl (cfilter.hpp:606-628) --------
// The reference samples with pcl::RandomSample seeded by time(NULL); here the kept subset of a cloud is the k
// points with the smallest key splitmix64(seed, cloud, original index) (uniform, reproducible, order preserved).
// k-th smallest key per cloud = 8-pass radix select (256-bin histogram per pass), then one marking pass.
__device__ __forceinline__ uint64_t sample_key(uint32_t seed, uint32_t cloud_id, uint32_t index) {
    uint64_t z = (((uint64_t)seed << 40) ^ ((uint64_t)cloud_id << 32) ^ (uint64_t)index) + 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

__global__ void k_keepless_plan(DeviceArrays A, int n_pairs) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pairs) return;
    const PairConst &pc = A.pc[p];
    PairState &ps = A.ps[p];
    for (int s = 0; s < kNumSegs; ++s) {
        ps.kl_keep[s] = -1;
        ps.kl_prefix[s] = 0;
        ps.kl_rank[s] = 0;
        for (int b = 0; b < 256; ++b) ps.kl_hist[s][b] = 0;
    }
    if (!pc.keep_less) return;
    const int S = kNumClasses; // source segments follow the six target segments
    auto plan = [&](int seg, int keep) { // random_downsample_pcl: untouched if size <= keep_number
        if ((int)ps.seg_count[seg] > keep) {
            ps.kl_keep[seg] = keep;
            ps.kl_rank[seg] = (uint32_t)keep;
        }
        return ((int)ps.seg_count[seg] > keep) ? keep : (int)ps.seg_count[seg];
    };
    // order and rates of :2882-2890 (target_down_rate 2, ground_down_rate 4, facade_down_rate 2)
    const int tg = plan(MULLS_GROUND, (int)(ps.seg_count[MULLS_GROUND] / 2));
    const int tf = plan(MULLS_FACADE, (int)(ps.seg_count[MULLS_FACADE] / 2));
    plan(S + MULLS_GROUND, tg / 4);
    plan(S + MULLS_FACADE, tf / 2);
    plan(S + MULLS_PILLAR, (int)ps.seg_count[MULLS_PILLAR]);
    plan(S + MULLS_BEAM, (int)ps.seg_count[MULLS_BEAM]);
    plan(S + MULLS_ROOF, (int)ps.seg_count[MULLS_ROOF]);
    plan(S + MULLS_VERTEX, (int)ps.seg_count[MULLS_VERTEX]);
}

// pass = 0..7: histogram of byte `pass` (from the top) of the keys whose higher bytes equal the prefix found so far
__global__ void __launch_bounds__(kIngestBlock) k_keepless_hist(DeviceArrays A, int pass) {
    const ChunkDesc cd = A.in_chunks[blockIdx.x];
    const PairConst &pc = A.pc[cd.pair];
    PairState &ps = A.ps[cd.pair];
    const uint32_t seg = cd.seg;
    if (ps.kl_keep[seg] <= 0) return; // untouched, or cleared entirely
    __shared__ uint32_t s_hist[256];
    s_hist[threadIdx.x] = 0; // kIngestBlock == 256
    __syncthreads();
    const uint32_t local = cd.first + threadIdx.x;
    if (local < pc.in_n[seg]) {
        const size_t gi = (size_t)pc.in_off[seg] + local;
        if (A.keys_a[gi] != ~0ull) {
            const uint64_t key = sample_key(pc.random_seed, seg, local);
            const int shift = 56 - 8 * pass;
            const bool match = (pass == 0) || ((key >> (shift + 8)) == (ps.kl_prefix[seg] >> (shift + 8)));
            if (match) atomicAdd(&s_hist[(key >> shift) & 0xff], 1u);
        }
    }
    __syncthreads();
    if (s_hist[threadIdx.x]) atomicAdd(&ps.kl_hist[seg][threadIdx.x], s_hist[threadIdx.x]);
}

__global__ void k_keepless_step(DeviceArrays A, int n_pairs, int pass) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pairs) return;
    PairState &ps = A.ps[p];
    for (int s = 0; s < kNumSegs; ++s) {
        if (ps.kl_keep[s] <= 0) continue;
        uint32_t cum = 0, rank = ps.kl_rank[s];
        int d = 0;
        for (; d < 256; ++d) {
            const uint32_t h = ps.kl_hist[s][d];
            if (cum + h >= rank) break;
            cum += h;
        }
        ps.kl_prefix[s] |= (uint64_t)d << (56 - 8 * pass);
        ps.kl_rank[s] = rank - cum;
        for (int b = 0; b < 256; ++b) ps.kl_hist[s][b] = 0;
    }
}

// drop the points whose key exceeds the k-th smallest one (keys are a bijection of the index: exactly k remain); their
// digits leave the segment's histograms
__global__ void __launch_bounds__(kIngestBlock) k_keepless_mark(DeviceArrays A) {
    const ChunkDesc cd = A.in_chunks[blockIdx.x];
    const PairConst &pc = A.pc[cd.pair];
    PairState &ps = A.ps[cd.pair];
    const uint32_t seg = cd.seg;
    const int keep = ps.kl_keep[seg];
    if (keep < 0) return;
    __shared__ uint32_t s_hist[kSortPasses][kSortBins];
    for (int i = threadIdx.x; i < kSortPasses * kSortBins; i += kIngestBlock) s_hist[i / kSortBins][i % kSortBins] = 0;
    __syncthreads();
    const uint32_t local = cd.first + threadIdx.x;
    bool drop = false;
    uint64_t m = 0;
    if (local < pc.in_n[seg]) {
        const size_t gi = (size_t)pc.in_off[seg] + local;
        m = A.keys_a[gi];
        if (m != ~0ull) {
            drop = (keep == 0) || sample_key(pc.random_seed, seg, local) > ps.kl_prefix[seg];
            if (drop) A.keys_a[gi] = ~0ull;
        }
    }
    digit_hist_add(s_hist, drop, m);
    const unsigned b = __ballot_sync(0xffffffffu, drop);
    if ((threadIdx.x & 31) == 0 && b) atomicSub(&ps.seg_count[seg], (unsigned)__popc(b));
    __syncthreads();
    digit_hist_flush(s_hist, digit_hist_of(A, cd.pair, seg), true);
}

// Exclusive scan over a block of kThreads threads (a multiple of 32, at most 1024); *total = the sum of all v.
template <int kThreads>
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t *s_warp, uint32_t &total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp[w] = incl;
    __syncthreads();
    if (w == 0) {
        const uint32_t x = lane < kThreads / 32 ? s_warp[lane] : 0u;
        uint32_t xi = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, xi, o);
            if (lane >= o) xi += t;
        }
        if (lane < kThreads / 32) s_warp[lane] = xi - x;
        if (lane == 31) s_warp[32] = xi;
    }
    __syncthreads();
    total = s_warp[32];
    const uint32_t r = s_warp[w] + incl - v;
    __syncthreads(); // s_warp may be reused
    return r;
}

// ---- k_digit_scan: one block per (pair, segment): each digit's counts -> the bin's first position inside the segment
__global__ void __launch_bounds__(kSortBins) k_digit_scan(DeviceArrays A) {
    __shared__ uint32_t s_warp[33];
    uint32_t *h = A.digit_hist + (size_t)blockIdx.x * (kSortPasses * kSortBins);
    for (int d = 0; d < kSortPasses; ++d) {
        uint32_t total;
        const uint32_t v = h[d * kSortBins + threadIdx.x];
        h[d * kSortBins + threadIdx.x] = block_exclusive_scan<kSortBins>(v, s_warp, total);
    }
}

// ---- k_seg_offsets: single block; exclusive scan of the valid counts in (pair, seg) order gives the
//      start of every segment in the sorted array; also per-class sizes and :1195-1201.
__global__ void k_seg_offsets(DeviceArrays A, int n_pairs) {
    __shared__ uint32_t carry;
    __shared__ uint32_t warp_sums[32];
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int total = n_pairs * kNumSegs;
    for (int base = 0; base < total; base += blockDim.x) {
        const int i = base + threadIdx.x;
        uint32_t v = 0;
        if (i < total) v = A.ps[i / kNumSegs].seg_count[i % kNumSegs];
        uint32_t incl = v;
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if ((threadIdx.x & 31) >= o) incl += t;
        }
        if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = incl;
        __syncthreads();
        if (threadIdx.x < 32) {
            uint32_t w = (threadIdx.x < (blockDim.x >> 5)) ? warp_sums[threadIdx.x] : 0;
            uint32_t wi = w;
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
                if (threadIdx.x >= o) wi += t;
            }
            warp_sums[threadIdx.x] = wi - w; // exclusive
        }
        __syncthreads();
        const uint32_t excl = carry + warp_sums[threadIdx.x >> 5] + incl - v;
        if (i < total) A.ps[i / kNumSegs].seg_start[i % kNumSegs] = excl;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry = excl + v;
        __syncthreads();
    }
    for (int p = threadIdx.x; p < n_pairs; p += blockDim.x) {
        PairState &ps = A.ps[p];
        const PairConst &pc = A.pc[p];
        for (int c = 0; c < kNumClasses; ++c) {
            ps.n_tgt[c] = (int)ps.seg_count[c];
            ps.n_src[c] = (int)ps.seg_count[kNumClasses + c];
            ps.n_src_g[c] = ps.n_src[c];
            ps.n_corr[c] = 0;
            ps.n_corr_last[c] = 0;
        }
        int cnt = 0;
        if (pc.used[MULLS_PILLAR]) cnt += ps.n_src[MULLS_PILLAR];
        if (pc.used[MULLS_FACADE]) cnt += ps.n_src[MULLS_FACADE];
        if (pc.used[MULLS_BEAM]) cnt += ps.n_src[MULLS_BEAM];
        ps.source_feature_points_count = cnt;
    }
}

// Sorted elements i-1 and i (kcur = keys[i]): the target cells that start at i are those of levels 0..top, where top
// is the highest level at which the two Morton codes differ (every level at the start of a target segment); -1: none.
__device__ __forceinline__ int cell_top(const uint64_t *keys, uint32_t i, uint64_t kcur) {
    if (kcur == ~0ull || ((uint32_t)(kcur >> 36) % kNumSegs) >= kNumClasses) return -1;
    if (i == 0) return kMaxLevels - 1;
    const uint64_t kprev = keys[i - 1];
    if ((kprev >> 36) != (kcur >> 36)) return kMaxLevels - 1;
    const uint64_t diff = (kcur ^ kprev) & ((1ull << 36) - 1);
    if (diff == 0) return -1; // same finest cell: no boundary at any level
    return (63 - __clzll((long long)diff)) / 3;
}

// ---- k_sort_pass: pass kPass of the Morton sort inside every (pair, segment), a stable LSD radix sort by 9-bit digit.
// The batch is already grouped by segment, so a pass scatters inside the segment's own range: bin b of a tile goes to
// the segment's start + the bin's offset in the segment (k_digit_scan) + what the segment's earlier tiles put into b.
// The last comes from a decoupled look-back over those tiles (consecutive in sort_tiles; a block fetches its tile from a
// counter, so every earlier tile is held by a running block). A tile ranks its points in input order, so equal keys keep
// the order in which they came: pass 0 reads the keys k_make_keys wrote in input order, the points it keeps are what
// CUB's stable sort of [pair*12+seg | morton36] ordered. Passes 0-2 write the segment compacted to the front of its input
// range, each point as one word: the digits still to sort above its 31-bit index in the input cloud. Pass 3 writes the
// sorted order: the keys [pair*12+seg | morton36] (~0 for the filtered-out points, at the tail) and the SoA slices
// (targets, and source buffer 0), each point recomputed from the input by load_input_point (normal .w = its index in the
// input cloud). Look-back word: (2 * epoch + inclusive) << 32 | count; older passes carry smaller epochs.
struct SortSmem {
    union {
        uint32_t warp_bin[kIngestBlock / 32][kSortBins]; // ranking: per warp and bin, its points, then the warps' offsets
        struct {
            uint64_t item[kSortTile];                    // the tile in sorted order
            uint16_t bin[kSortTile];
        } stage;
    } u;
    uint32_t tile_start[kSortBins]; // first position of each bin in the tile's sorted order
    uint32_t out_base[kSortBins];   // destination of tile position p of bin b: out_base[b] + p
    uint32_t warp_sum[33];
    uint32_t tile, n_tile;
};

template <int kPass>
__device__ __forceinline__ uint32_t sort_digit(uint64_t e) {
    return (uint32_t)(kPass == 0 ? e : e >> 31) & (kSortBins - 1);
}

template <int kPass, bool kUndistort>
__global__ void __launch_bounds__(kIngestBlock, 3) k_sort_pass(DeviceArrays A, const uint64_t *in, uint64_t *out, int n_pairs,
                                                            uint32_t epoch) {
    constexpr bool kLast = kPass == kSortPasses - 1;
    __shared__ SortSmem s;
    if (threadIdx.x == 0) s.tile = atomicAdd(&A.sort_ctr[kPass], 1u);
    for (int i = threadIdx.x; i < (kIngestBlock / 32) * kSortBins; i += kIngestBlock) (&s.u.warp_bin[0][0])[i] = 0;
    __syncthreads();
    const uint32_t t = s.tile;
    const ChunkDesc td = A.sort_tiles[t];
    const PairConst &pc = A.pc[td.pair];
    const PairState &ps = A.ps[td.pair];
    const uint32_t seg = td.seg;
    const uint32_t n = kPass == 0 ? pc.in_n[seg] : ps.seg_count[seg]; // points of the segment in `in`
    if (kLast) { // filtered-out points: ~0 keys after the last kept point of the batch
        const PairState &pl = A.ps[n_pairs - 1];
        const uint32_t kept = pl.seg_start[kNumSegs - 1] + pl.seg_count[kNumSegs - 1];
        const uint32_t tail = kept + (pc.in_off[seg] - ps.seg_start[seg]) - n;
        for (uint32_t i = max(td.first, n) + threadIdx.x; i < min(td.first + kSortTile, pc.in_n[seg]); i += kIngestBlock)
            out[tail + i] = ~0ull;
    }
    if (td.first >= n) return; // block-uniform; no later tile of the segment has points either: nobody looks back here
    const uint64_t *src = in + pc.in_off[seg];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned lt = (1u << lane) - 1u;
    // rank: warp w takes the tile's w-th slice; item j of the lanes is a coalesced row, rows in input order
    uint64_t item[kSortItems];
    uint32_t rb[kSortItems]; // rank among the warp's points of the same bin | bin << 16 (bin kSortBins: no point)
#pragma unroll
    for (int j = 0; j < kSortItems; ++j) {
        const uint32_t idx = td.first + (w * kSortItems + j) * 32 + lane;
        uint64_t e = idx < n ? src[idx] : ~0ull;
        const bool valid = e != ~0ull; // (no packed word is ~0: it has at most 27 + 31 bits)
        const uint32_t b = valid ? sort_digit<kPass>(e) : kSortBins;
        const unsigned peers = __match_any_sync(0xffffffffu, b);
        uint32_t r = 0;
        if (valid) r = s.u.warp_bin[w][b] + (uint32_t)__popc(peers & lt);
        __syncwarp();
        if (valid && (peers & lt) == 0) s.u.warp_bin[w][b] += (uint32_t)__popc(peers);
        __syncwarp();
        if (kPass == 0) e = ((e >> kSortDigitBits) << 31) | idx;
        else if (!kLast) e = ((e >> (31 + kSortDigitBits)) << 31) | (e & 0x7fffffffu);
        else e &= 0x7fffffffu;
        item[j] = e;
        rb[j] = r | (b << 16);
    }
    __syncthreads();
    // bins 2 tid and 2 tid + 1: the warps' offsets, the tile's counts and their scan
    uint32_t cnt[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        const int b = 2 * threadIdx.x + q;
        uint32_t run = 0;
#pragma unroll
        for (int v = 0; v < kIngestBlock / 32; ++v) {
            const uint32_t c = s.u.warp_bin[v][b];
            s.u.warp_bin[v][b] = run;
            run += c;
        }
        cnt[q] = run;
    }
    uint32_t n_tile;
    const uint32_t ex = block_exclusive_scan<kIngestBlock>(cnt[0] + cnt[1], s.warp_sum, n_tile);
    s.tile_start[2 * threadIdx.x] = ex;
    s.tile_start[2 * threadIdx.x + 1] = ex + cnt[0];
    // look-back: publish the tile's counts, add up the earlier tiles' counts until one carries its inclusive prefix
    volatile uint64_t *status = A.sort_status;
    const uint64_t agg = (uint64_t)(2u * epoch) << 32, inc = (uint64_t)(2u * epoch + 1u) << 32;
#pragma unroll
    for (int q = 0; q < 2; ++q) status[(size_t)t * kSortBins + 2 * threadIdx.x + q] = (td.first == 0 ? inc : agg) | cnt[q];
    const uint32_t *dig = digit_hist_of(A, td.pair, seg) + kPass * kSortBins;
    const uint32_t base = kLast ? ps.seg_start[seg] : pc.in_off[seg];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        const int b = 2 * threadIdx.x + q;
        uint32_t prefix = 0;
        if (td.first != 0) {
            for (uint32_t k = t - 1;; --k) {
                uint64_t v;
                do v = status[(size_t)k * kSortBins + b];
                while ((uint32_t)(v >> 32) < 2u * epoch);
                prefix += (uint32_t)v;
                if ((uint32_t)(v >> 32) & 1u) break;
            }
            status[(size_t)t * kSortBins + b] = inc | (prefix + cnt[q]);
        }
        s.out_base[b] = base + dig[b] + prefix - s.tile_start[b];
    }
    __syncthreads();
    uint32_t pos[kSortItems];
#pragma unroll
    for (int j = 0; j < kSortItems; ++j) {
        const uint32_t b = rb[j] >> 16;
        pos[j] = b < kSortBins ? s.tile_start[b] + s.u.warp_bin[w][b] + (rb[j] & 0xffffu) : 0u;
    }
    __syncthreads(); // warp_bin gives way to the staged tile
#pragma unroll
    for (int j = 0; j < kSortItems; ++j) {
        const uint32_t b = rb[j] >> 16;
        if (b < kSortBins) {
            s.u.stage.item[pos[j]] = item[j];
            s.u.stage.bin[pos[j]] = (uint16_t)b;
        }
    }
    __syncthreads();
    if (!kLast) {
        for (uint32_t p = threadIdx.x; p < n_tile; p += kIngestBlock) out[s.out_base[s.u.stage.bin[p]] + p] = s.u.stage.item[p];
        return;
    }
    const uint32_t sg = td.pair * kNumSegs + seg;
    // kGather points per thread at a time: their input rows are all loaded before any of them is stored
    constexpr int kGather = 4;
    const uint32_t dst_base = seg < kNumClasses ? pc.tgt_base[seg] : pc.src_base[seg - kNumClasses];
    const int index_shift = (seg >= kNumClasses && pc.sharded) ? (int)pc.src_index_base[seg - kNumClasses] : 0;
    float4 *dst_pos = seg < kNumClasses ? A.tgt_pos : A.src_pos[0];
    float4 *dst_nrm = seg < kNumClasses ? A.tgt_nrm : A.src_nrm[0];
    // (src_prevj and src_cert need no initial value: iteration 0 reads no previous match, and a certificate is read only
    // after k_search<1> has written it, kernels_iterate.cuh)
    for (uint32_t p0 = threadIdx.x; p0 < n_tile; p0 += kGather * kIngestBlock) {
        float4 pt[kGather], nrm[kGather];
#pragma unroll
        for (int g = 0; g < kGather; ++g) {
            const uint32_t p = p0 + g * kIngestBlock;
            if (p < n_tile) load_input_point<kUndistort, true>(pc, seg, (uint32_t)s.u.stage.item[p], pt[g], nrm[g]);
        }
#pragma unroll
        for (int g = 0; g < kGather; ++g) {
            const uint32_t p = p0 + g * kIngestBlock;
            if (p >= n_tile) break;
            const uint32_t i = s.out_base[s.u.stage.bin[p]] + p;
            out[i] = ((uint64_t)sg << 36) | cell_morton(ps, pt[g]);
            const uint32_t d = dst_base + (i - ps.seg_start[seg]);
            nrm[g].w = __int_as_float(__float_as_int(nrm[g].w) + index_shift);
            dst_pos[d] = pt[g];
            dst_nrm[d] = nrm[g];
        }
    }
}

// ---- k_cell_count: the grid cells of every (pair, class) in the sorted keys -> PairState::hash_entries, from which
//      k_hash_layout sizes the tables. (Not part of the last sort pass: a cell boundary needs the key before it, and a
//      tile of that pass does not hold the key before the first point of each of its bins.)
__global__ void __launch_bounds__(256) k_cell_count(DeviceArrays A, const uint64_t *keys, uint32_t n_total) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t key = i < n_total ? keys[i] : ~0ull;
    const uint32_t sg = (uint32_t)(key >> 36);
    const uint32_t pair = sg / kNumSegs, seg = sg % kNumSegs;
    const int top = cell_top(keys, i, key);
    const int cnt = top < 0 ? 0 : min(top, A.ps[pair].n_levels - 1) + 1;
    // one atomic per warp when all its lanes hold points of the same target segment (the common case)
    const bool is_tgt = key != ~0ull && seg < kNumClasses;
    const unsigned grp = __match_any_sync(0xffffffffu, is_tgt ? sg : 0xffffffffu);
    if (grp == 0xffffffffu) {
        const int tot = __reduce_add_sync(0xffffffffu, cnt);
        if ((threadIdx.x & 31) == 0 && tot > 0) atomicAdd(&A.ps[pair].hash_entries[seg], (unsigned)tot);
    } else if (cnt > 0) {
        atomicAdd(&A.ps[pair].hash_entries[seg], (unsigned)cnt);
    }
}

// Launches sort pass `pass` (k_sort_pass) over the batch's n_tiles sort tiles: keys_a -> keys_b -> keys_a -> keys_b ->
// keys_a, so the sorted keys end in keys_a. `epoch` counts the context's passes (the look-back words).
inline void enqueue_sort_pass(const DeviceArrays &A, cudaStream_t st, int pass, unsigned n_tiles, int n_pairs, bool undistort,
                              uint32_t &epoch) {
    const uint64_t *in = (pass & 1) ? A.keys_b : A.keys_a;
    uint64_t *out = (pass & 1) ? A.keys_a : A.keys_b;
    ++epoch;
    if (pass == 0) k_sort_pass<0, false><<<n_tiles, kIngestBlock, 0, st>>>(A, in, out, n_pairs, epoch);
    else if (pass == 1) k_sort_pass<1, false><<<n_tiles, kIngestBlock, 0, st>>>(A, in, out, n_pairs, epoch);
    else if (pass == 2) k_sort_pass<2, false><<<n_tiles, kIngestBlock, 0, st>>>(A, in, out, n_pairs, epoch);
    else if (undistort) k_sort_pass<3, true><<<n_tiles, kIngestBlock, 0, st>>>(A, in, out, n_pairs, epoch);
    else k_sort_pass<3, false><<<n_tiles, kIngestBlock, 0, st>>>(A, in, out, n_pairs, epoch);
}

// ---- hashed multi-level grid over a target class --------------------------------------------
// Entry = {key_lo, key_hi | child mask << 16, start, count} (grid_key.cuh); (0, 0) marks an empty slot.
// The slot follows from the key alone; the child mask rides along in the claimed word.
__device__ __forceinline__ void hash_insert(HashEntry *table, uint32_t hmask, uint32_t klo, uint32_t khi, uint32_t children,
                                            uint32_t start, uint32_t count) {
    uint32_t slot = cell_hash(klo, khi) & hmask;
    const unsigned long long packed = (unsigned long long)klo | ((unsigned long long)(khi | (children << 16)) << 32);
    while (true) {
        unsigned long long *kp = reinterpret_cast<unsigned long long *>(&table[slot]);
        if (atomicCAS(kp, 0ull, packed) == 0ull) {
            *reinterpret_cast<uint2 *>(&table[slot].start) = make_uint2(start, count);
            return;
        }
        slot = (slot + 1) & hmask;
    }
}

// End of the cell of sorted element b at the level of `shift` (= 3 * level): the keys in [b, end) are those equal to
// p = keys[b] >> shift, a prefix of [b, hi) since the keys are sorted. Galloping search: O(log size) loads, starting
// next to b, so the many small cells cost a load or two.
__device__ __forceinline__ uint32_t cell_end(const uint64_t *keys, uint32_t b, uint32_t hi, uint64_t p, int shift) {
    uint32_t in = b, out = hi, step = 1;
    while (in + step < hi) {
        if ((keys[in + step] >> shift) != p) {
            out = in + step;
            break;
        }
        in += step;
        step <<= 1;
    }
    while (out - in > 1) {
        const uint32_t mid = in + (out - in) / 2;
        if ((keys[mid] >> shift) == p) in = mid;
        else out = mid;
    }
    return out;
}

// k_hash_build: thread i opens the cells that start at sorted element i (cell_top), at levels 0..min(top, L-1), and
// writes each entry complete. A level-l cell ends where the last of its children (level l-1 cells, contiguous in Morton
// order) ends; the first child is the level-(l-1) cell opened at i, the others are found by galloping from its end, and
// their octants (x bit | y bit << 1 | z bit << 2 of the child's coordinates) make the child mask.
__global__ void __launch_bounds__(256) k_hash_build(DeviceArrays A, const uint64_t *keys, uint32_t n_total) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_total || A.hash_used[1]) return;
    const uint64_t kcur = keys[i];
    const int top = cell_top(keys, i, kcur);
    if (top < 0) return;
    const uint32_t sg = (uint32_t)(kcur >> 36);
    const uint32_t pair = sg / kNumSegs, cls = sg % kNumSegs;
    const PairState &ps = A.ps[pair];
    const int L = ps.n_levels;
    const uint32_t seg_begin = ps.seg_start[cls], seg_end = seg_begin + ps.seg_count[cls];
    HashEntry *table = A.hash + ps.hash_base[cls];
    const uint32_t hmask = ps.hash_mask[cls];
    const uint64_t m = kcur & ((1ull << 36) - 1);
    const uint32_t x0 = compact12(m), y0 = compact12(m >> 1), z0 = compact12(m >> 2);
    uint32_t end = cell_end(keys, i, seg_end, kcur, 0);
    for (int l = 0; l <= top && l < L; ++l) {
        uint32_t children = 0;
        if (l > 0) {
            const int shift = 3 * l;
            const uint64_t p = kcur >> shift;
            children = 1u << ((kcur >> (shift - 3)) & 7u);
            while (end < seg_end) {
                const uint64_t k = keys[end];
                if ((k >> shift) != p) break;
                children |= 1u << ((k >> (shift - 3)) & 7u);
                end = cell_end(keys, end, seg_end, k >> (shift - 3), shift - 3);
            }
        }
        const uint32_t x = x0 >> l, y = y0 >> l, z = z0 >> l;
        hash_insert(table, hmask, cell_key_lo(x, y, z), cell_key_hi(z, l), children, i - seg_begin, end - i);
    }
}

// k_hash_layout: single block. Power-of-two table per (pair, class) with load factor <= 0.5, carved out
// of the pool in order; flags overflow instead of writing out of bounds.
constexpr uint64_t kHashSlack = 4; // first choice: table capacity >= kHashSlack x cells
__device__ __forceinline__ uint64_t hash_table_cap(int attempt, uint32_t cells) {
    const uint64_t want = (attempt == 0) ? kHashSlack * cells : (attempt == 1) ? 2ull * cells : (5ull * cells) / 4 + 1;
    uint64_t cap = 16;
    while (cap < want) cap <<= 1;
    return cap;
}
__global__ void k_hash_layout(DeviceArrays A, int n_pairs) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    // load factor <= 1/kHashSlack if the pool allows it (a miss costs ~1.4 probes instead of 2.5 at 1/2), else
    // <= 0.5, else <= 0.8 (longer probe chains, same results), else give up
    for (int attempt = 0; attempt < 3; ++attempt) {
        uint64_t used = 0;
        bool overflow = false;
        for (int p = 0; p < n_pairs && !overflow; ++p) {
            PairState &ps = A.ps[p];
            for (int c = 0; c < kNumClasses; ++c) {
                const uint64_t cap = hash_table_cap(attempt, ps.hash_entries[c]);
                if (used + cap > A.hash_pool_entries) {
                    overflow = true;
                    break;
                }
                ps.hash_base[c] = (uint32_t)used;
                ps.hash_mask[c] = (uint32_t)(cap - 1);
                used += cap;
            }
        }
        A.hash_used[0] = overflow ? 0u : (uint32_t)used;
        A.hash_used[1] = overflow ? 1u : 0u;
        if (!overflow) return;
    }
    // overflow: [2] = the pool the last attempt needs (saturated), from which the host grows the pool and runs the call
    // again; [0] stays 0 (k_hash_clear clears nothing). The tables are degenerate and never searched (the searches check
    // hash_used[1]), and every pair stops here: the iteration phases after the search would otherwise read neighbour
    // indices that no search of this run has written.
    uint64_t need = 0;
    for (int p = 0; p < n_pairs; ++p) {
        PairState &ps = A.ps[p];
        for (int c = 0; c < kNumClasses; ++c) {
            need += hash_table_cap(2, ps.hash_entries[c]);
            ps.hash_base[c] = 0;
            ps.hash_mask[c] = 0;
        }
        if (ps.status == kRunning) {
            ps.status = kDone;
            *A.h_running = atomicSub(A.running, 1) - 1;
        }
    }
    __threadfence_system();
    A.hash_used[2] = need < 0xffffffffull ? (uint32_t)need : 0xffffffffu;
}

__global__ void __launch_bounds__(256) k_hash_clear(DeviceArrays A) {
    const uint32_t used = A.hash_used[0];
    const uint4 z = make_uint4(0, 0, 0, 0);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < used; i += gridDim.x * blockDim.x)
        reinterpret_cast<uint4 *>(A.hash)[i] = z;
}

} // namespace mulls
