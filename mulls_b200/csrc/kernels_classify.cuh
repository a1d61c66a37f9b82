// Non-ground feature classification: lo::CFilter<PointT>::classify_nground_pts (include/common/cfilter.hpp:2058-2290).
// The cloud is the <= unground_down_fixed_num (20000) points the PCA kernel has just processed, so — like the local map —
// this is latency work on small arrays: per-point kernels where points are independent, and 1024-thread single-block
// kernels (order-preserving compaction, radix select, chunked greedy NMS) where the reference is sequential. Every
// order-dependent step reproduces the sequential result exactly:
//   * vertex-neighbourhood promotion (:2169-2210) reads labels that the same loop has just written for smaller
//     indices: resolved by monotone rounds (a candidate waits while an earlier undecided candidate could still tip it);
//   * non_max_suppress (:1243-1312) is the greedy maximal independent set in score order: kernels_nms.cuh, shared
//     with mulls_non_max_suppress.
#pragma once
#include "device_math.cuh"
#include "device_types.cuh"
#include "kernels_map.cuh"
#include "kernels_nms.cuh"
#include "kernels_pca.cuh"

namespace mulls {

constexpr int kClsBlock = kMapBlock; // 1024: map_tile_slot is written for this block size

struct ClsState {
    uint32_t n_cls[4];   // pillar, beam, facade, roof after the threshold loop (:2103-2166)
    uint32_t n_cls2[4];  // ... after the promotion loop (:2169-2210): final class clouds
    uint32_t n_down[4];  // *_down after the thresholds / the NMS
    uint32_t n_down2[4]; // ... after the fixed-number down-sampling
    uint32_t n_vertex;
    uint32_t nms_ran[4]; // the class cloud was sorted by non_max_suppress (NmsArgs::ran)
};

struct ClsArgs {
    mulls_classify_params P;
    uint32_t n;        // points of cloud_in (after its own random down-sampling)
    int stride;        // pca_down_rate
    float4 *rows;      // cloud_in, 3 float4 per point, modified in place (normals)
    PcaArgs F;         // PCA results, indexed like rows
    uint8_t *label0;   // after the threshold loop: 0 none, 1 pillar, 2 beam, 3 facade, 4 roof
    uint8_t *label;    // final labels
    uint8_t *downflag; // thresholds of the *_down clouds passed (sharpen_with_nms off)
    uint8_t *st4;      // promotion state (see k_cls_promote)
    uint8_t *vflag;    // point yields a keypoint
    float4 *cls[4];    // class clouds in push order
    float4 *cls_sorted[4];
    float4 *down[4];
    float4 *down2[4];
    float4 *sect;      // one sector of xy_normal_balanced_downsample (n rows)
    float4 *vrows;     // keypoint rows by point index (n rows)
    float4 *vertex;
    ClsState *st;
};

struct ClsFeat { // pca_feature_t (pca.hpp:23-54): eigenvalues and ratios are doubles
    int pt_num;
    double curvature, linear_2, planar_2;
    float pdir[3], ndir[3];
};

// The ratios divide by l1, which is 0 for a neighbourhood of identical points. x86 SSE answers 0/0 with the default
// NaN (0xfff8000000000000, sign set); the device's canonical NaN has the sign clear. The reference's x86 build defines
// the value, so the device writes that one.
__device__ __forceinline__ double cls_ratio(double num, double den) {
    return (num == 0.0 && den == 0.0) ? __longlong_as_double((long long)0xfff8000000000000ull) : num / den;
}

// (float) of a ratio as cvtsd2ss converts it: a NaN keeps its sign and the top of its payload (0xfff8... -> 0xffc00000).
// The device's double-to-float conversion is not relied on to keep a NaN's sign.
__device__ __forceinline__ float cls_to_float(double v) {
    if (!isnan(v)) return (float)v;
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    return __uint_as_float(((unsigned)(b >> 32) & 0x80000000u) | 0x7fc00000u | ((unsigned)(b >> 29) & 0x3fffffu));
}

__device__ __forceinline__ ClsFeat cls_feat(const PcaArgs &F, uint32_t i) {
    ClsFeat f;
    f.pt_num = F.pt_num[i];
    f.curvature = f.linear_2 = f.planar_2 = 0.0;
    for (int d = 0; d < 3; ++d) f.pdir[d] = f.ndir[d] = 0.f;
    if (f.pt_num > 3) { // get_pca_feature, pca.hpp:390-434
        const double l1 = F.eigenvalues[3 * (size_t)i], l2 = F.eigenvalues[3 * (size_t)i + 1], l3 = F.eigenvalues[3 * (size_t)i + 2];
        f.curvature = ((l1 + l2 + l3) == 0) ? 0 : l3 / (l1 + l2 + l3); // the guard leaves no 0/0
        f.linear_2 = cls_ratio(l1 - l2, l1);
        f.planar_2 = cls_ratio(l2 - l3, l1);
        for (int d = 0; d < 3; ++d) f.pdir[d] = F.principal[3 * (size_t)i + d], f.ndir[d] = F.normal[3 * (size_t)i + d];
    }
    return f;
}

// ---- k_cls_label: the PCA's own assign_normal (pca.hpp:346-347, min_k = 1) and the threshold loop (:2103-2166)
__global__ void __launch_bounds__(256) k_cls_label(ClsArgs C) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C.n) return;
    const mulls_classify_params &P = C.P;
    const ClsFeat f = cls_feat(C.F, i);
    float4 *row = C.rows + 3 * (size_t)i;
    const float z = row[0].z;
    float4 nb = row[1];
    if (f.pt_num > 1) nb = make_float4(f.ndir[0], f.ndir[1], f.ndir[2], cls_to_float(f.planar_2)); // a NaN lands here
    int label = 0, down = 0;
    if (f.pt_num > P.neigh_k_min) {
        if (f.linear_2 > (double)P.edge_thre) {
            const float az = fabsf(f.pdir[2]);
            if (az > P.linear_vertical_sin_high_thre)
                label = 1;
            else if (az < P.linear_vertical_sin_low_thre && z < P.beam_height_max)
                label = 2;
            if (label) nb = make_float4(f.pdir[0], f.pdir[1], f.pdir[2], cls_to_float(f.linear_2));
            if (!P.sharpen_with_nms && f.linear_2 > (double)P.edge_thre_down) down = label;
        } else if (f.planar_2 > (double)P.planar_thre) {
            const float az = fabsf(f.ndir[2]);
            if (az > P.planar_vertical_sin_high_thre && z > P.roof_height_min)
                label = 4;
            else if (az < P.planar_vertical_sin_low_thre)
                label = 3;
            if (label) nb = make_float4(f.ndir[0], f.ndir[1], f.ndir[2], cls_to_float(f.planar_2));
            if (!P.sharpen_with_nms && f.planar_2 > (double)P.planar_thre_down) down = label;
        }
    }
    row[1] = nb;
    C.label0[i] = (uint8_t)label;
    C.label[i] = (uint8_t)label;
    C.downflag[i] = (uint8_t)down;
    // promotion candidates (:2177): state 1 = undecided
    const int method = (P.curvature_thre < 1e-8) ? 0 : P.extract_vertex_points_method;
    C.st4[i] = (method == 2 && label == 0 && f.pt_num > P.neigh_k_min && f.curvature > (double)P.curvature_thre) ? 1 : 0;
}

// ---- k_cls_compact: blocks 0..3 gather the class clouds, blocks 4..7 the *_down clouds of the threshold loop
__global__ void __launch_bounds__(kClsBlock) k_cls_compact(ClsArgs C) {
    __shared__ uint32_t s_warp[kClsBlock / 32];
    __shared__ uint32_t s_total;
    const int b = blockIdx.x, want = (b & 3) + 1;
    const uint8_t *flag = (b < 4) ? C.label0 : C.downflag;
    float4 *out = (b < 4) ? C.cls[b] : C.down[b - 4];
    if (threadIdx.x == 0) s_total = 0;
    __syncthreads();
    for (uint32_t tile = 0; tile < C.n; tile += kClsBlock) {
        const uint32_t i = tile + threadIdx.x;
        const bool keep = i < C.n && flag[i] == want;
        const uint32_t slot = map_tile_slot(keep, s_warp, &s_total);
        if (keep) {
            const float4 *r = C.rows + 3 * (size_t)i;
            float4 *o = out + 3 * (size_t)slot;
            o[0] = r[0], o[1] = r[1], o[2] = r[2];
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (b < 4)
            C.st->n_cls[b] = s_total;
        else
            C.st->n_down[b - 4] = s_total;
    }
}

// ---- the promotion loop (:2169-2210). Sequential semantics: when point i is visited, the labels of the earlier
//      promoted points are already in index_with_feature. st4: 0 no candidate, 1 undecided, 2 not promoted, 3 promoted
//      but neither pillar nor beam, 4 promoted pillar, 5 promoted beam.
__device__ __forceinline__ uint8_t promote_state(const ClsArgs &C, uint32_t i) {
    const float az = fabsf(C.F.principal[3 * (size_t)i + 2]);
    if (az > C.P.linear_vertical_sin_high_thre) return 4;
    if (az < C.P.linear_vertical_sin_low_thre && C.rows[3 * (size_t)i].z < C.P.beam_height_max) return 5;
    return 3;
}

// k_cls_promote_pre (all SMs): what can be settled without knowing the other candidates' fate. The count of labelled
// neighbours only grows during the loop, so "enough threshold-loop neighbours" is final, and "not enough even if every
// earlier candidate neighbour were promoted" is final too. (Other threads' decisions are invisible here: any non-zero
// st4 of an earlier neighbour counts as "may still be promoted".)
__global__ void __launch_bounds__(256) k_cls_promote_pre(ClsArgs C) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C.n || C.st4[i] != 1) return;
    const float thre = C.P.feature_pts_ratio_guess / (float)C.stride;
    const int pt_num = C.F.pt_num[i];
    int sure = 0, maybe = 0;
    for (int t = 0; t < pt_num; ++t) {
        const uint32_t j = C.F.nbr[(size_t)i * C.F.k + t] & 0x7fffffffu;
        if (C.label0[j])
            ++sure;
        else if (j < i && ((volatile uint8_t *)C.st4)[j] != 0)
            ++maybe;
    }
    if (1.0 * sure / pt_num > (double)thre)
        C.st4[i] = promote_state(C, i);
    else if (!(1.0 * (sure + maybe) / pt_num > (double)thre))
        C.st4[i] = 2;
}

// k_cls_promote (one block): the candidates that depend on each other, in monotone rounds, then the row updates
__global__ void __launch_bounds__(kClsBlock) k_cls_promote(ClsArgs C) {
    const float thre = C.P.feature_pts_ratio_guess / (float)C.stride;
    volatile uint8_t *st4 = C.st4;
    while (true) {
        int pending = 0;
        for (uint32_t i = threadIdx.x; i < C.n; i += kClsBlock) {
            if (st4[i] != 1) continue;
            const int pt_num = C.F.pt_num[i];
            int sure = 0, maybe = 0;
            for (int t = 0; t < pt_num; ++t) {
                const uint32_t j = C.F.nbr[(size_t)i * C.F.k + t] & 0x7fffffffu;
                if (C.label0[j]) {
                    ++sure;
                } else if (j < i) {
                    const uint8_t s = st4[j];
                    if (s >= 4)
                        ++sure;
                    else if (s == 1)
                        ++maybe;
                }
            }
            if (1.0 * sure / pt_num > (double)thre)
                st4[i] = promote_state(C, i);
            else if (1.0 * (sure + maybe) / pt_num > (double)thre)
                pending = 1; // an earlier candidate is still open and could tip this one
            else
                st4[i] = 2;
        }
        if (!__syncthreads_or(pending)) break;
    }
}

// k_cls_promote_apply: assign_normal(pt, feature, false), normal[3] = 5 * curvature (:2194-2195), labels
__global__ void __launch_bounds__(256) k_cls_promote_apply(ClsArgs C) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C.n) return;
    const uint8_t s = C.st4[i];
    if (s < 3) return;
    const ClsFeat f = cls_feat(C.F, i);
    // the curvature is never NaN (cls_feat): the plain conversion is the x86 one
    C.rows[3 * (size_t)i + 1] = make_float4(f.pdir[0], f.pdir[1], f.pdir[2], (float)(5.0 * f.curvature));
    if (s == 4) C.label[i] = 1;
    if (s == 5) C.label[i] = 2;
}

// ---- k_cls_compact2: blocks 0/1 append the promoted pillars / beams behind the threshold loop's
__global__ void __launch_bounds__(kClsBlock) k_cls_compact2(ClsArgs C) {
    __shared__ uint32_t s_warp[kClsBlock / 32];
    __shared__ uint32_t s_total;
    const int b = blockIdx.x;
    if (b >= 2) {
        if (threadIdx.x == 0) C.st->n_cls2[b] = C.st->n_cls[b];
        return;
    }
    if (threadIdx.x == 0) s_total = C.st->n_cls[b];
    __syncthreads();
    for (uint32_t tile = 0; tile < C.n; tile += kClsBlock) {
        const uint32_t i = tile + threadIdx.x;
        const bool keep = i < C.n && C.st4[i] == 4 + b;
        const uint32_t slot = map_tile_slot(keep, s_warp, &s_total);
        if (keep) {
            const float4 *r = C.rows + 3 * (size_t)i;
            float4 *o = C.cls[b] + 3 * (size_t)slot;
            o[0] = r[0], o[1] = r[1], o[2] = r[2];
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) C.st->n_cls2[b] = s_total;
}

// ---- k_cls_encode: encode_stable_points (:1071-1181) for one point per thread; the rows are gathered afterwards
__global__ void __launch_bounds__(256) k_cls_encode(ClsArgs C) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C.n) return;
    const mulls_classify_params &P = C.P;
    const int min_feature_pts = (int)(P.feature_pts_ratio_guess / (float)C.stride * (float)P.neighbor_k) - 1;
    const float min_curvature = (float)(0.3 * (double)P.curvature_thre);
    const ClsFeat f = cls_feat(C.F, i);
    bool is_v = false;
    if (f.pt_num > P.neigh_k_min && f.pt_num > 3 && f.curvature > (double)min_curvature) {
        int all[5] = {0, 0, 0, 0, 0}, cl[5] = {0, 0, 0, 0, 0}, fa[5] = {0, 0, 0, 0, 0};
        float accu_intensity = 0.0f;
        const int total = f.pt_num;
        for (int t = 0; t < total; ++t) {
            const uint32_t e = C.F.nbr[(size_t)i * C.F.k + t];
            const uint32_t j = e & 0x7fffffffu;
            const int lab = C.label[j];
            if (lab >= 1) {
                all[lab]++;
                if (e >> 31)
                    cl[lab]++;
                else
                    fa[lab]++;
            }
            accu_intensity += C.rows[3 * (size_t)j + 2].x;
        }
        if (all[1] + all[2] + all[3] + all[4] >= min_feature_pts) {
            is_v = true;
            int a[5], c[5], r[5];
            for (int l = 1; l <= 4; ++l) {
                a[l] = 100 * all[l] / total;
                c[l] = 100 * cl[l] / total;
                r[l] = 100 * fa[l] / total;
            }
            const int descriptor = a[1] * 1000000 + a[2] * 10000 + a[3] * 100 + a[4];
            const int descriptor_1 = c[1] * 1000000 + c[2] * 10000 + c[3] * 100 + c[4];
            const int descriptor_2 = r[1] * 1000000 + r[2] * 10000 + r[3] * 100 + r[4];
            const float4 *row = C.rows + 3 * (size_t)i;
            float4 ra = row[0], rb = row[1], rc = row[2];
            rb.w = (float)f.curvature; // never NaN (cls_feat)
            rc.y = (float)descriptor;
            rb.x = (float)descriptor_1;
            rb.y = (float)descriptor_2;
            rc.x = accu_intensity / (float)total;
            float4 *o = C.vrows + 3 * (size_t)i;
            o[0] = ra, o[1] = rb, o[2] = rc;
        }
    }
    C.vflag[i] = is_v ? 1 : 0;
}

__global__ void __launch_bounds__(kClsBlock) k_cls_compact_vertex(ClsArgs C) {
    __shared__ uint32_t s_warp[kClsBlock / 32];
    __shared__ uint32_t s_total;
    if (threadIdx.x == 0) s_total = 0;
    __syncthreads();
    for (uint32_t tile = 0; tile < C.n; tile += kClsBlock) {
        const uint32_t i = tile + threadIdx.x;
        const bool keep = i < C.n && C.vflag[i];
        const uint32_t slot = map_tile_slot(keep, s_warp, &s_total);
        if (keep) {
            const float4 *r = C.vrows + 3 * (size_t)i;
            float4 *o = C.vertex + 3 * (size_t)slot;
            o[0] = r[0], o[1] = r[1], o[2] = r[2];
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) C.st->n_vertex = s_total;
}

// ---- fixed-number down-sampling (:2257-2267) -----------------------------------------------------------------------
struct SampleShared {
    uint32_t warp[kClsBlock / 32];
    uint32_t total;
    uint32_t hist[256];
    uint64_t prefix;
    uint32_t rank;
    uint32_t single;
};

// random_downsample_pcl (cfilter.hpp:606-628) of in[0..n) appended to out at *out_n: the points with the keep_number
// smallest splitmix64(seed, cloud, position) keys, order preserved; untouched if n <= keep_number.
__device__ void block_sample_append(const float4 *in, uint32_t n, long long keep_num, uint32_t seed, uint32_t cloud, float4 *out,
                                    SampleShared &S) {
    const bool sample = keep_num >= 0 && (long long)n > keep_num;
    if (threadIdx.x == 0) S.prefix = 0, S.rank = (uint32_t)(sample ? keep_num : 0);
    __syncthreads();
    if (sample && keep_num > 0) {
        int pass = 0;
        for (; pass < 8; ++pass) {
            if (threadIdx.x < 256) S.hist[threadIdx.x] = 0;
            __syncthreads();
            const int shift = 56 - 8 * pass;
            const uint64_t prefix = S.prefix;
            for (uint32_t i = threadIdx.x; i < n; i += kClsBlock) {
                const uint64_t key = sample_key(seed, cloud, i);
                if (pass == 0 || (key >> (shift + 8)) == (prefix >> (shift + 8))) atomicAdd(&S.hist[(key >> shift) & 0xff], 1u);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                uint32_t cum = 0;
                const uint32_t rank = S.rank;
                int d = 0;
                for (; d < 256; ++d) {
                    if (cum + S.hist[d] >= rank) break;
                    cum += S.hist[d];
                }
                S.prefix = prefix | ((uint64_t)d << shift);
                S.rank = rank - cum;
                S.single = (S.hist[d] == 1u) ? 1u : 0u;
            }
            __syncthreads();
            if (S.single) break; // one key carries this prefix: it is the k-th smallest, fetch its low bytes directly
        }
        if (pass < 7) {
            const int shift = 56 - 8 * pass;
            const uint64_t prefix = S.prefix;
            __syncthreads();
            for (uint32_t i = threadIdx.x; i < n; i += kClsBlock) {
                const uint64_t key = sample_key(seed, cloud, i);
                if ((key >> shift) == (prefix >> shift)) S.prefix = key;
            }
            __syncthreads();
        }
    }
    const uint64_t thr = S.prefix;
    for (uint32_t tile = 0; tile < n; tile += kClsBlock) {
        const uint32_t i = tile + threadIdx.x;
        const bool keep = i < n && (!sample || (keep_num > 0 && sample_key(seed, cloud, i) <= thr));
        const uint32_t slot = map_tile_slot(keep, S.warp, &S.total);
        if (keep) {
            const float4 *r = in + 3 * (size_t)i;
            float4 *o = out + 3 * (size_t)slot;
            o[0] = r[0], o[1] = r[1], o[2] = r[2];
        }
    }
    __syncthreads();
}

// k_rows_sample: cloud_in's own down-sampling (:2086-2087)
__global__ void __launch_bounds__(kClsBlock) k_rows_sample(const float4 *in, uint32_t n, int keep, uint32_t seed, uint32_t cloud,
                                                           float4 *out) {
    __shared__ SampleShared S;
    if (threadIdx.x == 0) S.total = 0;
    __syncthreads();
    block_sample_append(in, n, keep, seed, cloud, out, S);
}

// one block per *_down cloud: pillar / roof random_downsample_pcl, facade / beam xy_normal_balanced_downsample
__global__ void __launch_bounds__(kClsBlock) k_cls_fixed(ClsArgs C) {
    __shared__ SampleShared S;
    __shared__ uint32_t s_warp2[kClsBlock / 32];
    __shared__ uint32_t s_sect;
    const int c = blockIdx.x; // 0 pillar, 1 beam, 2 facade, 3 roof
    const mulls_classify_params &P = C.P;
    const uint32_t n = C.st->n_down[c];
    const float4 *in = C.down[c];
    float4 *out = C.down2[c];
    if (threadIdx.x == 0) S.total = 0;
    __syncthreads();
    if (c == 0 || c == 3) {
        block_sample_append(in, n, c == 0 ? P.pillar_down_fixed_num : P.roof_down_fixed_num, P.random_seed, c == 0 ? 19u : 28u, out, S);
    } else {
        const int sector_num = 4;
        const int keep = (int)((c == 2 ? P.facade_down_fixed_num : P.beam_down_fixed_num) / sector_num);
        const uint32_t cloud0 = (c == 2) ? 20u : 24u;
        if ((long long)n <= (long long)keep) { // :554-555 untouched
            block_sample_append(in, n, -1, 0, 0, out, S);
        } else {
            float4 *sect = C.sect + (size_t)(c == 2 ? 0 : 1) * 3 * (size_t)C.n;
            const double angle_per_sector = 360.0 / sector_num;
            for (int j = 0; j < sector_num; ++j) {
                if (threadIdx.x == 0) s_sect = 0;
                __syncthreads();
                for (uint32_t tile = 0; tile < n; tile += kClsBlock) {
                    const uint32_t i = tile + threadIdx.x;
                    bool mine = false;
                    if (i < n) {
                        const float4 nb = in[3 * (size_t)i + 1];
                        // std::atan2(float, float) is the float overload: the angle is rounded to float before the
                        // double wrap. On a boundary that decides the sector: (+-0, -1) is float(+-pi), sector 2 / 1,
                        // and (0, -1) is -float(pi / 2), whose wrap lies below 270 degrees, sector 2.
                        double ang = (double)(float)atan2((double)nb.y, (double)nb.x);
                        if (ang < 0) ang += 2 * M_PI;
                        ang *= (180.0 / M_PI);
                        int sid = (int)(ang / angle_per_sector);
                        if (sid >= sector_num) sid = sector_num - 1;
                        mine = sid == j;
                    }
                    const uint32_t slot = map_tile_slot(mine, s_warp2, &s_sect);
                    if (mine) {
                        const float4 *r = in + 3 * (size_t)i;
                        float4 *o = sect + 3 * (size_t)slot;
                        o[0] = r[0], o[1] = r[1], o[2] = r[2];
                    }
                }
                __syncthreads();
                block_sample_append(sect, s_sect, keep, P.random_seed, cloud0 + (uint32_t)j, out, S);
            }
        }
    }
    if (threadIdx.x == 0) C.st->n_down2[c] = S.total;
}

} // namespace mulls
