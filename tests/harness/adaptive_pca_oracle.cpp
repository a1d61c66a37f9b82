// TEST INFRASTRUCTURE, NOT PRODUCT CODE. CPU restatement of distance-adaptive PCA neighbourhoods, the checker of
// mulls_pca_features_adaptive and of mulls_classify_nground / mulls_extract_semantic_pts with use_distance_adaptive_pca:
// lo::PrincipleComponentAnalysis<PointT>::get_pc_pca_feature with distance_adaptive_on (include/common/pca.hpp:310-326),
// as lo::CFilter<PointT>::classify_nground_pts calls it (cfilter.hpp:2093, unit_distance 30).
// oracle/mulls_oracle.cpp is included here, not changed: classify_nground_adaptive below is the oracle's classify_nground
// with its PCA call taken through pca_core_adaptive, everything after the PCA is the oracle's text. With unit_dist <= 0
// the search is the fixed radius, and the classification equals the oracle's bit for bit (tests/test_adaptive_pca.py
// checks that). Nothing of the library is included.
// Built by tests/test_adaptive_pca.py with the flags oracle/Makefile builds the oracle with (-O3 -fopenmp -ffp-contract=off).
#include "../../oracle/mulls_oracle.cpp"

#include <unordered_map>

namespace {

// pca.hpp:310-326: double dist = std::sqrt(x*x + y*y + z*z) on the float coordinates (the float overload, widened);
// if (dist > unit_dist) neighborhood_r = std::sqrt(dist / unit_dist) * radius, narrowed to float.
static float adaptive_radius(const Pt &p, float radius, float unit_dist) {
    const double dist = std::sqrt(p.x * p.x + p.y * p.y + p.z * p.z);
    if (dist > unit_dist) return (float)(std::sqrt(dist / unit_dist) * radius);
    return radius;
}

// pca_core (oracle) with a radius per query: unit_dist > 0 adapts it, else every query searches `radius`. Brute force
// through a hashed uniform grid of base-radius cells, so clouds kilometres wide stay cheap.
static int pca_core_adaptive(const Cloud &C, float radius, int k, int stride, float unit_dist, mulls_pca_out *out,
                             std::vector<NbrList> *lists) {
    const long n = (long)C.size();
    float mn[3] = {1e30f, 1e30f, 1e30f};
    for (long i = 0; i < n; ++i) {
        mn[0] = std::min(mn[0], C[i].x);
        mn[1] = std::min(mn[1], C[i].y);
        mn[2] = std::min(mn[2], C[i].z);
    }
    const double h = radius;
    auto cell_of = [&](const Pt &p, long long c[3]) {
        c[0] = (long long)std::floor((p.x - (double)mn[0]) / h);
        c[1] = (long long)std::floor((p.y - (double)mn[1]) / h);
        c[2] = (long long)std::floor((p.z - (double)mn[2]) / h);
    };
    auto key_of = [](long long x, long long y, long long z) { return (x * 2097152LL + y) * 2097152LL + z; };
    std::unordered_map<long long, std::vector<int>> cells;
    for (long i = 0; i < n; ++i) {
        long long c[3];
        cell_of(C[i], c);
        cells[key_of(c[0], c[1], c[2])].push_back((int)i);
    }
    if (lists) lists->assign((size_t)n, NbrList());
    for (long i = 0; i < n; ++i) {
        out->pt_num[i] = 0;
        for (int d = 0; d < 3; ++d) out->eigenvalues[3 * i + d] = out->principal[3 * i + d] = out->normal[3 * i + d] = 0.f;
    }
#pragma omp parallel for schedule(dynamic, 16)
    for (long i = 0; i < n; i += stride) {
        const float r = unit_dist > 0.f ? adaptive_radius(C[i], radius, unit_dist) : radius;
        const float r2 = (float)((double)r * (double)r); // KdTreeFLANN::radiusSearch casts radius*radius to float
        const long long span = (long long)std::ceil((double)r / h) + 1;
        long long c[3];
        cell_of(C[i], c);
        std::vector<std::pair<float, int>> nb;
        const float q[3] = {C[i].x, C[i].y, C[i].z};
        for (long long dz = -span; dz <= span; ++dz)
            for (long long dy = -span; dy <= span; ++dy)
                for (long long dx = -span; dx <= span; ++dx) {
                    const auto it = cells.find(key_of(c[0] + dx, c[1] + dy, c[2] + dz));
                    if (it == cells.end()) continue;
                    for (int j : it->second) {
                        const float d2 = KdTree::flann_l2(q, C[j]);
                        if (d2 < r2) nb.push_back(std::make_pair(d2, j)); // FLANN result sets keep dist < radius
                    }
                }
        std::sort(nb.begin(), nb.end());
        if (k > 0 && (int)nb.size() > k) nb.resize(k);
        const int m = (int)nb.size();
        out->pt_num[i] = m;
        if (lists) (*lists)[i] = nb;
        if (m <= 3) continue; // pca.hpp:396-397
        // pcl::PCA: float centroid, float covariance / (n-1), as the oracle's pca_core
        float mu[3] = {0, 0, 0};
        for (int t = 0; t < m; ++t) {
            mu[0] += C[nb[t].second].x;
            mu[1] += C[nb[t].second].y;
            mu[2] += C[nb[t].second].z;
        }
        mu[0] /= (float)m;
        mu[1] /= (float)m;
        mu[2] /= (float)m;
        float cov[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
        for (int t = 0; t < m; ++t) {
            float d[3] = {C[nb[t].second].x - mu[0], C[nb[t].second].y - mu[1], C[nb[t].second].z - mu[2]};
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b) cov[a][b] += d[a] * d[b];
        }
        double A[3][3], w[3], V[3][3];
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) A[a][b] = (double)(cov[a][b] / (float)(m - 1));
        jacobi_eig3(A, w, V);
        int ord[3] = {0, 1, 2};
        std::sort(ord, ord + 3, [&](int a, int b) { return w[a] > w[b]; });
        double e0[3] = {V[0][ord[0]], V[1][ord[0]], V[2][ord[0]]};
        double e1[3] = {V[0][ord[1]], V[1][ord[1]], V[2][ord[1]]};
        double e2[3] = {e0[1] * e1[2] - e0[2] * e1[1], e0[2] * e1[0] - e0[0] * e1[2], e0[0] * e1[1] - e0[1] * e1[0]};
        double n0 = std::sqrt(e0[0] * e0[0] + e0[1] * e0[1] + e0[2] * e0[2]);
        double n2 = std::sqrt(e2[0] * e2[0] + e2[1] * e2[1] + e2[2] * e2[2]);
        for (int d = 0; d < 3; ++d) {
            out->eigenvalues[3 * i + d] = (float)w[ord[d]];
            out->principal[3 * i + d] = (float)(e0[d] / n0);
            out->normal[3 * i + d] = (float)(e2[d] / n2);
        }
    }
    return 0;
}

// oracle/mulls_oracle.cpp classify_nground (cfilter.hpp:2058-2290) with the adaptive PCA. The close / far split keeps
// the base radius (pca.hpp:337) and the NMS does not adapt (cfilter.hpp:2233-2256): both stay as the oracle states them.
static void classify_nground_adaptive(Rows &cloud_in, const mulls_classify_params &P, float unit_dist, Rows out[MULLS_OUT_COUNT]) {
    Rows &pillar = out[MULLS_OUT_PILLAR], &beam = out[MULLS_OUT_BEAM], &facade = out[MULLS_OUT_FACADE], &roof = out[MULLS_OUT_ROOF];
    Rows &pillar_down = out[MULLS_OUT_PILLAR_DOWN], &beam_down = out[MULLS_OUT_BEAM_DOWN],
         &facade_down = out[MULLS_OUT_FACADE_DOWN], &roof_down = out[MULLS_OUT_ROOF_DOWN], &vertex = out[MULLS_OUT_VERTEX];
    // :2086-2087
    if (P.fixed_num_downsampling) rows_random_downsample(cloud_in, P.unground_down_fixed_num, P.random_seed, 18);
    const int n = (int)cloud_in.size();
    // :2089-2097 get_pc_pca_feature(cloud_in, features, tree, radius, k, 1, pca_down_rate, ...)
    Cloud C(n);
    for (int i = 0; i < n; ++i) {
        Pt p = {cloud_in[i].f[RX], cloud_in[i].f[RY], cloud_in[i].f[RZ], 0, 0, 0, 0, 0};
        C[i] = p;
    }
    std::vector<float> ev(3 * (size_t)n + 1), pr(3 * (size_t)n + 1), nr(3 * (size_t)n + 1);
    std::vector<int32_t> cnt((size_t)n + 1);
    mulls_pca_out po = {ev.data(), pr.data(), nr.data(), cnt.data()};
    std::vector<NbrList> lists;
    const int stride = P.pca_down_rate > 0 ? P.pca_down_rate : 1;
    pca_core_adaptive(C, P.neighbor_searching_radius, P.neighbor_k, stride, unit_dist, &po, &lists); // the one change
    std::vector<PcaFeat> feat(n);
    const float radius = P.neighbor_searching_radius;
    for (int i = 0; i < n; i += stride) {
        PcaFeat &f = feat[i];
        f.pt_num = cnt[i];
        if (f.pt_num > 3) { // get_pca_feature, pca.hpp:390-434
            const double l1 = ev[3 * i], l2 = ev[3 * i + 1], l3 = ev[3 * i + 2];
            f.curvature = ((l1 + l2 + l3) == 0) ? 0 : l3 / (l1 + l2 + l3);
            f.linear_2 = (l1 - l2) / l1;
            f.planar_2 = (l2 - l3) / l1;
            for (int d = 0; d < 3; ++d) f.pdir[d] = pr[3 * i + d], f.ndir[d] = nr[3 * i + d];
            f.nbr.resize(f.pt_num);
            f.close.resize(f.pt_num);
            for (int j = 0; j < f.pt_num; ++j) {
                f.nbr[j] = lists[i][j].second;
                f.close[j] = (lists[i][j].first < 0.64 * radius * radius) ? 1 : 0; // pca.hpp:337
            }
        }
        if (f.pt_num > 1) assign_normal(cloud_in[i], f, true); // min_k = 1, pca.hpp:346-347
    }
    // :2100-2166
    std::vector<int> index_with_feature(n, 0); // 0 none, 1 pillar, 2 beam, 3 facade, 4 roof
    for (int i = 0; i < n; ++i) {
        const PcaFeat &f = feat[i];
        if (f.pt_num > P.neigh_k_min) {
            if (f.linear_2 > P.edge_thre) {
                if (std::abs(f.pdir[2]) > P.linear_vertical_sin_high_thre) {
                    assign_normal(cloud_in[i], f, false);
                    pillar.push_back(cloud_in[i]);
                    index_with_feature[i] = 1;
                } else if (std::abs(f.pdir[2]) < P.linear_vertical_sin_low_thre && cloud_in[i].f[RZ] < P.beam_height_max) {
                    assign_normal(cloud_in[i], f, false);
                    beam.push_back(cloud_in[i]);
                    index_with_feature[i] = 2;
                }
                if (!P.sharpen_with_nms && f.linear_2 > P.edge_thre_down) {
                    if (std::abs(f.pdir[2]) > P.linear_vertical_sin_high_thre)
                        pillar_down.push_back(cloud_in[i]);
                    else if (std::abs(f.pdir[2]) < P.linear_vertical_sin_low_thre && cloud_in[i].f[RZ] < P.beam_height_max)
                        beam_down.push_back(cloud_in[i]);
                }
            } else if (f.planar_2 > P.planar_thre) {
                if (std::abs(f.ndir[2]) > P.planar_vertical_sin_high_thre && cloud_in[i].f[RZ] > P.roof_height_min) {
                    assign_normal(cloud_in[i], f, true);
                    roof.push_back(cloud_in[i]);
                    index_with_feature[i] = 4;
                } else if (std::abs(f.ndir[2]) < P.planar_vertical_sin_low_thre) {
                    assign_normal(cloud_in[i], f, true);
                    facade.push_back(cloud_in[i]);
                    index_with_feature[i] = 3;
                }
                if (!P.sharpen_with_nms && f.planar_2 > P.planar_thre_down) {
                    if (std::abs(f.ndir[2]) > P.planar_vertical_sin_high_thre && cloud_in[i].f[RZ] > P.roof_height_min)
                        roof_down.push_back(cloud_in[i]);
                    else if (std::abs(f.ndir[2]) < P.planar_vertical_sin_low_thre)
                        facade_down.push_back(cloud_in[i]);
                }
            }
        }
    }
    // :2169-2210
    int method = P.extract_vertex_points_method;
    if (P.curvature_thre < 1e-8) method = 0;
    if (method == 2) {
        const float vertex_feature_ratio_thre = P.feature_pts_ratio_guess / stride;
        for (int i = 0; i < n; ++i) {
            const PcaFeat &f = feat[i];
            if (index_with_feature[i] == 0 && f.pt_num > P.neigh_k_min && f.curvature > P.curvature_thre) {
                int geo_feature_point_count = 0;
                for (size_t j = 0; j < f.nbr.size(); ++j)
                    if (index_with_feature[f.nbr[j]]) geo_feature_point_count++;
                if (1.0 * geo_feature_point_count / f.pt_num > vertex_feature_ratio_thre) {
                    assign_normal(cloud_in[i], f, false);
                    cloud_in[i].f[RN3] = (float)(5.0 * f.curvature);
                    if (std::abs(f.pdir[2]) > P.linear_vertical_sin_high_thre) {
                        pillar.push_back(cloud_in[i]);
                        index_with_feature[i] = 1;
                    } else if (std::abs(f.pdir[2]) < P.linear_vertical_sin_low_thre && cloud_in[i].f[RZ] < P.beam_height_max) {
                        beam.push_back(cloud_in[i]);
                        index_with_feature[i] = 2;
                    }
                }
            }
        }
    }
    // :2219-2223 encode_stable_points (:1071-1181)
    {
        const int min_neighbor_feature_pts = (int)(P.feature_pts_ratio_guess / stride * P.neighbor_k) - 1;
        const float min_curvature = 0.3 * P.curvature_thre;
        for (int i = 0; i < n; ++i) {
            const PcaFeat &f = feat[i];
            if (f.pt_num > P.neigh_k_min && f.pt_num > 3 && f.curvature > min_curvature) {
                float accu_intensity = 0.0;
                Row pt = cloud_in[i];
                pt.f[RN3] = (float)f.curvature;
                int cnt_all[5] = {0, 0, 0, 0, 0}, cnt_close[5] = {0, 0, 0, 0, 0}, cnt_far[5] = {0, 0, 0, 0, 0};
                const int neighbor_total_count = (int)f.nbr.size();
                for (int j = 0; j < neighbor_total_count; ++j) {
                    const int lab = index_with_feature[f.nbr[j]];
                    if (lab >= 1 && lab <= 4) {
                        cnt_all[lab]++;
                        if (f.close[j])
                            cnt_close[lab]++;
                        else
                            cnt_far[lab]++;
                    }
                    accu_intensity += cloud_in[f.nbr[j]].f[RINT];
                }
                if (cnt_all[1] + cnt_all[2] + cnt_all[3] + cnt_all[4] < min_neighbor_feature_pts) continue;
                int a[5], c[5], r[5];
                for (int l = 1; l <= 4; ++l) {
                    a[l] = 100 * cnt_all[l] / neighbor_total_count;
                    c[l] = 100 * cnt_close[l] / neighbor_total_count;
                    r[l] = 100 * cnt_far[l] / neighbor_total_count;
                }
                const int descriptor = a[1] * 1000000 + a[2] * 10000 + a[3] * 100 + a[4];
                const int descriptor_1 = c[1] * 1000000 + c[2] * 10000 + c[3] * 100 + c[4];
                const int descriptor_2 = r[1] * 1000000 + r[2] * 10000 + r[3] * 100 + r[4];
                pt.f[RCURV] = descriptor;
                pt.f[RNX] = descriptor_1;
                pt.f[RNY] = descriptor_2;
                pt.f[RINT] = accu_intensity / neighbor_total_count;
                vertex.push_back(pt);
            }
        }
    }
    // :2229-2253
    if (P.sharpen_with_nms) {
        const float nms_radius = 0.25 * P.neighbor_searching_radius;
        if (P.pillar_down_fixed_num > 0) non_max_suppress(pillar, pillar_down, nms_radius);
        if (P.facade_down_fixed_num > 0) non_max_suppress(facade, facade_down, nms_radius);
        if (P.beam_down_fixed_num > 0) non_max_suppress(beam, beam_down, nms_radius);
        if (P.roof_down_fixed_num > 0) non_max_suppress(roof, roof_down, nms_radius);
    }
    // :2257-2267
    if (P.fixed_num_downsampling) {
        rows_random_downsample(pillar_down, P.pillar_down_fixed_num, P.random_seed, 19);
        const int sector_num = 4;
        xy_normal_balanced_downsample(facade_down, (int)(P.facade_down_fixed_num / sector_num), sector_num, P.random_seed, 20);
        xy_normal_balanced_downsample(beam_down, (int)(P.beam_down_fixed_num / sector_num), sector_num, P.random_seed, 24);
        rows_random_downsample(roof_down, P.roof_down_fixed_num, P.random_seed, 28);
    }
    out[MULLS_OUT_UNGROUND] = cloud_in;
}
} // namespace

extern "C" {

// get_pc_pca_feature(..., distance_adaptive_on = unit_dist > 0, unit_dist): outputs as orc_pca_features; `nbr` (optional,
// needs k >= 1) receives every query's neighbour list as radiusSearch returns it, [n][k] indices, -1 past pt_num.
int orc_pca_features_adaptive(const mulls_cloud_view cloud, float radius, int k, int stride, float unit_dist,
                              mulls_pca_out *out, int32_t *nbr) {
    if (stride < 1 || !(radius > 0.f) || (nbr && k < 1)) return MULLS_E_ARG;
    Cloud C;
    load_cloud(cloud, C);
    std::vector<NbrList> lists;
    pca_core_adaptive(C, radius, k, stride, unit_dist, out, nbr ? &lists : nullptr);
    if (nbr)
        for (size_t i = 0; i < C.size(); ++i)
            for (int t = 0; t < k; ++t) nbr[i * k + t] = t < (int)lists[i].size() ? lists[i][t].second : -1;
    return 0;
}

// orc_classify_nground with use_distance_adaptive_pca honoured: pca_unit_distance is the unit, and the flag without a
// positive unit is refused with MULLS_E_UNSUPPORTED, as mulls_classify_nground does.
int orc_classify_nground_adaptive(const mulls_cloud_view cloud_in, const mulls_classify_params *params, mulls_classify_out *out) {
    if (params->use_distance_adaptive_pca && !(params->pca_unit_distance > 0.f)) return MULLS_E_UNSUPPORTED;
    const float unit_dist = params->use_distance_adaptive_pca ? params->pca_unit_distance : 0.f;
    Rows in(cloud_in.n);
    if (cloud_in.n) std::memcpy(in.data(), cloud_in.aos48, cloud_in.n * sizeof(Row));
    Rows res[MULLS_OUT_COUNT];
    classify_nground_adaptive(in, *params, unit_dist, res);
    for (int k = 0; k < MULLS_OUT_COUNT; ++k) {
        out->n[k] = res[k].size();
        if (out->rows[k] && !res[k].empty()) std::memcpy(out->rows[k], res[k].data(), res[k].size() * sizeof(Row));
    }
    return 0;
}

} // extern "C"
