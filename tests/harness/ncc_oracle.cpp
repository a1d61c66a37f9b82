// TEST INFRASTRUCTURE, NOT PRODUCT CODE. CPU restatement of lo::CRegistration<PointT>::find_feature_correspondence_ncc
// (include/common/cregistration.hpp:409-601), the checker of mulls_ncc_correspondences. Restated line by line on 48-byte
// pcl::PointXYZINormal rows (x y z data[3] | normal_x normal_y normal_z normal[3] | intensity curvature _ _), with the
// reference's types: float descriptors (Eigen::VectorXf there), a float distance table filled on up to six OpenMP
// threads, int pair indices. Instead of appending rows it reports the (target, source) row index of each appended pair.
// The readings (kernels_ncc.cuh states the same list):
//  1. fewer than 10 keypoints in either cloud: returns 0 (the reference's false), nothing is reported;
//  2. the intensity range uses the macros of utility.hpp:31-32 from FLT_MAX and 0, over the target only;
//  3. (int) of a float is the x86-64 conversion (cvttss2si: INT_MIN for NaN and out-of-range values), which is what g++
//     emits for this cast on x86-64; the digit pairs use C++ integer division and remainder;
//  4. the distance is the float sum in component order; built with -ffp-contract=off;
//  5-6. plain and reciprocal mode are the reference's loops as written;
//  7. fixed-number mode: std::sort's order of equal keys is left open by the reference; here std::stable_sort over the
//     pairs in push order (pair index i * n_s + j) with NaN after every number, i.e. the total order (distance, pair
//     index). NaN is undefined behaviour in the reference's comparator. n_t * n_s > INT_MAX returns -101 (the reference's
//     int pair index would overflow). corr_num = min_(corr_num, dist_array.size()) keeps the int / size_t comparison;
//  8. more pairs than `cap`: -101.
// Built by tests/test_ncc.py with the flags oracle/Makefile builds the oracle with (-O3 -fopenmp -ffp-contract=off).
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <utility>
#include <vector>

#ifdef _OPENMP
#include <omp.h>
#endif

#define max_(a, b) (((a) > (b)) ? (a) : (b)) // utility.hpp:31-32
#define min_(a, b) (((a) < (b)) ? (a) : (b))

namespace {

struct KptRow { // pcl::PointXYZINormal
    float data[4];
    float normal[4];
    float intensity, curvature, pad2, pad3;
};
static_assert(sizeof(KptRow) == 48, "48-byte rows");

typedef std::vector<float> Descriptor; // Eigen::VectorXf temp_descriptor(11)

// reading 3: the x86-64 conversion, written out so that it does not depend on what the compiler makes of an
// out-of-range cast
int x86_int(float f) { return (f >= -2147483648.0f && f < 2147483648.0f) ? (int)f : INT_MIN; }

Descriptor descriptor_of(const KptRow &p, float intensity_min, float intensity_max) {
    Descriptor temp_descriptor(11);
    int temp_descriptor_close = x86_int(p.normal[0]);
    int temp_descriptor_far = x86_int(p.normal[1]);
    temp_descriptor[0] = temp_descriptor_close / 1000000;
    temp_descriptor[1] = (temp_descriptor_close % 1000000) / 10000;
    temp_descriptor[2] = (temp_descriptor_close % 10000) / 100;
    temp_descriptor[3] = temp_descriptor_close % 100;
    temp_descriptor[4] = temp_descriptor_far / 1000000;
    temp_descriptor[5] = (temp_descriptor_far % 1000000) / 10000;
    temp_descriptor[6] = (temp_descriptor_far % 10000) / 100;
    temp_descriptor[7] = temp_descriptor_far % 100;
    float cur_i = p.intensity;
    temp_descriptor[8] = (cur_i - intensity_min) / (intensity_max - intensity_min) * 255.0;
    temp_descriptor[9] = p.normal[3] * 100;
    temp_descriptor[10] = p.data[3] * 30;
    return temp_descriptor;
}

// reading 7: NaN after every number, so that equal keys (and all NaNs) form the classes stable_sort keeps in order
bool dist_less(const std::pair<int, float> &a, const std::pair<int, float> &b) {
    if (std::isnan(a.second)) return false;
    if (std::isnan(b.second)) return true;
    return a.second < b.second;
}

} // namespace

extern "C" {

// returns 1 (performed), 0 (fewer than 10 keypoints) or -101; threads 0: min(6, every core) as the reference
int orc_ncc(const float *target_rows, long target_n, const float *source_rows, long source_n, int fixed_num_corr, int corr_num,
            int reciprocal_on, int threads, int32_t *tgt_idx, int32_t *src_idx, size_t cap, size_t *n_out) {
    const KptRow *target_kpts = reinterpret_cast<const KptRow *>(target_rows);
    const KptRow *source_kpts = reinterpret_cast<const KptRow *>(source_rows);
    *n_out = 0;
    int target_kpts_num = (int)target_n;
    int source_kpts_num = (int)source_n;
    float dist_margin_thre = 0.0;
    if (target_kpts_num < 10 || source_kpts_num < 10)
        return 0;
    if (fixed_num_corr && (long long)target_kpts_num * source_kpts_num > INT_MAX)
        return -101;
    std::vector<std::pair<int32_t, int32_t>> corrs;

    float intensity_min = FLT_MAX;
    float intensity_max = 0;
    for (int i = 0; i < target_kpts_num; i++) {
        float cur_i = target_kpts[i].intensity;
        intensity_min = min_(intensity_min, cur_i);
        intensity_max = max_(intensity_max, cur_i);
    }
    std::vector<Descriptor> target_kpts_descriptors, source_kpts_descriptors;
    for (int i = 0; i < target_kpts_num; i++)
        target_kpts_descriptors.push_back(descriptor_of(target_kpts[i], intensity_min, intensity_max));
    for (int i = 0; i < source_kpts_num; i++)
        source_kpts_descriptors.push_back(descriptor_of(source_kpts[i], intensity_min, intensity_max));

    std::vector<std::vector<float>> dist_table(target_kpts_num);
    for (int i = 0; i < target_kpts_num; i++)
        dist_table[i].resize(source_kpts_num);
    std::vector<std::pair<int, float>> dist_array;
#ifdef _OPENMP
    const int nt = threads > 0 ? threads : min_(6, omp_get_max_threads());
#else
    const int nt = 1;
#endif
#pragma omp parallel for num_threads(nt) if (nt > 1)
    for (int i = 0; i < target_kpts_num; i++) {
        for (int j = 0; j < source_kpts_num; j++) {
            for (int k = 0; k < 11; k++)
                dist_table[i][j] += std::abs(target_kpts_descriptors[i][k] - source_kpts_descriptors[j][k]);
        }
    }
    if (!fixed_num_corr) {
        for (int i = 0; i < target_kpts_num; i++) {
            int min_dist_col_index = 0;
            float min_dist_row = FLT_MAX;
            for (int j = 0; j < source_kpts_num; j++) {
                if (dist_table[i][j] < min_dist_row) {
                    min_dist_row = dist_table[i][j];
                    min_dist_col_index = j;
                }
            }
            bool refined_corr = true;
            if (reciprocal_on) {
                for (int j = 0; j < target_kpts_num; j++) {
                    if (min_dist_row > dist_table[j][min_dist_col_index] + dist_margin_thre) {
                        refined_corr = false;
                        break;
                    }
                }
            }
            if (refined_corr)
                corrs.emplace_back(i, min_dist_col_index);
        }
    } else {
        for (int i = 0; i < target_kpts_num; i++) {
            for (int j = 0; j < source_kpts_num; j++) {
                std::pair<int, float> temp_pair;
                temp_pair.first = i * source_kpts_num + j;
                temp_pair.second = dist_table[i][j];
                dist_array.push_back(temp_pair);
            }
        }
        std::vector<std::vector<float>>().swap(dist_table); // freed before the sort rather than at :595: halves the peak
        std::stable_sort(dist_array.begin(), dist_array.end(), dist_less);
        corr_num = min_(corr_num, dist_array.size());

        std::vector<int> count_target_kpt(target_kpts_num, 0);
        std::vector<int> count_source_kpt(source_kpts_num, 0);
        int max_corr_num = 6;
        for (int k = 0; k < corr_num; k++) {
            int index = dist_array[k].first;
            int i = index / source_kpts_num;
            int j = index % source_kpts_num;
            if (count_target_kpt[i] > max_corr_num || count_source_kpt[j] > max_corr_num)
                continue;
            count_target_kpt[i]++;
            count_source_kpt[j]++;
            corrs.emplace_back(i, j);
        }
    }
    if (corrs.size() > cap)
        return -101;
    for (size_t k = 0; k < corrs.size(); ++k)
        tgt_idx[k] = corrs[k].first, src_idx[k] = corrs[k].second;
    *n_out = corrs.size();
    return 1;
}

} // extern "C"
