// TEST INFRASTRUCTURE, NOT PRODUCT CODE. CPU restatement of lo::CRegistration<PointT>::coarse_reg_ransac
// (include/common/cregistration.hpp:604-661), the checker of mulls_coarse_reg_ransac. Restated line by line on 48-byte
// pcl::PointXYZINormal rows: CorrespondenceRejectorSampleConsensus::getRemainingCorrespondences,
// RandomSampleConsensus::computeModel and SampleConsensus::refineModel of PCL 1.10, sequentially. The readings and
// the pieces both sides must compute alike (sample stream, Umeyama fit, transform-and-compare, summation order, the
// adaptive-k walk) come from mulls_b200/csrc/ransac_core.cuh and run here on the host; the median is std::nth_element
// as in SampleConsensusModel::computeVariance. Besides the result it reports the sample triples, the count of every
// hypothesis, the best hypothesis and the sizes of prev_inliers at the start of each refinement round.
// Built by tests/test_ransac.py with nvcc as host code (-x cu), host flags -O2 -ffp-contract=off.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../mulls_b200/csrc/ransac_core.cuh"

using namespace mulls;

namespace {

struct Model { // SampleConsensusModelRegistration over the correspondences i <-> i
    const float *src, *tgt;
    size_t n;
    std::vector<float> c6; // sx sy sz tx ty tz
    void fit(const std::vector<int> &inliers, float T[12]) const { // optimizeModelCoefficients
        std::vector<uint8_t> flag(n, 0);
        for (int i : inliers) flag[i] = 1;
        double ms[6], mean[6], cs[9];
        auto in = [&](int j) { return flag[j] != 0; };
        rc_sums_serial<6>((int)n, in, [&](int j, double x[6]) { rc_point_terms(&c6[6 * (size_t)j], x); }, ms);
        const double one_over_n = 1.0 / (double)inliers.size();
        rc_umeyama_means(ms, one_over_n, mean);
        rc_sums_serial<9>((int)n, in, [&](int j, double x[9]) { rc_cross_terms(&c6[6 * (size_t)j], mean, x); }, cs);
        rc_umeyama_finish(mean, cs, one_over_n, T);
    }
    int count(const float T[12], double threshold) const { // countWithinDistance
        const double thresh = threshold * threshold;
        int nr_p = 0;
        for (size_t i = 0; i < n; ++i)
            if (rc_within(T, &c6[6 * i], thresh)) nr_p++;
        return nr_p;
    }
    void select(const float T[12], double threshold, std::vector<int> &inliers, std::vector<double> &errs) const {
        const double thresh = threshold * threshold;
        inliers.clear();
        errs.clear();
        for (size_t i = 0; i < n; ++i) {
            const float distance = rc_sq_error(T, &c6[6 * i]);
            if ((double)distance < thresh) {
                inliers.push_back((int)i);
                errs.push_back((double)distance);
            }
        }
    }
};

double compute_variance(std::vector<double> dists) { // SampleConsensusModel::computeVariance
    const size_t medIdx = dists.size() >> 1;
    std::nth_element(dists.begin(), dists.begin() + medIdx, dists.end());
    return 2.1981 * dists[medIdx];
}

struct Trace {
    int *samples;
    long samples_cap;
    int *counts;
    int *sizes;
    int sizes_cap;
    int n_sizes = 0;
    int best = -1;
};

} // namespace

extern "C" {

// returns 0; status / n_inliers / n_hypotheses as mulls_coarse_reg_ransac; tran written when status >= 0
int orc_ransac(const float *t48, long nt, const float *s48, long ns, float noise_bound, int min_inlier_num, int max_iter_num,
               double *tran_mat, int *status, int *n_inliers, int *n_hypotheses, int *samples_out, long samples_cap,
               int *counts_out, int *sizes_out, int sizes_cap, int *n_sizes, int *best_out) {
    Trace tr{samples_out, samples_cap, counts_out, sizes_out, sizes_cap};
    const size_t N = (size_t)nt;
    (void)ns;
    float best_transformation[12] = {1.f, 0.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 0.f, 1.f, 0.f}; // uninitialised in PCL
    size_t remaining = 0;
    int iterations = 0;
    if (N > 0) { // getCorrespondences: an empty input returns at once
        Model model{s48, t48, N, std::vector<float>(N * 6)};
        for (size_t i = 0; i < N; ++i)
            for (int c = 0; c < 3; ++c) model.c6[6 * i + c] = s48[12 * i + c], model.c6[6 * i + 3 + c] = t48[12 * i + c];
        std::vector<int> shuffled(N);
        for (size_t i = 0; i < N; ++i) shuffled[i] = (int)i;
        SacSampler sampler{SacMt19937(), shuffled.data(), N, s48, rc_sample_dist_threshold(s48, N)};
        const double threshold_ = noise_bound;
        // ---- RandomSampleConsensus::computeModel ----
        SacWalk W(N, max_iter_num);
        float model_coefficients_[12];
        bool have_model = false;
        while (W.wants()) {
            int sel[3];
            if (!sampler.draw(sel)) break; // No samples could be selected
            float T[12];
            rc_fit_sample(model.c6.data(), sel, T);
            const int n_inliers_count = model.count(T, threshold_);
            const int h = W.iterations;
            if (h < tr.samples_cap) {
                std::memcpy(tr.samples + 3 * (size_t)h, sel, sizeof(sel));
                tr.counts[h] = n_inliers_count;
            }
            W.take(n_inliers_count);
            if (W.best == h) {
                std::memcpy(model_coefficients_, T, sizeof(T));
                have_model = true;
            }
        }
        iterations = W.iterations;
        tr.best = W.best;
        bool ok = have_model;
        std::vector<int> inliers_;
        std::vector<double> err_;
        if (ok) model.select(model_coefficients_, threshold_, inliers_, err_);
        if (!ok) { // computeModel failed: all correspondences, identity
            remaining = N;
        } else {
            // ---- SampleConsensus::refineModel(3, 1000) ----
            const double inlier_distance_threshold_sqr = threshold_ * threshold_;
            double error_threshold = threshold_;
            const double sigma_sqr = kRcRefineSigma * kRcRefineSigma;
            unsigned refine_iterations = 0;
            const unsigned max_iterations = kRcRefineRounds;
            bool inlier_changed = false, oscillating = false;
            std::vector<int> new_inliers, prev_inliers = inliers_;
            std::vector<double> errs;
            std::vector<size_t> inliers_sizes;
            float new_model_coefficients[12];
            std::memcpy(new_model_coefficients, model_coefficients_, sizeof(new_model_coefficients));
            do {
                model.fit(prev_inliers, new_model_coefficients);
                inliers_sizes.push_back(prev_inliers.size());
                if (tr.n_sizes < tr.sizes_cap) tr.sizes[tr.n_sizes] = (int)prev_inliers.size();
                tr.n_sizes++;
                model.select(new_model_coefficients, error_threshold, new_inliers, errs);
                if (new_inliers.empty()) {
                    refine_iterations++;
                    if (refine_iterations >= max_iterations) break;
                    continue;
                }
                const double variance = compute_variance(errs);
                error_threshold = sqrt(std::min(inlier_distance_threshold_sqr, sigma_sqr * variance));
                inlier_changed = false;
                std::swap(prev_inliers, new_inliers);
                if (new_inliers.size() != prev_inliers.size()) {
                    if (inliers_sizes.size() >= 4) {
                        if (inliers_sizes[inliers_sizes.size() - 1] == inliers_sizes[inliers_sizes.size() - 3] &&
                            inliers_sizes[inliers_sizes.size() - 2] == inliers_sizes[inliers_sizes.size() - 4]) {
                            oscillating = true;
                            break;
                        }
                    }
                    inlier_changed = true;
                    continue;
                }
                for (size_t i = 0; i < prev_inliers.size(); ++i)
                    if (prev_inliers[i] != new_inliers[i]) {
                        inlier_changed = true;
                        break;
                    }
            } while (inlier_changed && ++refine_iterations < max_iterations);
            bool refined;
            if (new_inliers.empty()) refined = false;
            else if (oscillating) refined = true;
            else if (!inlier_changed) {
                std::swap(inliers_, new_inliers);
                std::memcpy(model_coefficients_, new_model_coefficients, sizeof(new_model_coefficients));
                refined = true;
            } else refined = false;
            // ---- back in getRemainingCorrespondences ----
            if (!refined) {
                remaining = 0; // "Returning an empty solution"; best_transformation_ untouched
            } else if (inliers_.size() < 3) {
                remaining = N;
            } else {
                remaining = inliers_.size();
                std::memcpy(best_transformation, model_coefficients_, sizeof(best_transformation));
            }
        }
    }
    // ---- coarse_reg_ransac ----
    int stat = -1;
    if (remaining >= (size_t)(int64_t)min_inlier_num) {
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 4; ++c) tran_mat[4 * r + c] = (double)best_transformation[4 * r + c];
        tran_mat[12] = tran_mat[13] = tran_mat[14] = 0.0;
        tran_mat[15] = 1.0;
        stat = (remaining >= (size_t)(int64_t)(int32_t)((uint32_t)min_inlier_num * 2u)) ? 1 : 0;
    }
    *status = stat;
    *n_inliers = (int)remaining;
    *n_hypotheses = iterations;
    *n_sizes = tr.n_sizes;
    *best_out = tr.best;
    return 0;
}

// the first n outputs of the shared mt19937(12345) stream
void orc_mt_draws(uint32_t *out, long n) {
    SacMt19937 mt;
    for (long i = 0; i < n; ++i) out[i] = mt.next();
}
// the sample distance threshold of R1
double orc_sample_threshold(const float *s48, long n) { return rc_sample_dist_threshold(s48, (size_t)n); }

} // extern "C"
