// TEST INFRASTRUCTURE, NOT PRODUCT CODE. CPU restatement of lo::CFilter<PointT>::sor_filter (include/common/cfilter.hpp:
// 203-247) -> pcl::StatisticalOutlierRemoval (PCL 1.10, SURVEY Appendix B item 10), the checker of mulls_sor_filter.
// Its exact k-nearest search runs on the oracle's kd-tree (KdTree, the stand-in for FLANN's KDTreeSingleIndex):
// oracle/mulls_oracle.cpp is included here, not copied or changed. PCL's loops are restated verbatim; the queries may
// run on several OpenMP threads, the two sums stay sequential. Nothing of the library is included.
// Built by tests/test_sor.py with the flags oracle/Makefile builds the oracle with (-O3 -fopenmp -ffp-contract=off).
#include "../../oracle/mulls_oracle.cpp"

// ---------------------------------------------------------------------------------------------
// cfilter.hpp:203-247 sor_filter -> pcl::StatisticalOutlierRemoval<PointT>::applyFilterIndices (PCL 1.10) [3P], the
// searcher a pcl::search::KdTree<PointT>(false) (FLANN, exact, L2_Simple float distance). SURVEY Appendix B item 10.
// ---------------------------------------------------------------------------------------------
// `sqrt (nn_dists[k])` with float nn_dists, summed into a double: read as the double overload. The one place of that
// choice in the CPU restatement (kernels_sor.cuh has the device's).
static inline double sor_sqrt(float d2) { return std::sqrt(static_cast<double>(d2)); }

// exact k nearest neighbours on the oracle's kd-tree, any k: list ascending under the total order (d2, index)
struct SorKnn {
    int k = 0;
    std::vector<float> d2;
    std::vector<int> idx;
    float worst() const { return (int)d2.size() < k ? std::numeric_limits<float>::infinity() : d2.back(); }
    void insert(float d, int i) {
        const int n = (int)d2.size();
        if (n == k && !(d < d2[n - 1] || (d == d2[n - 1] && i < idx[n - 1]))) return;
        if (n == k) d2.pop_back(), idx.pop_back();
        int pos = (int)d2.size();
        while (pos > 0 && (d < d2[pos - 1] || (d == d2[pos - 1] && i < idx[pos - 1]))) --pos;
        d2.insert(d2.begin() + pos, d);
        idx.insert(idx.begin() + pos, i);
    }
};
static void sor_knn_rec(const KdTree &t, int node, const float q[3], float mindist, float dists[3], SorKnn &best) {
    const KdNode &nd = t.nodes[node];
    if (nd.dim < 0) {
        for (int k = nd.left; k < nd.right; ++k) best.insert(KdTree::flann_l2(q, (*t.pts)[t.idx[k]]), t.idx[k]);
        return;
    }
    const float val = q[nd.dim];
    const float diff1 = val - nd.lo, diff2 = val - nd.hi;
    int first, second;
    float cut;
    if (diff1 + diff2 < 0) {
        first = nd.left, second = nd.right, cut = diff2 * diff2;
    } else {
        first = nd.right, second = nd.left, cut = diff1 * diff1;
    }
    sor_knn_rec(t, first, q, mindist, dists, best);
    const float saved = dists[nd.dim];
    const float md = mindist + cut - saved;
    dists[nd.dim] = cut;
    if (md * 0.99999f <= best.worst()) sor_knn_rec(t, second, q, md, dists, best);
    dists[nd.dim] = saved;
}

// distances[] as PCL's, the statistics and the keep decision. Points with a non-finite coordinate never enter the tree
// (defined here; PCL would hand them to FLANN). MULLS_E_ARG for mean_k < 1 or at most mean_k finite points.
static int sor_filter(const Cloud &C, int mean_k, double std_mul, int threads, std::vector<float> &distances,
                      std::vector<uint8_t> &keep, mulls_sor_stats &st) {
    if (mean_k < 1) return MULLS_E_ARG;
    const long n = (long)C.size();
    Cloud F;
    for (long i = 0; i < n; ++i)
        if (std::isfinite(C[i].x) && std::isfinite(C[i].y) && std::isfinite(C[i].z)) F.push_back(C[i]);
    if ((long)F.size() <= (long)mean_k) return MULLS_E_ARG;
    std::vector<long> forig;
    for (long i = 0; i < n; ++i)
        if (std::isfinite(C[i].x) && std::isfinite(C[i].y) && std::isfinite(C[i].z)) forig.push_back(i);
    KdTree tree;
    tree.build(F);
    distances.assign(n, 0.0f); // invalid points: distances[iii] = 0
#ifdef _OPENMP
    const int nt = threads > 0 ? threads : omp_get_max_threads();
#else
    const int nt = 1;
#endif
#pragma omp parallel for schedule(dynamic, 256) num_threads(nt) if (nt > 1)
    for (long f = 0; f < (long)F.size(); ++f) {
        const float q[3] = {F[f].x, F[f].y, F[f].z};
        float dists[3] = {0, 0, 0};
        float mind = 0;
        for (int d = 0; d < 3; ++d) {
            if (q[d] < tree.bmin[d]) dists[d] = (q[d] - tree.bmin[d]) * (q[d] - tree.bmin[d]);
            if (q[d] > tree.bmax[d]) dists[d] = (q[d] - tree.bmax[d]) * (q[d] - tree.bmax[d]);
            mind += dists[d];
        }
        SorKnn nn;
        nn.k = mean_k + 1; // nearestKSearch (i, mean_k_ + 1, ...): position 0 is the point itself
        sor_knn_rec(tree, 0, q, mind, dists, nn);
        double dist_sum = 0;
        for (int k = 1; k < mean_k + 1; ++k) dist_sum += sor_sqrt(nn.d2[k]);
        distances[forig[f]] = static_cast<float>(dist_sum / mean_k);
    }
    // the two sums, sequential in index order; the product is the float one
    double sum = 0, sq_sum = 0;
    for (long i = 0; i < n; ++i) {
        sum += distances[i];
        sq_sum += distances[i] * distances[i];
    }
    const long valid_distances = (long)F.size();
    const double mean = sum / static_cast<double>(valid_distances);
    const double variance = (sq_sum - sum * sum / static_cast<double>(valid_distances)) / (static_cast<double>(valid_distances) - 1);
    const double stddev = std::sqrt(variance);
    const double distance_threshold = mean + std_mul * stddev;
    keep.assign(n, 0);
    uint64_t kept = 0;
    for (long i = 0; i < n; ++i) {
        if (distances[i] > distance_threshold) continue; // outlier (negative_ = false)
        keep[i] = 1;
        ++kept;
    }
    st.mean = mean;
    st.stddev = stddev;
    st.threshold = distance_threshold;
    st.n_valid = (uint64_t)valid_distances;
    st.n_kept = kept;
    return 0;
}

extern "C" {

// cfilter.hpp:203-247 (both overloads). keep_bits [(n+7)/8]: bit i % 8 of byte i / 8 set for a kept point; distances
// [n] or NULL; stats or NULL. threads: 0 = every core, n > 0 = n threads (1: reference-shaped). The sums stay sequential.
int orc_sor_filter(const mulls_cloud_view cloud, int mean_k, double n_std, uint8_t *keep_bits, float *distances,
                   mulls_sor_stats *stats, int threads) {
    Cloud C;
    load_cloud(cloud, C);
    std::vector<float> dist;
    std::vector<uint8_t> keep;
    mulls_sor_stats st;
    const int rc = sor_filter(C, mean_k, n_std, threads, dist, keep, st);
    if (rc != 0) return rc;
    std::memset(keep_bits, 0, (C.size() + 7) / 8);
    for (size_t i = 0; i < C.size(); ++i)
        if (keep[i]) keep_bits[i / 8] |= (uint8_t)(1u << (i % 8));
    if (distances) std::memcpy(distances, dist.data(), C.size() * sizeof(float));
    if (stats) *stats = st;
    return 0;
}

} // extern "C"
