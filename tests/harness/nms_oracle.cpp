// TEST INFRASTRUCTURE, NOT PRODUCT CODE. CPU restatement of lo::CFilter<PointT>::non_max_suppress, the in-place overload
// (include/common/cfilter.hpp:1183-1240) that test/mulls_reg.cpp:147-148 and test/mulls_slam.cpp:462 call; the checker of
// mulls_non_max_suppress. oracle/mulls_oracle.cpp is included here, not copied or changed: its kd-tree (KdTree, the
// stand-in for FLANN's KDTreeSingleIndex) gives the radius candidates, and its FLANN distance decides them. The readings
// are those abi.h states for mulls_non_max_suppress. Nothing of the library is included.
// Built by tests/test_nms.py with the flags oracle/Makefile builds the oracle with (-O3 -fopenmp -ffp-contract=off).
#include "../../oracle/mulls_oracle.cpp"

namespace {

// every point of the tree whose box distance to q does not rule it out: a superset of the points with flann_l2 < r2.
// The box distance is in double, exact for float boxes; the float FLANN sum can lie below the true squared distance by a
// few units in its last place (and by a subnormal's worth where a square underflows), so the bound keeps a margin.
void radius_candidates(const KdTree &t, int node, const double q[3], double lo[3], double hi[3], double bound,
                       std::vector<int> &out) {
    double d2 = 0;
    for (int d = 0; d < 3; ++d) {
        const double e = q[d] < lo[d] ? lo[d] - q[d] : (q[d] > hi[d] ? q[d] - hi[d] : 0.0);
        d2 += e * e;
    }
    if (d2 > bound) return;
    const KdNode &nd = t.nodes[node];
    if (nd.dim < 0) {
        for (int k = nd.left; k < nd.right; ++k) out.push_back(t.idx[k]);
        return;
    }
    const double save_hi = hi[nd.dim], save_lo = lo[nd.dim];
    hi[nd.dim] = nd.lo; // the left child holds the coordinates <= lo along dim
    radius_candidates(t, nd.left, q, lo, hi, bound, out);
    hi[nd.dim] = save_hi;
    lo[nd.dim] = nd.hi; // the right child those >= hi
    radius_candidates(t, nd.right, q, lo, hi, bound, out);
    lo[nd.dim] = save_lo;
}

bool finite3(const float *r) { return std::isfinite(r[0]) && std::isfinite(r[1]) && std::isfinite(r[2]); }

// cfilter.hpp:1183-1240 on 48-byte rows; `order` receives the input positions of the rows the cloud keeps, in order
bool non_max_suppress_in_place(const float *rows, long n, float non_max_radius, std::vector<int> &order) {
    order.clear();
    if (n < 10) return false; // :1189-1191, the cloud stays unsorted
    // std::sort by normal[3] (float 7), descending: equal scores in input order, +0 == -0 (the float comparison), NaN
    // after every number in input order
    std::vector<int> perm(n);
    for (long i = 0; i < n; ++i) perm[i] = (int)i;
    std::stable_sort(perm.begin(), perm.end(), [&](int a, int b) {
        const float sa = rows[12 * (size_t)a + 7], sb = rows[12 * (size_t)b + 7];
        if (std::isnan(sa) || std::isnan(sb)) return !std::isnan(sa) && std::isnan(sb);
        return sa > sb;
    });
    // the sorted cloud; the tree holds its finite points (a non-finite point is within the radius of no point)
    Cloud S(n), F;
    std::vector<int> fpos;
    for (long k = 0; k < n; ++k) {
        const float *r = rows + 12 * (size_t)perm[k];
        S[k] = Pt{r[0], r[1], r[2], r[4], r[5], r[6], r[8], r[9]};
        if (finite3(r)) F.push_back(S[k]), fpos.push_back((int)k);
    }
    KdTree tree;
    tree.build(F);
    const float r2 = (float)((double)non_max_radius * (double)non_max_radius);
    const double bound = (double)r2 * (1.0 + 1e-5) + 1e-40;
    std::vector<char> visited(n, 0);
    std::vector<int> cand;
    for (long id = 0; id < n; ++id) {
        if (visited[id]) continue;
        order.push_back(perm[id]); // cloud_temp->points.push_back(cloud_in_out->points[id])
        visited[id] = 1;
        const float q[3] = {S[id].x, S[id].y, S[id].z};
        if (F.empty() || !std::isfinite(q[0]) || !std::isfinite(q[1]) || !std::isfinite(q[2]) || !(r2 > 0.f)) continue;
        // radiusSearch(points[id], non_max_radius): every point j with flann_l2(q, j) < r2 is visited
        cand.clear();
        const double qd[3] = {q[0], q[1], q[2]};
        double lo[3], hi[3];
        for (int d = 0; d < 3; ++d) lo[d] = tree.bmin[d], hi[d] = tree.bmax[d];
        radius_candidates(tree, 0, qd, lo, hi, bound, cand);
        for (int f : cand)
            if (KdTree::flann_l2(q, F[f]) < r2) visited[fpos[f]] = 1;
    }
    return true;
}

} // namespace

extern "C" {

// kept_idx [cloud.n]: the input row indices the cloud keeps, in order; *performed: what the member returns
int orc_non_max_suppress(const mulls_cloud_view cloud, float non_max_radius, int32_t *kept_idx, size_t *n_kept, int *performed) {
    std::vector<int> order;
    const bool ran = non_max_suppress_in_place(cloud.aos48, (long)cloud.n, non_max_radius, order);
    for (size_t k = 0; k < order.size(); ++k) kept_idx[k] = order[k];
    *n_kept = order.size();
    *performed = ran ? 1 : 0;
    return 0;
}

} // extern "C"
