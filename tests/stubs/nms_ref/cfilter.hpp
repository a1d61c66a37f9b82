// TEST STAND-IN for the reference's include/common/cfilter.hpp with the three non_max_suppress overloads
// (cfilter.hpp:1183, :1243, :1314) and the pcl::search::KdTree pointer they take: what tests/stubs/nms_caller.cpp
// needs to show which calls the drop-in keeps and which reach the reference. The other stand-ins come from
// tests/stubs/utility.hpp, as for ref/cfilter.hpp.
#ifndef STUB_REFERENCE_NMS_CFILTER_HPP
#define STUB_REFERENCE_NMS_CFILTER_HPP
#include <vector>

#include "../utility.hpp"

namespace pcl {
namespace search {
template <typename P>
struct KdTree {
    typedef boost::shared_ptr<KdTree<P>> Ptr;
};
} // namespace search
struct PointIndices {};
typedef boost::shared_ptr<PointIndices> PointIndicesPtr;
} // namespace pcl

namespace lo {
struct pca_feature_t {};
template <typename PointT>
class CFilter {
  public:
    bool non_max_suppress(typename pcl::PointCloud<PointT>::Ptr &, float, bool = false,
                          const typename pcl::search::KdTree<PointT>::Ptr & = NULL) {
        reference_nms_ran = 1183;
        return false;
    }
    bool non_max_suppress(typename pcl::PointCloud<PointT>::Ptr &, typename pcl::PointCloud<PointT>::Ptr &, float, bool = false,
                          float = 35.0, bool = false, const typename pcl::search::KdTree<PointT>::Ptr & = NULL) {
        reference_nms_ran = 1243;
        return false;
    }
    bool non_max_suppress(std::vector<pca_feature_t> &, pcl::PointIndicesPtr &, float) {
        reference_nms_ran = 1314;
        return false;
    }
    bool reference_body_ran = false;
    int reference_nms_ran = 0; // the line of the reference overload that ran last
};
} // namespace lo
#endif
