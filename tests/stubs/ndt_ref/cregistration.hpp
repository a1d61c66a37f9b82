// TEST STAND-IN for the reference's include/common/cregistration.hpp with its omp_ndt (cregistration.hpp:945-1021):
// the members of tests/stubs/ref/cregistration.hpp plus omp_ndt, whose body marks that the reference member ran. Used
// only by tests/stubs/ndt_caller.cpp (tests/test_ndt.py, tests/test_gpu_ndt.py).
#ifndef STUB_REFERENCE_CREGISTRATION_HPP
#define STUB_REFERENCE_CREGISTRATION_HPP
#include <string>

#include "utility.hpp"

namespace lo {
template <typename PointT>
class CRegistration {
  public:
    int mm_lls_icp(constraint_t &, int = 20, float = 1.5, float = 0.002, float = 0.01, float = 0.4, float = 1.1,
                   std::string = "111110", std::string = "1101", float = 1.0, float = 0.1, float = 0.1, float = 0.1,
                   Eigen::Matrix4d = Eigen::Matrix4d::Identity(), bool = true, bool = false, bool = false, float = 45.0,
                   bool = false, bool = false, float = 0.5, float = 0.03, float = 45.0) {
        return -99; // the reference's CPU body
    }
    bool mm_lls_icp_4dof_global(constraint_t &, float, int = 20, float = 1.5, float = 0.005, float = 0.05, float = 0.5,
                                float = 1.05, float = 15.0) {
        return false;
    }
    bool determine_source_target_cloud(const cloudblock_Ptr &block_1, const cloudblock_Ptr &block_2, constraint_t &registration_cons) {
        const bool first = block_1->down_feature_point_num > block_2->down_feature_point_num;
        registration_cons.block1 = first ? block_1 : block_2;
        registration_cons.block2 = first ? block_2 : block_1;
        return true;
    }
    bool assign_source_target_cloud(const cloudblock_Ptr &block_1, const cloudblock_Ptr &block_2, constraint_t &registration_cons) {
        registration_cons.block1 = block_1;
        registration_cons.block2 = block_2;
        return true;
    }
    bool coarse_reg_ransac(int marker) { return marker == 7; } // "inherited, untouched"
    int omp_ndt(constraint_t &registration_cons, float = 1.0, bool = true, Eigen::Matrix4d = Eigen::Matrix4d::Identity(),
                bool = true, float = 10.0) {
        registration_cons.Trans1_2(0, 3) = 77.0;
        return -77; // the reference's CPU body
    }
};
} // namespace lo
#endif
