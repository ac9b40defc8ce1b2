// ref_shim_segment stub (test infrastructure): the part of geometry::PointCloud that SegmentPlane reads, its points_,
// and the declaration of SegmentPlane (geometry/PointCloud.h) that PointCloudSegmentation.cpp defines.
#pragma once
#include <Eigen/Dense>
#include <atomic>
#include <cmath>
#include <cstddef>
#include <limits>
#include <mutex>
#include <tuple>
#include <vector>
namespace open3d {
namespace geometry {
class PointCloud {
public:
    std::vector<Eigen::Vector3d> points_;
    std::tuple<Eigen::Vector4d, std::vector<size_t>> SegmentPlane(const double distance_threshold = 0.01,
                                                                  const int ransac_n = 3,
                                                                  const int num_iterations = 100,
                                                                  const double probability = 0.99999999) const;
};
}  // namespace geometry
}  // namespace open3d
