// ref_shim_dbscan stub (test infrastructure): the part of geometry::PointCloud that ClusterDBSCAN reads, its points_,
// and the declaration of ClusterDBSCAN (geometry/PointCloud.h) that PointCloudCluster.cpp defines.
#pragma once
#include <array>
#include <cstddef>
#include <vector>
namespace open3d {
namespace geometry {
class PointCloud {
public:
    std::vector<std::array<double, 3>> points_;
    std::vector<int> ClusterDBSCAN(double eps, std::size_t min_points, bool print_progress = false) const;
};
}  // namespace geometry
}  // namespace open3d
