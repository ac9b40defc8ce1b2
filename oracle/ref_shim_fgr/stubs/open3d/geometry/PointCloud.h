// ref_shim_fgr stub (test infrastructure): the legacy PointCloud with what the registration files use.  Transform
// is PointCloud::Transform's point and normal loops (geometry/Geometry3D.cpp TransformPoints / TransformNormals) in the
// stated product order: p = (T (x, y, z, 1)).head<3>() / w, n = (T (nx, ny, nz, 0)).head<3>().
#pragma once
#include <Eigen/Core>
#include "open3d/utility/Eigen.h"
#include <vector>
namespace open3d {
namespace geometry {
class PointCloud {
public:
    bool HasPoints() const { return !points_.empty(); }
    bool HasNormals() const { return !points_.empty() && normals_.size() == points_.size(); }
    PointCloud& Transform(const Eigen::Matrix4d& T) {
        for (auto& p : points_) {
            const Eigen::Vector4d q = T * Eigen::Vector4d(p(0), p(1), p(2), 1.0);
            p = q.head<3>() / q(3);
        }
        for (auto& n : normals_) {
            const Eigen::Vector4d q = T * Eigen::Vector4d(n(0), n(1), n(2), 0.0);
            n = q.head<3>();
        }
        return *this;
    }
    std::vector<Eigen::Vector3d> points_;
    std::vector<Eigen::Vector3d> normals_;
};
}  // namespace geometry
}  // namespace open3d
