// ref_shim_segment stub (test infrastructure): the declaration of TriangleMesh::ComputeTrianglePlane
// (geometry/TriangleMesh.h); ref_shim_segment.cpp defines it.
#pragma once
#include <Eigen/Dense>
namespace open3d {
namespace geometry {
class TriangleMesh {
public:
    static Eigen::Vector4d ComputeTrianglePlane(const Eigen::Vector3d& p0, const Eigen::Vector3d& p1,
                                                const Eigen::Vector3d& p2);
};
}  // namespace geometry
}  // namespace open3d
