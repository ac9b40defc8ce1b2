// ref_shim_ransac stub (test infrastructure): the typedefs of utility/Eigen.h the registration files use, and
// TransformMatrix4dToVector6d, which CorrespondenceCheckerBasedOnSourceRotation calls (declared here, defined in the
// shim so that the file links; the tests never run that checker).
#pragma once
#include <Eigen/Core>
namespace Eigen {
typedef Matrix<double, 6, 6> Matrix6d;
typedef Matrix<double, 6, 1> Vector6d;
typedef Matrix<double, 4, 4, DontAlign> Matrix4d_u;
}  // namespace Eigen
namespace open3d {
namespace utility {
Eigen::Vector6d TransformMatrix4dToVector6d(const Eigen::Matrix4d& input);
}  // namespace utility
}  // namespace open3d
