// ref_shim_fgr stub (test infrastructure): the typedefs of utility/Eigen.h the registration files use, and the
// declarations of its functions they call: SolveLinearSystemPSD and TransformVector6dToMatrix4d (restated in the
// shim), TransformMatrix4dToVector6d (CorrespondenceCheckerBasedOnSourceRotation; defined in the shim so that the file
// links, never run).
#pragma once
#include <Eigen/Core>
#include <tuple>
namespace Eigen {
typedef Matrix<double, 6, 6> Matrix6d;
typedef Matrix<double, 6, 1> Vector6d;
typedef Matrix<double, 4, 4, DontAlign> Matrix4d_u;
}  // namespace Eigen
namespace open3d {
namespace utility {
Eigen::Vector6d TransformMatrix4dToVector6d(const Eigen::Matrix4d& input);
Eigen::Matrix4d TransformVector6dToMatrix4d(const Eigen::Vector6d& input);
std::tuple<bool, Eigen::VectorXd> SolveLinearSystemPSD(const Eigen::MatrixXd& A, const Eigen::VectorXd& b,
                                                       bool prefer_sparse = false, bool check_symmetric = false,
                                                       bool check_det = false, bool check_psd = false);
}  // namespace utility
}  // namespace open3d
