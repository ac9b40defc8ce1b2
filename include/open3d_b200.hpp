// open3d_b200.hpp — header-only C++17 mirror of the reference's host interface for the hot
// path, over the C ABI of open3d_b200.h.  Same names, argument meaning and error behaviour
// (std::runtime_error, as utility::LogError throws) as
//   open3d::t::pipelines::registration::{ICP, EvaluateRegistration, ICPConvergenceCriteria,
//       RegistrationResult, RobustKernel, TransformationEstimationPointToPlane}
//       (cpp/open3d/t/pipelines/registration/{Registration.h, TransformationEstimation.h, RobustKernel.h})
//   open3d::t::pipelines::slam::{Model, Frame}            (cpp/open3d/t/pipelines/slam/{Model.h, Frame.h})
//   open3d::t::pipelines::odometry::{RGBDOdometryMultiScale (PointToPlane), OdometryResult, ...}   (odometry/RGBDOdometry.h)
//   open3d::t::geometry::{PointCloud, VoxelBlockGrid}     (the members this path touches)
// core::Tensor is replaced by raw device pointers + sizes (the library has no tensor runtime;
// INTEGRATION.md shows the forwarding stubs for a real Open3D build).
#pragma once

#include <algorithm>
#include <array>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <functional>
#include <limits>
#include <stdexcept>
#include <string>
#include <vector>

#include "open3d_b200.h"

namespace open3d_b200 {

inline void Check(int rc) {
    if (rc < 0) throw std::runtime_error(o3db_last_error());
}

namespace t {
namespace geometry {

/// t::geometry::PointCloud restricted to what the path reads: contiguous Float32 [N,3]
/// device arrays (kernel/Registration.cpp:56-59 calls .Contiguous()).
struct PointCloud {
    const float* positions = nullptr;  // device
    const float* normals = nullptr;    // device, may be null
    int64_t num_points = 0;
    const float* colors = nullptr;     // device, may be null
    const float* dopplers = nullptr;   // device [N], may be null (the "dopplers" attribute DopplerICP reads)
    const float* directions = nullptr; // device [N,3], may be null (the "directions" attribute)
    const float* color_gradients = nullptr;   // device, may be null ("color_gradients" attribute)
    bool HasPointPositions() const { return positions != nullptr && num_points > 0; }
    bool HasPointNormals() const { return normals != nullptr && num_points > 0; }
    bool HasPointColors() const { return colors != nullptr && num_points > 0; }

    /// PointCloud::EstimateColorGradients (t/geometry/PointCloud.cpp:723-767, hybrid search) into a
    /// caller-owned [N,3] device buffer, which becomes this cloud's color_gradients attribute.
    /// exact_solver = false (default): upstream's solve_svd3x3<float>, bit for bit; true: exact pseudo-inverse (extension).
    void EstimateColorGradients(float* gradients_dev, int max_nn = 30, double radius = 0.0, void* stream = nullptr,
                                bool exact_solver = false) {
        if (!HasPointColors()) throw std::runtime_error("PointCloud must have colors attribute to estimate color gradients.");
        if (!HasPointNormals()) throw std::runtime_error("PointCloud must have normals attribute to estimate color gradients.");
        Check(o3db_estimate_color_gradients_solver(positions, normals, colors, num_points, radius, max_nn,
                                                   exact_solver ? O3DB_GRADIENT_SOLVER_EXACT : O3DB_GRADIENT_SOLVER_REFERENCE,
                                                   gradients_dev, stream));
        color_gradients = gradients_dev;
    }
};

}  // namespace geometry

namespace pipelines {
namespace registration {

/// RobustKernel.h:15-23
enum class RobustKernelMethod { L2Loss = 0, L1Loss = 1, HuberLoss = 2, CauchyLoss = 3, GMLoss = 4, TukeyLoss = 5, GeneralizedLoss = 6 };

/// RobustKernel.h:33-58
class RobustKernel {
public:
    explicit RobustKernel(RobustKernelMethod type = RobustKernelMethod::L2Loss, double scaling_parameter = 1.0,
                          double shape_parameter = 1.0)
        : type_(type), scaling_parameter_(scaling_parameter), shape_parameter_(shape_parameter) {}
    RobustKernelMethod type_;
    double scaling_parameter_;
    double shape_parameter_;
};

/// Registration.h:43-48
class ICPConvergenceCriteria {
public:
    ICPConvergenceCriteria(double relative_fitness = 1e-6, double relative_rmse = 1e-6, int max_iteration = 30)
        : relative_fitness_(relative_fitness), relative_rmse_(relative_rmse), max_iteration_(max_iteration) {}
    double relative_fitness_;
    double relative_rmse_;
    int max_iteration_;
};

/// Registration.h:65-98.  transformation_: row-major 4x4 Float64 on the host;
/// correspondences_: optional device buffer [N] int64 supplied by the caller (-1 = none).
class RegistrationResult {
public:
    std::array<double, 16> transformation_{{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}};
    int64_t* correspondences_ = nullptr;
    double inlier_rmse_ = 0.0;
    double fitness_ = 0.0;
    bool converged_ = false;
    int num_iterations_ = 0;
    std::vector<std::array<double, 2>> per_iteration_;  // (fitness, inlier_rmse) seen by the callback
};

/// TransformationEstimation.h:101-149: the estimator upstream's ICP uses by default.  Positions only, no robust kernel.
class TransformationEstimationPointToPoint {
public:
    /// kernel::ComputeRtPointToPoint + RtToTransformation (TransformationEstimation.cpp:132-159): the row-major 4x4
    /// Float64 transformation on the host.  Throws "No valid correspondence present." when every entry is -1.
    std::array<double, 16> ComputeTransformation(const geometry::PointCloud& source, const geometry::PointCloud& target,
                                                 const int64_t* correspondences_dev, void* stream = nullptr) const {
        if (!target.HasPointPositions() || !source.HasPointPositions())
            throw std::runtime_error("Source and/or Target pointcloud is empty.");
        double R[9], t[3];
        Check(o3db_compute_rt_point_to_point(source.positions, target.positions, correspondences_dev, source.num_points, R,
                                             t, nullptr, stream));
        return {{R[0], R[1], R[2], t[0], R[3], R[4], R[5], t[1], R[6], R[7], R[8], t[2], 0, 0, 0, 1}};
    }
};

/// TransformationEstimation.h:155-212
class TransformationEstimationPointToPlane {
public:
    TransformationEstimationPointToPlane() = default;
    explicit TransformationEstimationPointToPlane(const RobustKernel& kernel) : kernel_(kernel) {}

    /// kernel::ComputePosePointToPlane + PoseToTransformation (TransformationEstimation.cpp:196-227):
    /// returns the row-major 4x4 Float64 update.  pose_dev: [6] f64 device scratch, the reference's
    /// `pose` tensor (kernel/Registration.cpp:43); copy_to_host: a device->host memcpy (e.g. cudaMemcpy).
    std::array<double, 16> ComputeTransformation(const geometry::PointCloud& source, const geometry::PointCloud& target,
                                                 const int64_t* correspondences_dev, double* pose_dev,
                                                 const std::function<void(void* dst, const void* src, size_t)>& copy_to_host,
                                                 void* stream = nullptr) const {
        if (!target.HasPointPositions() || !source.HasPointPositions())
            throw std::runtime_error("Source and/or Target pointcloud is empty.");
        if (!target.HasPointNormals()) throw std::runtime_error("Target pointcloud missing normals attribute.");
        o3db_robust_kernel k{static_cast<int>(kernel_.type_), kernel_.scaling_parameter_, kernel_.shape_parameter_};
        float residual = 0;
        int inliers = 0;
        Check(o3db_compute_pose_point_to_plane(source.positions, target.positions, target.normals, correspondences_dev,
                                               source.num_points, &k, nullptr, pose_dev, &residual, &inliers, stream));
        double pose[6];
        copy_to_host(pose, pose_dev, sizeof(pose));
        std::array<double, 16> T;
        o3db_pose_to_transformation(pose, T.data());
        return T;
    }

    RobustKernel kernel_;
};

/// TransformationEstimation.h:214-270: Rusinkiewicz's symmetric objective; both clouds need normals.
class TransformationEstimationSymmetric {
public:
    TransformationEstimationSymmetric() = default;
    explicit TransformationEstimationSymmetric(const RobustKernel& kernel) : kernel_(kernel) {}

    /// kernel::ComputeTransformationSymmetric (TransformationEstimation.cpp:276-292): the row-major 4x4 Float64
    /// transformation on the host, the identity without a valid correspondence.  Throws on a correspondence outside
    /// [-1, target.num_points).
    std::array<double, 16> ComputeTransformation(const geometry::PointCloud& source, const geometry::PointCloud& target,
                                                 const int64_t* correspondences_dev, void* stream = nullptr) const {
        if (!target.HasPointPositions() || !source.HasPointPositions())
            throw std::runtime_error("Source and/or Target pointcloud is empty.");
        if (!source.HasPointNormals() || !target.HasPointNormals())
            throw std::runtime_error("SymmetricICP requires both source and target to have normals.");
        o3db_robust_kernel k{static_cast<int>(kernel_.type_), kernel_.scaling_parameter_, kernel_.shape_parameter_};
        std::array<double, 16> T;
        Check(o3db_compute_transformation_symmetric(source.positions, target.positions, source.normals, target.normals,
                                                    correspondences_dev, source.num_points, target.num_points, &k, T.data(),
                                                    nullptr, stream));
        return T;
    }

    RobustKernel kernel_;
};

/// TransformationEstimation.h:356-425: DICP's point-to-plane + Doppler objective, with the C++ constructor's arguments.
/// |period| < 1e-3 throws "Time period too small."; a lambda_doppler outside [0, 1] becomes 0.01.
class TransformationEstimationForDopplerICP {
public:
    explicit TransformationEstimationForDopplerICP(double period = 0.1, double lambda_doppler = 0.01,
                                                   bool reject_dynamic_outliers = false,
                                                   double doppler_outlier_threshold = 2.0,
                                                   std::size_t outlier_rejection_min_iteration = 2,
                                                   std::size_t geometric_robust_loss_min_iteration = 0,
                                                   std::size_t doppler_robust_loss_min_iteration = 2,
                                                   const RobustKernel& geometric_kernel = RobustKernel(),
                                                   const RobustKernel& doppler_kernel = RobustKernel(),
                                                   const std::array<double, 16>& transform_vehicle_to_sensor =
                                                           {{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}})
        : period_(period),
          lambda_doppler_((lambda_doppler < 0 || lambda_doppler > 1.0) ? 0.01 : lambda_doppler),
          reject_dynamic_outliers_(reject_dynamic_outliers),
          doppler_outlier_threshold_(doppler_outlier_threshold),
          outlier_rejection_min_iteration_(outlier_rejection_min_iteration),
          geometric_robust_loss_min_iteration_(geometric_robust_loss_min_iteration),
          doppler_robust_loss_min_iteration_(doppler_robust_loss_min_iteration),
          geometric_kernel_(geometric_kernel),
          doppler_kernel_(doppler_kernel),
          transform_vehicle_to_sensor_(transform_vehicle_to_sensor) {
        if (std::abs(period) < 1e-3) throw std::runtime_error("Time period too small.");
    }

    o3db_doppler_params Params() const {
        o3db_doppler_params p{};
        p.period = period_;
        p.lambda_doppler = lambda_doppler_;
        p.reject_dynamic_outliers = reject_dynamic_outliers_ ? 1 : 0;
        p.doppler_outlier_threshold = doppler_outlier_threshold_;
        p.outlier_rejection_min_iteration = static_cast<int64_t>(outlier_rejection_min_iteration_);
        p.geometric_robust_loss_min_iteration = static_cast<int64_t>(geometric_robust_loss_min_iteration_);
        p.doppler_robust_loss_min_iteration = static_cast<int64_t>(doppler_robust_loss_min_iteration_);
        p.geometric_kernel = {static_cast<int>(geometric_kernel_.type_), geometric_kernel_.scaling_parameter_,
                              geometric_kernel_.shape_parameter_};
        p.doppler_kernel = {static_cast<int>(doppler_kernel_.type_), doppler_kernel_.scaling_parameter_,
                            doppler_kernel_.shape_parameter_};
        for (int i = 0; i < 16; ++i) p.transform_vehicle_to_sensor[i] = transform_vehicle_to_sensor_[i];
        return p;
    }

    static void CheckInputs(const geometry::PointCloud& source, const geometry::PointCloud& target) {
        if (!target.HasPointPositions() || !source.HasPointPositions())
            throw std::runtime_error("Source and/or Target pointcloud is empty.");
        if (!target.HasPointNormals()) throw std::runtime_error("Target pointcloud missing normals attribute.");
        if (source.dopplers == nullptr) throw std::runtime_error("Source pointcloud missing dopplers attribute.");
        if (source.directions == nullptr) throw std::runtime_error("Source pointcloud missing directions attribute.");
    }

    /// kernel::ComputePoseDopplerICP + PoseToTransformation (TransformationEstimation.cpp:469-519) for iteration
    /// `iteration` of the accumulated transformation current_transform: the row-major 4x4 Float64 update.  pose_dev
    /// and copy_to_host as TransformationEstimationPointToPlane::ComputeTransformation's.
    std::array<double, 16> ComputeTransformation(const geometry::PointCloud& source, const geometry::PointCloud& target,
                                                 const int64_t* correspondences_dev,
                                                 const std::array<double, 16>& current_transform, std::size_t iteration,
                                                 double* pose_dev,
                                                 const std::function<void(void* dst, const void* src, size_t)>& copy_to_host,
                                                 void* stream = nullptr) const {
        CheckInputs(source, target);
        const o3db_doppler_params p = Params();
        Check(o3db_compute_pose_doppler_icp(source.positions, source.dopplers, source.directions, target.positions,
                                            target.normals, correspondences_dev, source.num_points, current_transform.data(),
                                            static_cast<int64_t>(iteration), &p, nullptr, pose_dev, nullptr, nullptr,
                                            stream));
        double pose[6];
        copy_to_host(pose, pose_dev, sizeof(pose));
        std::array<double, 16> T;
        o3db_pose_to_transformation(pose, T.data());
        return T;
    }

    double period_;
    double lambda_doppler_;
    bool reject_dynamic_outliers_;
    double doppler_outlier_threshold_;
    std::size_t outlier_rejection_min_iteration_;
    std::size_t geometric_robust_loss_min_iteration_;
    std::size_t doppler_robust_loss_min_iteration_;
    RobustKernel geometric_kernel_;
    RobustKernel doppler_kernel_;
    std::array<double, 16> transform_vehicle_to_sensor_;
};

/// TransformationEstimation.h:318-395 (lambda_geometric outside [0,1] falls back to 0.968, :337-340)
class TransformationEstimationForColoredICP {
public:
    explicit TransformationEstimationForColoredICP(double lambda_geometric = 0.968, const RobustKernel& kernel = RobustKernel())
        : lambda_geometric_((lambda_geometric < 0 || lambda_geometric > 1.0) ? 0.968 : lambda_geometric), kernel_(kernel) {}
    double lambda_geometric_;
    RobustKernel kernel_;
};

using IterationCallback = std::function<void(int iteration_index, double fitness, double inlier_rmse)>;

/// The C result of a finished loop as the reference's result type, with the callback replayed (Registration.cpp:330-345).
inline RegistrationResult ToRegistrationResult(const o3db_icp_result& r, const std::vector<double>& per,
                                               int64_t* correspondences_dev, const IterationCallback& callback_after_iteration) {
    RegistrationResult out;
    for (int i = 0; i < 16; ++i) out.transformation_[i] = r.transformation[i];
    out.correspondences_ = correspondences_dev;
    out.fitness_ = r.fitness;
    out.inlier_rmse_ = r.inlier_rmse;
    out.converged_ = r.converged != 0;
    out.num_iterations_ = r.num_iterations;
    const int executed = r.num_iterations + (r.converged ? 1 : 0);
    for (int k = 0; k < executed; ++k) {
        out.per_iteration_.push_back({per[2 * k], per[2 * k + 1]});
        if (callback_after_iteration) callback_after_iteration(k, per[2 * k], per[2 * k + 1]);
    }
    return out;
}

namespace detail {
/// What every registration::ICP overload does after its estimator's own checks: the distance and voxel checks (the
/// overload's own voxel message), the options (kernel null: opt.kernel stays zeroed), the per-iteration buffer, the C
/// call run(options, result, per_iteration) and the result.
template <class Run>
inline RegistrationResult RunICP(double max_correspondence_distance, double voxel_size, const char* voxel_message,
                                 const ICPConvergenceCriteria& criteria, const RobustKernel* kernel,
                                 const IterationCallback& callback_after_iteration, int64_t* correspondences_dev,
                                 const Run& run) {
    if (max_correspondence_distance <= 0.0)
        throw std::runtime_error(" Max correspondence distance must be greater than 0, but got " +
                                 std::to_string(max_correspondence_distance) + " in scale: 0.");
    if (voxel_size > 0) throw std::runtime_error(voxel_message);
    o3db_icp_options opt{};
    opt.max_correspondence_distance = max_correspondence_distance;
    opt.max_iteration = criteria.max_iteration_;
    opt.relative_fitness = criteria.relative_fitness_;
    opt.relative_rmse = criteria.relative_rmse_;
    if (kernel) opt.kernel = {static_cast<int>(kernel->type_), kernel->scaling_parameter_, kernel->shape_parameter_};
    o3db_icp_result r{};
    std::vector<double> per(2 * static_cast<size_t>(criteria.max_iteration_ > 0 ? criteria.max_iteration_ : 1), 0.0);
    Check(run(&opt, &r, per.data()));
    return ToRegistrationResult(r, per, correspondences_dev, callback_after_iteration);
}
}  // namespace detail

/// registration::ICP (Registration.h:133-144, Registration.cpp:93-106) for
/// TransformationEstimationPointToPlane; voxel_size must be <= 0 here (down-sample with
/// o3db_voxel_down_sample beforehand; the Python surface builds the pyramid itself).
inline RegistrationResult ICP(const geometry::PointCloud& source, const geometry::PointCloud& target,
                              double max_correspondence_distance,
                              const std::array<double, 16>& init_source_to_target = {{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}},
                              const TransformationEstimationPointToPlane& estimation = TransformationEstimationPointToPlane(),
                              const ICPConvergenceCriteria& criteria = ICPConvergenceCriteria(),
                              double voxel_size = -1.0, const IterationCallback& callback_after_iteration = nullptr,
                              int64_t* correspondences_dev = nullptr, void* stream = nullptr) {
    // Registration.cpp:119-219 AssertInputMultiScaleICP
    if (!target.HasPointPositions() || !source.HasPointPositions())
        throw std::runtime_error("Source and/or Target pointcloud is empty.");
    if (!target.HasPointNormals())
        throw std::runtime_error("TransformationEstimationPointToPlane require pre-computed normal vectors for target PointCloud.");
    return detail::RunICP(
            max_correspondence_distance, voxel_size,
            "voxel_size > 0: apply PointCloud::VoxelDownSample first (o3db_voxel_down_sample); this header-only wrapper owns no device memory for the pyramid",
            criteria, &estimation.kernel_, callback_after_iteration, correspondences_dev,
            [&](const o3db_icp_options* opt, o3db_icp_result* r, double* per) {
                return o3db_icp_point_to_plane(source.positions, source.num_points, target.positions, target.normals,
                                               target.num_points, init_source_to_target.data(), opt, r, correspondences_dev,
                                               per, stream);
            });
}

/// registration::ICP for TransformationEstimationForColoredICP.  The target needs color_gradients
/// (PointCloud::EstimateColorGradients; upstream computes them with radius 2 * max_correspondence_distance
/// when missing, Registration.cpp:243-263 — here the caller owns the buffer, so it is required).
inline RegistrationResult ICP(const geometry::PointCloud& source, const geometry::PointCloud& target,
                              double max_correspondence_distance, const std::array<double, 16>& init_source_to_target,
                              const TransformationEstimationForColoredICP& estimation,
                              const ICPConvergenceCriteria& criteria = ICPConvergenceCriteria(), double voxel_size = -1.0,
                              const IterationCallback& callback_after_iteration = nullptr,
                              int64_t* correspondences_dev = nullptr, void* stream = nullptr) {
    if (!target.HasPointPositions() || !source.HasPointPositions())
        throw std::runtime_error("Source and/or Target pointcloud is empty.");
    if (!target.HasPointNormals()) throw std::runtime_error("ColoredICP requires target pointcloud to have normals.");
    if (!target.HasPointColors()) throw std::runtime_error("ColoredICP requires target pointcloud to have colors.");
    if (!source.HasPointColors()) throw std::runtime_error("ColoredICP requires source pointcloud to have colors.");
    if (!target.color_gradients) throw std::runtime_error("Target pointcloud missing color_gradients attribute.");
    return detail::RunICP(
            max_correspondence_distance, voxel_size,
            "voxel_size > 0: apply PointCloud::VoxelDownSample first (o3db_voxel_down_sample_attrs)", criteria,
            &estimation.kernel_, callback_after_iteration, correspondences_dev,
            [&](const o3db_icp_options* opt, o3db_icp_result* r, double* per) {
                return o3db_icp_colored(source.positions, source.colors, source.num_points, target.positions,
                                        target.normals, target.colors, target.color_gradients, target.num_points,
                                        init_source_to_target.data(), opt, estimation.lambda_geometric_, r,
                                        correspondences_dev, per, stream);
            });
}

/// registration::ICP for TransformationEstimationPointToPoint (upstream's default estimator, Registration.h:140):
/// neither cloud needs anything but positions.
inline RegistrationResult ICP(const geometry::PointCloud& source, const geometry::PointCloud& target,
                              double max_correspondence_distance, const std::array<double, 16>& init_source_to_target,
                              const TransformationEstimationPointToPoint&,
                              const ICPConvergenceCriteria& criteria = ICPConvergenceCriteria(), double voxel_size = -1.0,
                              const IterationCallback& callback_after_iteration = nullptr,
                              int64_t* correspondences_dev = nullptr, void* stream = nullptr) {
    if (!target.HasPointPositions() || !source.HasPointPositions())
        throw std::runtime_error("Source and/or Target pointcloud is empty.");
    return detail::RunICP(max_correspondence_distance, voxel_size,
                          "voxel_size > 0: apply PointCloud::VoxelDownSample first (o3db_voxel_down_sample)", criteria,
                          nullptr, callback_after_iteration, correspondences_dev,
                          [&](const o3db_icp_options* opt, o3db_icp_result* r, double* per) {
                              return o3db_icp_point_to_point(source.positions, source.num_points, target.positions,
                                                             target.num_points, init_source_to_target.data(), opt, r,
                                                             correspondences_dev, per, stream);
                          });
}

/// registration::ICP for TransformationEstimationSymmetric (and registration_symmetric_icp, Registration.cpp:108-117):
/// both clouds need normals; the working source's normals turn with its points.
inline RegistrationResult ICP(const geometry::PointCloud& source, const geometry::PointCloud& target,
                              double max_correspondence_distance, const std::array<double, 16>& init_source_to_target,
                              const TransformationEstimationSymmetric& estimation,
                              const ICPConvergenceCriteria& criteria = ICPConvergenceCriteria(), double voxel_size = -1.0,
                              const IterationCallback& callback_after_iteration = nullptr,
                              int64_t* correspondences_dev = nullptr, void* stream = nullptr) {
    if (!target.HasPointPositions() || !source.HasPointPositions())
        throw std::runtime_error("Source and/or Target pointcloud is empty.");
    if (!source.HasPointNormals() || !target.HasPointNormals())
        throw std::runtime_error("SymmetricICP requires both source and target pointclouds to have normals.");
    return detail::RunICP(max_correspondence_distance, voxel_size,
                          "voxel_size > 0: apply PointCloud::VoxelDownSample first (o3db_voxel_down_sample)", criteria,
                          &estimation.kernel_, callback_after_iteration, correspondences_dev,
                          [&](const o3db_icp_options* opt, o3db_icp_result* r, double* per) {
                              return o3db_icp_symmetric(source.positions, source.normals, source.num_points,
                                                        target.positions, target.normals, target.num_points,
                                                        init_source_to_target.data(), opt, r, correspondences_dev, per,
                                                        stream);
                          });
}

/// registration::ICP for TransformationEstimationForDopplerICP: the source needs dopplers and directions (never
/// transformed), the target normals.  Single scale, as the other overloads.
inline RegistrationResult ICP(const geometry::PointCloud& source, const geometry::PointCloud& target,
                              double max_correspondence_distance, const std::array<double, 16>& init_source_to_target,
                              const TransformationEstimationForDopplerICP& estimation,
                              const ICPConvergenceCriteria& criteria = ICPConvergenceCriteria(), double voxel_size = -1.0,
                              const IterationCallback& callback_after_iteration = nullptr,
                              int64_t* correspondences_dev = nullptr, void* stream = nullptr) {
    if (!target.HasPointPositions() || !source.HasPointPositions())
        throw std::runtime_error("Source and/or Target pointcloud is empty.");
    if (!target.HasPointNormals()) throw std::runtime_error("DopplerICP requires target pointcloud to have normals.");
    if (source.dopplers == nullptr)
        throw std::runtime_error("DopplerICP requires source pointcloud to have Doppler velocities.");
    if (source.directions == nullptr)
        throw std::runtime_error("DopplerICP requires source pointcloud to have pre-computed direction vectors.");
    const o3db_doppler_params p = estimation.Params();
    return detail::RunICP(max_correspondence_distance, voxel_size,
                          "voxel_size > 0: apply PointCloud::VoxelDownSample first (o3db_voxel_down_sample)", criteria,
                          nullptr, callback_after_iteration, correspondences_dev,
                          [&](const o3db_icp_options* opt, o3db_icp_result* r, double* per) {
                              return o3db_icp_doppler(source.positions, source.dopplers, source.directions,
                                                      source.num_points, target.positions, target.normals,
                                                      target.num_points, init_source_to_target.data(), opt, &p, r,
                                                      correspondences_dev, per, stream);
                          });
}

/// registration::GetInformationMatrix (Registration.cpp:446-485): row-major 6x6 Float64 GTG on the host.
inline std::array<double, 36> GetInformationMatrix(const geometry::PointCloud& source, const geometry::PointCloud& target,
                                                   double max_correspondence_distance,
                                                   const std::array<double, 16>& transformation, void* stream = nullptr) {
    if (!target.HasPointPositions() || !source.HasPointPositions())
        throw std::runtime_error("Source and/or Target pointcloud is empty.");
    std::array<double, 36> info{};
    Check(o3db_get_information_matrix(source.positions, source.num_points, target.positions, target.num_points,
                                      max_correspondence_distance, transformation.data(), info.data(), stream));
    return info;
}

}  // namespace registration

namespace odometry {

/// RGBDOdometry.h:24-30
enum class Method { PointToPlane, Intensity, Hybrid };

/// RGBDOdometry.h:33-52 (implicitly constructible from an iteration count, like upstream's {10, 5, 3})
class OdometryConvergenceCriteria {
public:
    OdometryConvergenceCriteria(int max_iteration, double relative_rmse = 1e-6, double relative_fitness = 1e-6)
        : max_iteration_(max_iteration), relative_rmse_(relative_rmse), relative_fitness_(relative_fitness) {}
    int max_iteration_;
    double relative_rmse_;
    double relative_fitness_;
};

/// RGBDOdometry.h:54-78
class OdometryResult {
public:
    std::array<double, 16> transformation_{{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}};
    double inlier_rmse_ = 0.0;
    double fitness_ = 0.0;
};

/// RGBDOdometry.h:80-114
class OdometryLossParams {
public:
    OdometryLossParams(float depth_outlier_trunc = 0.07f, float depth_huber_delta = 0.05f, float intensity_huber_delta = 0.1f)
        : depth_outlier_trunc_(depth_outlier_trunc), depth_huber_delta_(depth_huber_delta),
          intensity_huber_delta_(intensity_huber_delta) {}
    float depth_outlier_trunc_, depth_huber_delta_, intensity_huber_delta_;
};

/// A depth image on the device: UInt16 or Float32, [rows][cols].
struct DepthImage {
    const void* data = nullptr;
    bool is_f32 = false;
    int rows = 0, cols = 0;
};

/// RGBDOdometryMultiScale (RGBDOdometry.cpp:56-113) for Method::PointToPlane (only the depth images are read).
inline OdometryResult RGBDOdometryMultiScale(const DepthImage& source, const DepthImage& target,
                                             const std::array<double, 9>& intrinsics,
                                             const std::array<double, 16>& init_source_to_target = {{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}},
                                             float depth_scale = 1000.0f, float depth_max = 3.0f,
                                             const std::vector<OdometryConvergenceCriteria>& criteria_list = {10, 5, 3},
                                             Method method = Method::Hybrid, const OdometryLossParams& params = OdometryLossParams(),
                                             void* stream = nullptr) {
    if (method != Method::PointToPlane)
        throw std::runtime_error("open3d_b200 implements Method::PointToPlane; Intensity / Hybrid odometry are outside this build's scope.");
    if (!source.data || !target.data || source.rows <= 0 || source.cols <= 0)
        throw std::runtime_error("Invalid shape, expected a 1 channel image, but got an empty depth image");
    if (source.rows != target.rows || source.cols != target.cols)
        throw std::runtime_error("source and target depth images must have the same size");
    std::vector<o3db_odometry_criteria> c;
    for (const auto& k : criteria_list) c.push_back({k.max_iteration_, k.relative_rmse_, k.relative_fitness_});
    o3db_odometry_result r{};
    Check(o3db_rgbd_odometry_multi_scale_point_to_plane(
            source.data, source.is_f32 ? O3DB_DEPTH_F32 : O3DB_DEPTH_U16, target.data, target.is_f32 ? O3DB_DEPTH_F32 : O3DB_DEPTH_U16,
            source.rows, source.cols, intrinsics.data(), init_source_to_target.data(), depth_scale, depth_max, c.data(),
            static_cast<int>(c.size()), params.depth_outlier_trunc_, params.depth_huber_delta_, &r, nullptr, stream));
    OdometryResult out;
    for (int i = 0; i < 16; ++i) out.transformation_[i] = r.transformation[i];
    out.inlier_rmse_ = r.inlier_rmse;
    out.fitness_ = r.fitness;
    return out;
}

}  // namespace odometry

namespace slam {

/// slam::Frame (slam/Frame.h): intrinsics + device (or host) images.
struct Frame {
    int height = 0, width = 0;
    std::array<double, 9> intrinsics{{525.0, 0, 319.5, 0, 525.0, 239.5, 0, 0, 1}};
    const void* depth = nullptr;   // u16 (depth_is_f32 = false) or f32
    const void* color = nullptr;   // u8x3 or f32x3, may be null
    bool depth_is_f32 = false;
    bool images_on_host = false;
};

/// slam::Model (slam/Model.h, Model.cpp:23-36, 91-106): owns the voxel block grid
/// {tsdf f32, weight u16, color u16x3} and the current frame pose.
class Model {
public:
    Model(float voxel_size, int block_resolution = 16, int block_count = 10000,
          const std::array<double, 16>& T_init = {{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}}, void* stream = nullptr)
        : T_frame_to_world_(T_init) {
        Check(o3db_vbg_create(voxel_size, block_resolution, block_count, 1, stream, &vbg_));
    }
    ~Model() { o3db_vbg_destroy(vbg_); }
    Model(const Model&) = delete;
    Model& operator=(const Model&) = delete;

    const std::array<double, 16>& GetCurrentFramePose() const { return T_frame_to_world_; }
    void UpdateFramePose(int frame_id, const std::array<double, 16>& T_frame_to_world) {
        frame_id_ = frame_id;
        T_frame_to_world_ = T_frame_to_world;
    }

    /// Model::Integrate (Model.cpp:91-106)
    void Integrate(const Frame& f, float depth_scale = 1000.0f, float depth_max = 3.0f, float trunc_voxel_multiplier = 8.0f,
                   void* stream = nullptr) {
        const std::array<double, 16> E = Extrinsic();
        const int dd = f.depth_is_f32 ? O3DB_DEPTH_F32 : O3DB_DEPTH_U16;
        const int cd = f.color ? (f.depth_is_f32 ? O3DB_COLOR_F32 : O3DB_COLOR_U8) : O3DB_COLOR_NONE;
        Check((f.images_on_host ? o3db_vbg_integrate_frame_host : o3db_vbg_integrate_frame)(
                vbg_, f.depth, dd, f.color, cd, f.height, f.width, f.intrinsics.data(), E.data(), depth_scale, depth_max,
                trunc_voxel_multiplier, stream));
    }

    /// Model::TrackFrameToModel (Model.cpp:68-89): the input frame's depth against the ray-cast model depth
    /// (Float32 device buffer filled by SynthesizeModelFrame), identity initialisation.
    odometry::OdometryResult TrackFrameToModel(const Frame& input_frame, const float* raycast_depth_dev, float depth_scale = 1000.0f,
                                               float depth_max = 3.0f, float depth_diff = 0.07f,
                                               odometry::Method method = odometry::Method::PointToPlane,
                                               const std::vector<odometry::OdometryConvergenceCriteria>& criteria = {6, 3, 1},
                                               void* stream = nullptr) const {
        if (input_frame.images_on_host) throw std::runtime_error("TrackFrameToModel: the input frame must be on the device");
        odometry::DepthImage src{input_frame.depth, input_frame.depth_is_f32, input_frame.height, input_frame.width};
        odometry::DepthImage tgt{raycast_depth_dev, true, input_frame.height, input_frame.width};
        return odometry::RGBDOdometryMultiScale(src, tgt, input_frame.intrinsics, {{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}},
                                                depth_scale, depth_max, criteria, method, odometry::OdometryLossParams(depth_diff), stream);
    }

    /// Model::SynthesizeModelFrame (Model.cpp:38-66): ray-cast the blocks of the last integrated frame from
    /// the current pose.  depth_dev [h][w] f32 and color_dev [h][w][3] f32 are caller-owned device buffers
    /// (color_dev may be null = enable_color false).
    void SynthesizeModelFrame(int height, int width, const std::array<double, 9>& intrinsics, float* depth_dev,
                              float* color_dev, float depth_scale = 1000.0f, float depth_min = 0.1f, float depth_max = 3.0f,
                              float trunc_voxel_multiplier = 8.0f, float weight_threshold = -1.0f, void* stream = nullptr) {
        if (weight_threshold < 0) weight_threshold = std::min(frame_id_ * 1.0f, 3.0f);
        const std::array<double, 16> E = Extrinsic();
        o3db_raycast_outputs out{};
        out.depth = depth_dev;
        out.color = color_dev;
        Check(o3db_vbg_ray_cast(vbg_, nullptr, 0, intrinsics.data(), E.data(), width, height, &out, depth_scale, depth_min,
                                depth_max, weight_threshold, trunc_voxel_multiplier, 8, nullptr, stream));
    }

    int64_t NumBlocks(void* stream = nullptr) {
        const int64_t n = o3db_vbg_size(vbg_, stream);
        Check(n < 0 ? static_cast<int>(n) : 0);
        return n;
    }
    o3db_vbg* GetVoxelGrid() { return vbg_; }

    int frame_id_ = -1;

private:
    /// t::geometry::InverseTransformation (t/geometry/Utility.h:77-115) of the current pose
    std::array<double, 16> Extrinsic() const {
        const auto& T = T_frame_to_world_;
        std::array<double, 16> E{};
        E[0] = T[0]; E[1] = T[4]; E[2] = T[8];
        E[4] = T[1]; E[5] = T[5]; E[6] = T[9];
        E[8] = T[2]; E[9] = T[6]; E[10] = T[10];
        E[3] = -(E[0] * T[3] + E[1] * T[7] + E[2] * T[11]);
        E[7] = -(E[4] * T[3] + E[5] * T[7] + E[6] * T[11]);
        E[11] = -(E[8] * T[3] + E[9] * T[7] + E[10] * T[11]);
        E[15] = 1;
        return E;
    }

    o3db_vbg* vbg_ = nullptr;
    std::array<double, 16> T_frame_to_world_;
};

}  // namespace slam
}  // namespace pipelines
}  // namespace t
}  // namespace open3d_b200
