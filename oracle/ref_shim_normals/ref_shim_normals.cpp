// ref_shim_normals.cpp — TEST INFRASTRUCTURE.  Compiles the reference's own normal-estimation code, unmodified, from
// where it lies in the reference tree (t/geometry/kernel/PointCloudImpl.h, included as a header), against the stub
// core::Tensor / ParallelFor headers of ../ref_shim/stubs, and exports it through C functions so that the CPU oracle
// (oracle/normals/normals_oracle.c) can be checked against the real thing:
//   EstimatePointWiseRobustNormalizedCovarianceKernel<float> (:512-586), one point;
//   EstimatePointWiseNormalsWithFastEigen3x3<float> (:875-1009), one covariance;
//   EstimateNormalsFromCovariancesCPU (:1011-1065), the whole function with both orientation rules;
//   OrientNormalsToAlignWithDirectionCPU (:261-294) and OrientNormalsTowardsCameraLocationCPU (:296-351), whole.
// No reference source is copied into this repository.
#include <cmath>
#include <cstdint>
#include <cstring>

using std::abs;
using std::max;
using std::min;

#include "open3d/t/geometry/kernel/PointCloudImpl.h"   // from -I <reference>/cpp

namespace o3c = open3d::core;
namespace o3p = open3d::t::geometry::kernel::pointcloud;

extern "C" {

// indices[0..count) are the point's hybrid-search neighbours
void ref_covariance_point_f32(const float* points, const int32_t* indices, int32_t count, float covariance[9]) {
    o3p::EstimatePointWiseRobustNormalizedCovarianceKernel<float>(points, indices, count, covariance);
}

void ref_normal_from_covariance_f32(const float covariance[9], float normal[3]) {
    normal[0] = normal[1] = normal[2] = 0.0f;   // as EstimateNormalsFromCovariances initialises normals_output
    o3p::EstimatePointWiseNormalsWithFastEigen3x3<float>(covariance, normal);
}

// normals [n,3]: the prior normals on entry when has_normals, the result on return
void ref_normals_from_covariances_f32(const float* covariances, int64_t n, int has_normals, float* normals) {
    const o3c::Tensor c((void*)covariances, {n, 3, 3}, o3c::Float32);
    o3c::Tensor nn((void*)normals, {n, 3}, o3c::Float32);
    o3p::EstimateNormalsFromCovariancesCPU(c, nn, has_normals != 0);
}

void ref_orient_normals_to_align_with_direction_f32(float* normals, int64_t n, const float direction[3]) {
    o3c::Tensor nn((void*)normals, {n, 3}, o3c::Float32);
    const o3c::Tensor d((void*)direction, {3}, o3c::Float32);
    o3p::OrientNormalsToAlignWithDirectionCPU(nn, d);
}

void ref_orient_normals_towards_camera_location_f32(const float* points, float* normals, int64_t n,
                                                    const float camera[3]) {
    const o3c::Tensor p((void*)points, {n, 3}, o3c::Float32), c((void*)camera, {3}, o3c::Float32);
    o3c::Tensor nn((void*)normals, {n, 3}, o3c::Float32);
    o3p::OrientNormalsTowardsCameraLocationCPU(p, nn, c);
}

}  // extern "C"
