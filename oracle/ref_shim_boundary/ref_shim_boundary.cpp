// ref_shim_boundary.cpp — TEST INFRASTRUCTURE.  Compiles the reference's own boundary detection, unmodified, from where
// it lies in the reference tree (t/geometry/kernel/PointCloudImpl.h, included as a header), against the stub
// core::Tensor / ParallelFor headers of stubs/ and ../ref_shim/stubs, and exports it through C functions so that the
// CPU oracle (oracle/boundary/boundary_oracle.c) can be checked against the real thing:
//   GetCoordinateSystemOnPlane<float> (:354-379), one normal;
//   IsBoundaryPoints<float> (:424-440), one sorted angle list;
//   ComputeBoundaryPointsCPU (:444-506), the whole function over given neighbour lists.
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

void ref_coordinate_system_on_plane_f32(const float normal[3], float u[3], float v[3]) {
    o3p::GetCoordinateSystemOnPlane<float>(normal, u, v);
}

int ref_is_boundary_points_f32(const float* angles, int counts, double angle_threshold) {
    return o3p::IsBoundaryPoints<float>(angles, counts, angle_threshold) ? 1 : 0;
}

// indices [n, nn_size] and counts [n] are the hybrid search's; mask [n] (bool) must be zero on entry, as upstream's
void ref_compute_boundary_points_f32(const float* points, const float* normals, int64_t n, const int32_t* indices,
                                     int64_t nn_size, const int32_t* counts, uint8_t* mask, double angle_threshold) {
    const o3c::Tensor p((void*)points, {n, 3}, o3c::Float32), nrm((void*)normals, {n, 3}, o3c::Float32);
    const o3c::Tensor idx((void*)indices, {n, nn_size}, o3c::Int32), cnt((void*)counts, {n}, o3c::Int32);
    o3c::Tensor m((void*)mask, {n}, o3c::Bool);
    o3p::ComputeBoundaryPointsCPU(p, nrm, idx, cnt, m, angle_threshold);
}

}  // extern "C"
