// ref_shim_projection.cpp — TEST INFRASTRUCTURE.  Compiles the reference's own t/geometry/kernel/PointCloudCPU.cpp
// unmodified (ProjectCPU, and through its include of PointCloudImpl.h, UnprojectCPU), from where the file lies in the
// reference tree, against the stub core::Tensor / ParallelFor / TBB headers of ../ref_shim/stubs, and exports both
// through C functions so that the CPU oracle (oracle/projection/projection_oracle.c) can be checked against the real
// thing.  Only PointCloudCPU.cpp is included: PointCloudImpl.h has no include guard.  No reference source is copied
// into this repository.
#include <cmath>
#include <cstdint>
#include <cstring>

using std::abs;
using std::max;
using std::min;

#include "open3d/t/geometry/kernel/PointCloudCPU.cpp"   // from -I <reference>/cpp

namespace o3c = open3d::core;
namespace o3p = open3d::t::geometry::kernel::pointcloud;

extern "C" {

// UnprojectCPU (PointCloudImpl.h:43-144).  depth [rows][cols] u16 (depth_f32 == 0) or f32; color NULL or
// [rows][cols][3] f32 (upstream converts the colour image to Float32 first, PointCloud.cpp:1456).  Rows come in the
// atomic counter's order; returns their number.
int64_t ref_unproject(const void* depth, int depth_f32, int rows, int cols, const float* color, const double K[9],
                      const double E[16], float depth_scale, float depth_max, int stride, float* points_out,
                      float* colors_out) {
    const o3c::Tensor d((void*)depth, {rows, cols, 1}, depth_f32 ? o3c::Float32 : o3c::UInt16);
    const o3c::Tensor k((void*)K, {3, 3}, o3c::Float64), e((void*)E, {4, 4}, o3c::Float64);
    o3c::Tensor pts, cols_t;
    if (color) {
        const o3c::Tensor c((void*)color, {rows, cols, 3}, o3c::Float32);
        o3p::UnprojectCPU(d, c, pts, cols_t, k, e, depth_scale, depth_max, stride);
    } else {
        o3p::UnprojectCPU(d, std::nullopt, pts, std::nullopt, k, e, depth_scale, depth_max, stride);
    }
    const int64_t n = pts.GetShape(0);
    if (n > 0) {
        std::memcpy(points_out, pts.GetDataPtr<float>(), n * 3 * sizeof(float));
        if (color) std::memcpy(colors_out, cols_t.GetDataPtr<float>(), n * 3 * sizeof(float));
    }
    return n;
}

// ProjectCPU (PointCloudCPU.cpp:21-90) into depth_out [rows][cols] and color_out [rows][cols][3], which the caller
// zero-fills as ProjectToDepthImage / ProjectToRGBDImage do (PointCloud.cpp:1486-1518).
void ref_project(const float* points, const float* colors, int64_t n, const double K[9], const double E[16],
                 float depth_scale, float depth_max, int rows, int cols, float* depth_out, float* color_out) {
    o3c::Tensor depth((void*)depth_out, {rows, cols, 1}, o3c::Float32);
    const o3c::Tensor p((void*)points, {n, 3}, o3c::Float32);
    const o3c::Tensor k((void*)K, {3, 3}, o3c::Float64), e((void*)E, {4, 4}, o3c::Float64);
    if (colors) {
        o3c::Tensor img((void*)color_out, {rows, cols, 3}, o3c::Float32);
        const o3c::Tensor c((void*)colors, {n, 3}, o3c::Float32);
        o3p::ProjectCPU(depth, img, p, c, k, e, depth_scale, depth_max);
    } else {
        o3p::ProjectCPU(depth, std::nullopt, p, std::nullopt, k, e, depth_scale, depth_max);
    }
}

}  // extern "C"
