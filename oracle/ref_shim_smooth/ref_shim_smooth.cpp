// ref_shim_smooth.cpp — TEST INFRASTRUCTURE.  Compiles the reference's own smoothing code, unmodified, from where it
// lies in the reference tree (t/geometry/kernel/PointCloudImpl.h, included as a header), against the stub
// core::Tensor / ParallelFor headers of ../ref_shim/stubs and the brute-force NearestNeighborSearch of stubs/, and
// exports its four whole CPU functions through C so that the CPU oracle (oracle/smooth/smooth_oracle.c) can be
// checked against them: SmoothLaplacianCPU (:1408-1446), SmoothTaubinCPU (:1448-1495), SmoothMLSCPU (:1497-1657) and
// SmoothBilateralCPU (:1659-1753).  Each returns 0, or -1 when the reference raised.  No reference source is copied
// into this repository.
#include <cmath>
#include <cstdint>
#include <cstring>

using std::abs;
using std::max;
using std::min;

#include "open3d/t/geometry/kernel/PointCloudImpl.h"   // from -I <reference>/cpp

namespace o3c = open3d::core;
namespace o3p = open3d::t::geometry::kernel::pointcloud;

namespace {
template <typename F>
int guarded(F&& f) {
    try {
        f();
        return 0;
    } catch (const std::exception&) {
        return -1;
    }
}

void copy_out(const o3c::Tensor& t, float* out) {
    std::memcpy(out, t.GetDataPtr<float>(), (size_t)t.NumElements() * sizeof(float));
}
}  // namespace

extern "C" {

void ref_smooth_set_search(ref_smooth_knn_fn knn, ref_smooth_hybrid_fn hybrid) {
    o3c::nns::g_knn = knn;
    o3c::nns::g_hybrid = hybrid;
}

int ref_smooth_laplacian_f32(const float* points, int64_t n, int64_t iterations, double lambda, int max_nn, int fixed,
                             float* out) {
    return guarded([&] {
        const o3c::Tensor p((void*)points, {n, 3}, o3c::Float32);
        o3c::Tensor s;
        o3p::SmoothLaplacianCPU(p, s, (size_t)iterations, lambda, max_nn, fixed != 0);
        copy_out(s, out);
    });
}

int ref_smooth_taubin_f32(const float* points, int64_t n, int64_t iterations, double lambda, double mu, int max_nn,
                          int fixed, float* out) {
    return guarded([&] {
        const o3c::Tensor p((void*)points, {n, 3}, o3c::Float32);
        o3c::Tensor s;
        o3p::SmoothTaubinCPU(p, s, (size_t)iterations, lambda, mu, max_nn, fixed != 0);
        copy_out(s, out);
    });
}

// normals [n,3] (or NULL): updated in place, as upstream's result normals
int ref_smooth_mls_f32(const float* points, int64_t n, double radius, int max_nn, float* normals, float* out) {
    return guarded([&] {
        const o3c::Tensor p((void*)points, {n, 3}, o3c::Float32);
        o3c::Tensor s, nn;
        if (normals) nn = o3c::Tensor((void*)normals, {n, 3}, o3c::Float32);
        o3p::SmoothMLSCPU(p, s, nn, normals != nullptr, radius, max_nn);
        copy_out(s, out);
    });
}

int ref_smooth_bilateral_f32(const float* points, const float* normals, int64_t n, double radius, int max_nn,
                             double sigma_s, double sigma_r, float* out) {
    return guarded([&] {
        const o3c::Tensor p((void*)points, {n, 3}, o3c::Float32), nn((void*)normals, {n, 3}, o3c::Float32);
        o3c::Tensor s;
        o3p::SmoothBilateralCPU(p, nn, s, radius, max_nn, sigma_s, sigma_r);
        copy_out(s, out);
    });
}

}  // extern "C"
