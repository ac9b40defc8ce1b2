// ref_shim_symmetric.cpp — TEST INFRASTRUCTURE.  Compiles the reference's own CPU registration kernels, unmodified,
// from where they lie in the reference tree (t/pipelines/kernel/RegistrationCPU.cpp, included whole), against the stub
// core::Tensor / TBB headers of ../ref_shim/stubs, and exports ComputePoseSymmetricCPU (RegistrationCPU.cpp:124-218:
// GetJacobianSymmetric, the objective-residual weight and the 29-slot accumulation as one function) so that the CPU
// oracle (oracle/symmetric/symmetric_oracle.c) can be checked against it.  tbb::parallel_reduce is a stub that runs the
// body once over the whole range (the serial order); DecodeAndSolve6x6, which upstream implements with LAPACK, is
// replaced by a probe that hands the 29 reduced scalars back.  No reference source is copied into this repository.
#include <cmath>
#include <cstdint>
#include <cstring>

using std::abs;
using std::exp;
using std::max;
using std::min;
using std::pow;

#include "open3d/t/pipelines/kernel/RegistrationCPU.cpp"   // from -I <reference>/cpp

namespace {
thread_local double g_sums[29];
}

namespace open3d {
namespace t {
namespace pipelines {
namespace kernel {
// probe: TransformationConverter.cpp:189-226 receives exactly this tensor
void DecodeAndSolve6x6(const core::Tensor& A, core::Tensor&, float& inlier_residual, int& inlier_count) {
    for (int i = 0; i < 29; ++i)
        g_sums[i] = A.GetDtype() == core::Float32 ? (double)A.GetDataPtr<float>()[i] : A.GetDataPtr<double>()[i];
    inlier_residual = (float)g_sums[27];
    inlier_count = (int)g_sums[28];
}
}  // namespace kernel
}  // namespace pipelines
}  // namespace t
}  // namespace open3d

namespace o3c = open3d::core;
namespace o3k = open3d::t::pipelines::kernel;
namespace o3r = open3d::t::pipelines::registration;

extern "C" {

// ComputePoseSymmetricCPU (RegistrationCPU.cpp:182-218), Float32 clouds, about the given Float32 means
void ref_pose_symmetric_sums_f32(const float* src, const float* tgt, const float* src_n, const float* tgt_n,
                                 const int64_t* corr, int64_t n, int64_t m, const float ms[3], const float mt[3], int method,
                                 double scale, double shape, double sums29[29]) {
    o3c::Tensor s((void*)src, {n, 3}, o3c::Float32), t((void*)tgt, {m, 3}, o3c::Float32);
    o3c::Tensor sn((void*)src_n, {n, 3}, o3c::Float32), tn((void*)tgt_n, {m, 3}, o3c::Float32);
    o3c::Tensor sm((void*)ms, {3}, o3c::Float32), tm((void*)mt, {3}, o3c::Float32);
    o3c::Tensor c((void*)corr, {n}, o3c::Int64), pose;
    float residual;
    int count;
    o3r::RobustKernel k(static_cast<o3r::RobustKernelMethod>(method), scale, shape);
    o3k::ComputePoseSymmetricCPU(s, t, sn, tn, c, sm, tm, pose, residual, count, o3c::Float32, o3c::Device(), k);
    memcpy(sums29, g_sums, sizeof(g_sums));
}

}  // extern "C"
