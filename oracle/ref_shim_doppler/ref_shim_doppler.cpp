// ref_shim_doppler.cpp — TEST INFRASTRUCTURE.  Compiles the reference's own CPU registration kernels, unmodified,
// from where they lie in the reference tree (t/pipelines/kernel/RegistrationCPU.cpp, included whole), against the stub
// core::Tensor / TBB headers of ../ref_shim/stubs, and exports ComputePoseDopplerICPCPU (RegistrationCPU.cpp:427-493:
// PreComputeForDopplerICP, GetJacobianDopplerICP and ComputePoseDopplerICPKernelCPU with the dual robust dispatch) and
// PreComputeForDopplerICP (RegistrationImpl.h:525-541) so that the CPU oracle (oracle/doppler/doppler_oracle.c) can be
// checked against them.  tbb::parallel_reduce is a stub that runs the body once over the whole range (the serial
// order); DecodeAndSolve6x6, which upstream implements with LAPACK, is replaced by a probe that hands the 29 reduced
// scalars back.  The iteration switches live in kernel/Registration.cpp, which is not compiled here: the caller passes
// the kernels and the rejection flag in force.  No reference source is copied into this repository.
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

// ComputePoseDopplerICPCPU for Float32 clouds: R_S_to_V [9], r_v_to_s_in_V, w_v_in_V and v_v_in_V [3] in f32, the
// kernels and the rejection flag in force.  Returns 0, or 1 when the dual dispatch rejects a kernel.
int ref_pose_doppler_sums_f32(const float* src, const float* dops, const float* dirs, const float* tgt, const float* nrm,
                              const int64_t* corr, int64_t n, int64_t m, const float R[9], const float r[3],
                              const float w[3], const float v[3], double period, int reject, double threshold,
                              int method_g, double scale_g, double shape_g, int method_d, double scale_d, double shape_d,
                              double lambda_doppler, double sums29[29]) {
    o3c::Tensor s((void*)src, {n, 3}, o3c::Float32), t((void*)tgt, {m, 3}, o3c::Float32);
    o3c::Tensor d((void*)dops, {n}, o3c::Float32), dr((void*)dirs, {n, 3}, o3c::Float32);
    o3c::Tensor nt((void*)nrm, {m, 3}, o3c::Float32), c((void*)corr, {n}, o3c::Int64);
    o3c::Tensor Rt((void*)R, {9}, o3c::Float32), rt((void*)r, {3}, o3c::Float32);
    o3c::Tensor wt((void*)w, {3}, o3c::Float32), vt((void*)v, {3}, o3c::Float32), pose;
    float residual;
    int count;
    o3r::RobustKernel kg(static_cast<o3r::RobustKernelMethod>(method_g), scale_g, shape_g);
    o3r::RobustKernel kd(static_cast<o3r::RobustKernelMethod>(method_d), scale_d, shape_d);
    try {
        o3k::ComputePoseDopplerICPCPU(s, d, dr, t, nt, c, pose, residual, count, o3c::Float32, o3c::Device(), Rt, rt, wt,
                                      vt, period, reject != 0, threshold, kg, kd, lambda_doppler);
    } catch (const std::exception&) {
        return 1;
    }
    memcpy(sums29, g_sums, sizeof(g_sums));
    return 0;
}

// PreComputeForDopplerICP<float>
void ref_precompute_doppler_f32(const float R[9], const float r[3], const float w[3], const float v[3], float out[3]) {
    o3k::PreComputeForDopplerICP<float>(R, r, w, v, out);
}

}  // extern "C"
