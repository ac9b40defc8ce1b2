// ref_shim_fpfh.cpp — TEST INFRASTRUCTURE.  Compiles the reference's own FPFH kernel, unmodified, from where it lies in
// the reference tree (t/pipelines/kernel/FeatureImpl.h, included as a header), against the stub core::Tensor /
// ParallelFor headers of stubs/ and ../ref_shim/stubs, and exports it through C functions so that the CPU oracle
// (oracle/fpfh/fpfh_oracle.c) can be checked against the real thing:
//   ComputePairFeature<float> (:23-85), one pair;
//   ComputeFPFHFeatureCPU (:105-293), the whole unmasked function over given neighbour lists.
// No reference source is copied into this repository.
#include <cmath>
#include <cstdint>
#include <cstring>

#include "open3d/t/pipelines/kernel/FeatureImpl.h"   // from -I <reference>/cpp

namespace o3c = open3d::core;
namespace o3k = open3d::t::pipelines::kernel;

extern "C" {

void ref_pair_feature_f32(const float p1[3], const float n1[3], const float p2[3], const float n2[3], float f[4]) {
    o3k::ComputePairFeature<float>(p1, n1, p2, n2, f);
}

// indices / distance2 [n, nn_size] and counts [n] are the neighbour lists; fpfh [n, 33] must be zero on entry, as
// upstream's
void ref_compute_fpfh_feature_f32(const float* points, const float* normals, int64_t n, const int32_t* indices,
                                  const float* distance2, int64_t nn_size, const int32_t* counts, float* fpfh) {
    const o3c::Tensor p((void*)points, {n, 3}, o3c::Float32), nrm((void*)normals, {n, 3}, o3c::Float32);
    const o3c::Tensor idx((void*)indices, {n, nn_size}, o3c::Int32), d2((void*)distance2, {n, nn_size}, o3c::Float32);
    const o3c::Tensor cnt((void*)counts, {n}, o3c::Int32);
    o3c::Tensor out((void*)fpfh, {n, 33}, o3c::Float32);
    o3k::ComputeFPFHFeatureCPU(p, nrm, idx, d2, cnt, out, std::nullopt, std::nullopt);
}

}  // extern "C"
