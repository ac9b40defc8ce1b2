// ref_shim_boundary stub (test infrastructure): the shared core::Tensor stub of ../ref_shim/stubs, plus the one member
// ComputeBoundaryPointsCPU needs and it lacks: Full(shape, value, dtype), which allocates the angle buffer.  The shared
// stub's Full is unsupported(), which gcc treats as noreturn and so drops the function's whole body.  The shared class is
// compiled under another name and this one derives from it, so the other shims build exactly as before.
#pragma once

#define Tensor SharedStubTensor
#include_next "open3d/core/Tensor.h"
#undef Tensor

namespace open3d {
namespace core {

class Tensor : public SharedStubTensor {
public:
    using SharedStubTensor::SharedStubTensor;
    Tensor() = default;
    Tensor(const SharedStubTensor& t) : SharedStubTensor(t) {}
    // owning, every element set to value in dtype (Float32 or Float64)
    template <typename T>
    static Tensor Full(const SizeVector& shape, T value, Dtype dtype, const Device& d = Device()) {
        Tensor t(shape, dtype, d);
        const int64_t n = t.NumElements();
        if (dtype == Dtype::Float32) {
            float* p = t.GetDataPtr<float>();
            for (int64_t i = 0; i < n; ++i) p[i] = static_cast<float>(value);
        } else if (dtype == Dtype::Float64) {
            double* p = t.GetDataPtr<double>();
            for (int64_t i = 0; i < n; ++i) p[i] = static_cast<double>(value);
        } else {
            utility::LogError("ref_shim_boundary Tensor::Full: Float32 and Float64 only");
        }
        return t;
    }
    static Tensor Zeros(const SizeVector& shape, Dtype dtype, const Device& d = Device()) {
        return SharedStubTensor::Zeros(shape, dtype, d);
    }
    Tensor Contiguous() const { return *this; }
};

}  // namespace core
}  // namespace open3d
