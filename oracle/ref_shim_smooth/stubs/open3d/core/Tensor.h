// ref_shim_smooth stub (test infrastructure): the shared core::Tensor stub of ../ref_shim/stubs, plus the one member the
// smoothing functions need and it lacks: To(dtype) to the tensor's own dtype, which upstream answers with a shallow copy
// (SmoothLaplacianCPU and SmoothMLSCPU call indices.To(Int32) on the Int32 lists their search returns).  The shared
// class is compiled under another name and this one derives from it, so the other shims build exactly as before.
#pragma once

#define Tensor SharedStubTensor
#include_next "open3d/core/Tensor.h"
#undef Tensor

namespace open3d {
namespace core {

class Tensor : public SharedStubTensor {
public:
    using SharedStubTensor::SharedStubTensor;
    using SharedStubTensor::To;
    Tensor() = default;
    Tensor(const SharedStubTensor& t) : SharedStubTensor(t) {}
    Tensor To(const Dtype& dtype) const {
        if (dtype == GetDtype()) return *this;
        return SharedStubTensor::To(dtype);
    }
    static Tensor Zeros(const SizeVector& shape, Dtype dtype, const Device& d = Device()) {
        return SharedStubTensor::Zeros(shape, dtype, d);
    }
    static Tensor Empty(const SizeVector& shape, Dtype dtype, const Device& d = Device()) {
        return SharedStubTensor::Empty(shape, dtype, d);
    }
    Tensor Contiguous() const { return *this; }
    Tensor Clone() const { return SharedStubTensor::Clone(); }
};

}  // namespace core
}  // namespace open3d
