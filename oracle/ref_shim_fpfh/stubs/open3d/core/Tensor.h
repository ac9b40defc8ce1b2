// ref_shim_fpfh stub (test infrastructure): the shared core::Tensor stub of ../ref_shim/stubs, plus the members that
// ComputeFPFHFeatureCPU names only on its masked path (NonZero, GetItem, IndexSet, Arange and core::TensorKey).  The
// shim calls the unmasked path, so they are never run; they raise if they are.  The shared class is compiled under
// another name and this one derives from it, so the other shims build exactly as before.
#pragma once

#define Tensor SharedStubTensor
#include_next "open3d/core/Tensor.h"
#undef Tensor

namespace open3d {
namespace core {

struct TensorKey {
    static TensorKey Index(int64_t) { return TensorKey(); }
};

class Tensor : public SharedStubTensor {
public:
    using SharedStubTensor::SharedStubTensor;
    Tensor() = default;
    Tensor(const SharedStubTensor& t) : SharedStubTensor(t) {}
    static Tensor Zeros(const SizeVector& shape, Dtype dtype, const Device& d = Device()) {
        return SharedStubTensor::Zeros(shape, dtype, d);
    }
    static Tensor Empty(const SizeVector& shape, Dtype dtype, const Device& d = Device()) {
        return SharedStubTensor::Empty(shape, dtype, d);
    }
    template <typename T>
    static Tensor Full(const SizeVector&, T, Dtype, const Device& = Device()) { masked(); return Tensor(); }
    static Tensor Arange(int64_t, int64_t, int64_t, Dtype, const Device& = Device()) { masked(); return Tensor(); }
    Tensor NonZero() const { masked(); return Tensor(); }
    Tensor GetItem(const TensorKey&) const { masked(); return Tensor(); }
    void IndexSet(const std::vector<Tensor>&, const Tensor&) { masked(); }

private:
    static void masked() { utility::LogError("ref_shim_fpfh Tensor: the masked path is not stubbed"); }
};

}  // namespace core
}  // namespace open3d
