// ref_shim_fgr stub (test infrastructure): tbb::parallel_invoke on one thread, in argument order.
#pragma once
namespace tbb {
template <typename... F>
void parallel_invoke(const F&... f) {
    (f(), ...);
}
}  // namespace tbb
