// ref_shim_fgr stub (test infrastructure): one thread.
#pragma once
#include <atomic>
#include <cstddef>
namespace open3d {
namespace utility {
inline int EstimateMaxThreads() { return 1; }
inline bool InParallel() { return false; }
inline std::size_t& DefaultGrainSizeTBB() noexcept {
    static std::size_t g = 1;
    return g;
}
}  // namespace utility
}  // namespace open3d
