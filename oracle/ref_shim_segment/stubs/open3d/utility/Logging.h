// ref_shim_segment stub: utility::LogError throws (utility/Logging.h:44-53); LogDebug records SegmentPlane's summary
// line (PointCloudSegmentation.cpp:273-277: inlier count, fitness, rmse, evaluated hypotheses) for the shim to report;
// the rest is silent.
#pragma once
#include <cstddef>
#include <stdexcept>
#include <string>
namespace open3d {
namespace utility {
struct RansacDebug {
    size_t inliers = 0;
    double fitness = 0, rmse = 0;
    size_t iterations = 0;
};
inline RansacDebug g_ransac_debug;
template <typename... Args>
[[noreturn]] inline void LogError(const char* fmt, Args&&...) { throw std::runtime_error(fmt); }
template <typename... Args>
inline void LogWarning(const char*, Args&&...) {}
template <typename... Args>
inline void LogInfo(const char*, Args&&...) {}
template <typename... Args>
inline void LogDebug(const char*, Args&&...) {}
inline void LogDebug(const char*, size_t inliers, double fitness, double rmse, size_t iterations) {
    g_ransac_debug = RansacDebug{inliers, fitness, rmse, iterations};
}
}  // namespace utility
}  // namespace open3d
