// ref_shim_fgr stub (test infrastructure): LogError throws (utility/Logging.h:44-53) with the format string as its
// message; LogWarning counts its calls; LogDebug records the integers of FastGlobalRegistration.cpp's "Initial
// matchings : {}" and "{:d} tuples ({:d} trial, {:d} actual)." lines and of RANSAC's summary line.  Everything else is
// silent.
#pragma once
#include <cstring>
#include <stdexcept>
#include <type_traits>
namespace open3d {
namespace utility {
struct RansacLog {
    long long validations = -1;
    long long warnings = 0;
    long long cross = -1, tuples = -1, trials = -1, actual = -1;
};
inline RansacLog& ransac_log() {
    static RansacLog g;
    return g;
}
template <typename T>
long long as_ll(const T& v) {
    if constexpr (std::is_integral_v<std::decay_t<T>>)
        return (long long)v;
    else
        return -1;
}
template <typename... Args>
[[noreturn]] inline void LogError(const char* fmt, Args&&...) { throw std::runtime_error(fmt); }
template <typename... Args>
inline void LogWarning(const char*, Args&&...) { ++ransac_log().warnings; }
template <typename... Args>
inline void LogInfo(const char*, Args&&...) {}
template <typename... Args>
inline void LogDebug(const char* fmt, Args&&... args) {
    const long long v[] = {as_ll(args)..., -1};
    if (std::strncmp(fmt, "RANSAC exits after", 18) == 0) ransac_log().validations = v[0];
    if (std::strncmp(fmt, "Initial matchings", 17) == 0) ransac_log().cross = v[0];
    if (std::strncmp(fmt, "{:d} tuples", 11) == 0) {
        ransac_log().tuples = v[0];
        ransac_log().trials = v[1];
        ransac_log().actual = v[2];
    }
}
}  // namespace utility
}  // namespace open3d
