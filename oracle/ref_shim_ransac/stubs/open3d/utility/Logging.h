// ref_shim_ransac stub (test infrastructure): LogError throws (utility/Logging.h:44-53); LogWarning counts its calls;
// LogDebug records the validation count of RegistrationRANSACBasedOnCorrespondence's summary line
// ("RANSAC exits after {:d} validations ...", Registration.cpp:373-377).  Everything else is silent.
#pragma once
#include <cstring>
#include <stdexcept>
#include <type_traits>
namespace open3d {
namespace utility {
struct RansacLog {
    long long validations = -1;
    long long warnings = 0;
};
inline RansacLog& ransac_log() {
    static RansacLog g;
    return g;
}
template <typename... Args>
[[noreturn]] inline void LogError(const char* fmt, Args&&...) { throw std::runtime_error(fmt); }
template <typename... Args>
inline void LogWarning(const char*, Args&&...) { ++ransac_log().warnings; }
template <typename... Args>
inline void LogInfo(const char*, Args&&...) {}
template <typename First, typename... Args>
inline void LogDebug(const char* fmt, First&& first, Args&&...) {
    if constexpr (std::is_integral_v<std::decay_t<First>>)
        if (std::strncmp(fmt, "RANSAC exits after", 18) == 0) ransac_log().validations = (long long)first;
}
inline void LogDebug(const char*) {}
}  // namespace utility
}  // namespace open3d
