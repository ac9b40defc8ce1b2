// ref_shim_dbscan stub (test infrastructure): a progress bar that shows nothing.
#pragma once
#include <cstddef>
#include <string>
namespace open3d {
namespace utility {
class ProgressBar {
public:
    ProgressBar(std::size_t, const std::string&, bool = false) {}
    void Reset(std::size_t, const std::string&, bool) {}
    ProgressBar& operator++() { return *this; }
    ProgressBar& operator+=(std::size_t) { return *this; }
};
}  // namespace utility
}  // namespace open3d
