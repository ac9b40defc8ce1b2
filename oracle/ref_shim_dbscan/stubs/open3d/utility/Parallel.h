// ref_shim_dbscan stub (test infrastructure): the shared stub, plus the TBB grain size PointCloudCluster.cpp asks for.
#pragma once
#include_next "open3d/utility/Parallel.h"
#include <cstddef>
namespace open3d {
namespace utility {
inline std::size_t DefaultGrainSizeTBB() { return 1; }
}  // namespace utility
}  // namespace open3d
