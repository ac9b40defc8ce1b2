// ref_shim_smooth stub (test infrastructure): the NearestNeighborSearch that PointCloudImpl.h's smoothing functions
// call, answering KnnSearch and HybridSearch by brute force through the oracle's searches (oracle/knn's orc_knn_f32,
// oracle/icp_oracle.c's orc_hybrid_search_bruteforce_f32), which rank by the device's dist^2 and give ties to the lower
// index.  The caller installs them with ref_smooth_set_search.  It comes before ../ref_shim/stubs on the include path.
#pragma once
#include <algorithm>
#include <cstdint>
#include <tuple>
#include <utility>

#include "open3d/core/Tensor.h"

extern "C" {
typedef void (*ref_smooth_knn_fn)(const float* points, int64_t m, const float* queries, int64_t nq, int k,
                                  int32_t* idx, float* d2);
typedef void (*ref_smooth_hybrid_fn)(const float* points, int64_t m, const float* queries, int64_t nq, double radius,
                                     int max_knn, int32_t* idx, float* d2, int32_t* counts);
}

namespace open3d {
namespace core {
namespace nns {
inline ref_smooth_knn_fn g_knn = nullptr;
inline ref_smooth_hybrid_fn g_hybrid = nullptr;

class NearestNeighborSearch {
public:
    NearestNeighborSearch(const Tensor& data, const Dtype& = Int64) : data_(data) {}
    bool KnnIndex() { return g_knn != nullptr && data_.GetDtype() == Float32; }
    bool HybridIndex(double = 0) { return g_hybrid != nullptr && data_.GetDtype() == Float32; }
    bool FixedRadiusIndex(double = 0) { unsupported(); }
    std::pair<Tensor, Tensor> KnnSearch(const Tensor& q, int k) {
        const int64_t m = data_.GetLength(), nq = q.GetLength(), kp = std::min<int64_t>(k, m);
        Tensor idx({nq, kp}, Int32), d2({nq, kp}, Float32);
        g_knn(data_.GetDataPtr<float>(), m, q.GetDataPtr<float>(), nq, k, idx.GetDataPtr<int32_t>(),
              d2.GetDataPtr<float>());
        return {idx, d2};
    }
    std::tuple<Tensor, Tensor, Tensor> FixedRadiusSearch(const Tensor&, double, bool = true) { unsupported(); }
    std::tuple<Tensor, Tensor, Tensor> HybridSearch(const Tensor& q, double radius, int max_knn) const {
        const int64_t m = data_.GetLength(), nq = q.GetLength();
        Tensor idx({nq, (int64_t)max_knn}, Int32), d2({nq, (int64_t)max_knn}, Float32), cnt({nq}, Int32);
        g_hybrid(data_.GetDataPtr<float>(), m, q.GetDataPtr<float>(), nq, radius, max_knn, idx.GetDataPtr<int32_t>(),
                 d2.GetDataPtr<float>(), cnt.GetDataPtr<int32_t>());
        return {idx, d2, cnt};
    }

private:
    [[noreturn]] static void unsupported() { utility::LogError("ref_shim_smooth: fixed-radius search is not available"); }
    Tensor data_;
};
}  // namespace nns
}  // namespace core
}  // namespace open3d
