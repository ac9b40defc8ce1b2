// ref_shim_segment.cpp — TEST INFRASTRUCTURE.  Exports the reference's own geometry::PointCloud::SegmentPlane and its
// RandomSampler (geometry/PointCloudSegmentation.cpp, compiled unmodified as part of this translation unit, because
// RandomSampler is local to that file) and utility::random::Seed (utility/Random.cpp, compiled beside it) through C,
// so that the library's sampler and the CPU oracle (oracle/segment/segment_oracle.c) can be checked against them.
// No reference source is copied into this repository.
#include <cstdint>
#include <cstring>
#include <string>

#include "open3d/geometry/PointCloudSegmentation.cpp"
#include "open3d/utility/Random.h"

namespace open3d {
namespace geometry {

// TriangleMesh::ComputeTrianglePlane (geometry/TriangleMesh.cpp:1248-1262), restated: that file needs far more of the
// reference than this shim provides.
Eigen::Vector4d TriangleMesh::ComputeTrianglePlane(const Eigen::Vector3d& p0, const Eigen::Vector3d& p1,
                                                   const Eigen::Vector3d& p2) {
    const Eigen::Vector3d e0 = p1 - p0;
    const Eigen::Vector3d e1 = p2 - p0;
    Eigen::Vector3d abc = e0.cross(e1);
    double norm = abc.norm();
    if (norm == 0) return Eigen::Vector4d(0, 0, 0, 0);
    abc /= abc.norm();
    double d = -abc.dot(p0);
    return Eigen::Vector4d(abc(0), abc(1), abc(2), d);
}

}  // namespace geometry
}  // namespace open3d

static std::string g_error;

extern "C" {

const char* ref_segment_last_error() { return g_error.c_str(); }

void ref_random_seed(int seed) { open3d::utility::random::Seed(seed); }

// out [num_samples][sample_size]: what SegmentPlane's pre-generation loop (:183-188) draws for a cloud of n points.
void ref_random_sample(int64_t n, int sample_size, int num_samples, int64_t* out) {
    open3d::geometry::RandomSampler<size_t> sampler((size_t)n);
    for (int s = 0; s < num_samples; ++s) {
        const std::vector<size_t> row = sampler((size_t)sample_size);
        for (int k = 0; k < sample_size; ++k) out[(int64_t)s * sample_size + k] = (int64_t)row[k];
    }
}

// The reference's SegmentPlane on the f32 points [n,3], converted to f64 as t::geometry::PointCloud::ToLegacy does.
// inliers needs n entries.  debug receives the summary line: {fitness, rmse}, evaluated receives the hypothesis count.
// Returns 0, or -1 when the reference raised (its message in ref_segment_last_error).
int ref_segment_plane(const float* points, int64_t n, double distance_threshold, int ransac_n, int num_iterations,
                      double probability, double* plane, int64_t* inliers, int64_t* num_inliers, double* debug,
                      int64_t* evaluated) {
    try {
        open3d::geometry::PointCloud pc;
        pc.points_.resize((std::size_t)n);
        for (int64_t i = 0; i < n; ++i)
            pc.points_[i] = Eigen::Vector3d(points[3 * i], points[3 * i + 1], points[3 * i + 2]);
        open3d::utility::g_ransac_debug = {};
        auto [model, idx] = pc.SegmentPlane(distance_threshold, ransac_n, num_iterations, probability);
        for (int k = 0; k < 4; ++k) plane[k] = model(k);
        for (size_t k = 0; k < idx.size(); ++k) inliers[k] = (int64_t)idx[k];
        *num_inliers = (int64_t)idx.size();
        debug[0] = open3d::utility::g_ransac_debug.fitness;
        debug[1] = open3d::utility::g_ransac_debug.rmse;
        *evaluated = (int64_t)open3d::utility::g_ransac_debug.iterations;
        return 0;
    } catch (const std::exception& e) {
        g_error = e.what();
        return -1;
    }
}

}  // extern "C"
