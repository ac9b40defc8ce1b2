// ref_shim_dbscan.cpp — TEST INFRASTRUCTURE.  Exports the reference's own geometry::PointCloud::ClusterDBSCAN
// (geometry/PointCloudCluster.cpp:21-97, compiled unmodified beside this file) through C, so that the CPU oracle
// (oracle/dbscan/dbscan_oracle.c) can be checked against it.  Its neighbour search is the brute force of
// stubs/open3d/geometry/KDTreeFlann.h.  No reference source is copied into this repository.
#include <cstdint>

#include "open3d/geometry/PointCloud.h"

extern "C" {

// labels [n]: the reference's labels for the f32 points [n,3], converted to f64 as t::geometry::PointCloud::ToLegacy
// does.  Returns 0, or -1 when the reference raised.
int ref_cluster_dbscan_f32(const float* points, int64_t n, double eps, int64_t min_points, int32_t* labels) {
    try {
        open3d::geometry::PointCloud pc;
        pc.points_.resize((std::size_t)n);
        for (int64_t i = 0; i < n; ++i)
            for (int a = 0; a < 3; ++a) pc.points_[i][a] = (double)points[3 * i + a];
        const std::vector<int> out = pc.ClusterDBSCAN(eps, (std::size_t)min_points, false);
        for (int64_t i = 0; i < n; ++i) labels[i] = out[i];
        return 0;
    } catch (...) {
        return -1;
    }
}

}  // extern "C"
