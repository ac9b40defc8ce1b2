// ref_shim_dbscan stub (test infrastructure): KDTreeFlann::SearchRadius (geometry/KDTreeFlann.cpp:114-135) as a brute
// force with the predicate of the nanoflann radius search it calls, which is not in the reference tree: the query is
// passed with radius * radius, d2 = ((0 + dx dx) + dy dy) + dz dz in f64 with dx = query.x - point.x
// (L2_Adaptor::evalMetric, dimension 3), and a point is kept iff d2 < radius * radius (RadiusResultSet::addPoint).
#pragma once
#include <vector>
#include "open3d/geometry/PointCloud.h"
namespace open3d {
namespace geometry {
class KDTreeFlann {
public:
    explicit KDTreeFlann(const PointCloud& pc) : pc_(pc) {}
    template <typename T>
    int SearchRadius(const T& query, double radius, std::vector<int>& indices, std::vector<double>& distance2) const {
        const double r2 = radius * radius;
        indices.clear();
        distance2.clear();
        for (std::size_t j = 0; j < pc_.points_.size(); ++j) {
            const auto& p = pc_.points_[j];
            double d2 = 0;
            for (int a = 0; a < 3; ++a) {
                const double diff = query[a] - p[a];
                d2 += diff * diff;
            }
            if (d2 < r2) {
                indices.push_back((int)j);
                distance2.push_back(d2);
            }
        }
        return (int)indices.size();
    }

private:
    const PointCloud& pc_;
};
}  // namespace geometry
}  // namespace open3d
