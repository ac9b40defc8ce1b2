// ref_shim_fgr stub (test infrastructure): a brute-force f64 KDTreeFlann, over points or over feature columns.  SearchHybrid with max_nn 1 returns the
// nearest point with d^2 < radius^2 (strict, the bound nanoflann's radius search applies), d^2 = ((dx^2 + dy^2) + dz^2)
// with d = query - point, ties to the lowest index (nanoflann's tie order depends on its tree).  SearchKNN with knn 1
// over a Feature returns the column with the least sum over rows, in row order, of (q_r - f_r)^2, ties to the lowest.
#pragma once
#include <Eigen/Core>
#include <vector>
#include "open3d/geometry/PointCloud.h"
namespace open3d {
namespace pipelines {
namespace registration {
class Feature;
}
}  // namespace pipelines
namespace geometry {
class KDTreeFlann {
public:
    KDTreeFlann() = default;
    explicit KDTreeFlann(const PointCloud& g) { SetGeometry(g); }
    explicit KDTreeFlann(const pipelines::registration::Feature& f);   // defined in the shim
    template <typename T>
    int SearchKNN(const T& q, int knn, std::vector<int>& indices, std::vector<double>& distance2) const {
        double best = 0;
        int bi = -1;
        for (int j = 0; j < cols_; ++j) {
            double d2 = 0.0;
            for (int r = 0; r < dim_; ++r) {
                const double d = q(r) - feat_[(size_t)j * dim_ + r];
                d2 = d2 + d * d;
            }
            if (bi < 0 || d2 < best) {
                best = d2;
                bi = j;
            }
        }
        if (bi < 0 || knn < 1) return -1;
        indices.resize(1);
        distance2.resize(1);
        indices[0] = bi;
        distance2[0] = best;
        return 1;
    }
    std::vector<double> feat_;   // column-major [cols_][dim_]
    int dim_ = 0, cols_ = 0;
    KDTreeFlann(const KDTreeFlann&) = delete;
    bool SetGeometry(const PointCloud& g) {
        pts_ = &g.points_;
        return true;
    }
    template <typename T>
    int SearchHybrid(const T& q, double radius, int max_nn, std::vector<int>& indices,
                     std::vector<double>& distance2) const {
        const double r2 = radius * radius;
        double best = 0;
        int bi = -1;
        for (size_t j = 0; j < pts_->size(); ++j) {
            const Eigen::Vector3d d = Eigen::Vector3d(q(0), q(1), q(2)) - (*pts_)[j];
            const double d2 = d.squaredNorm();
            if (d2 < r2 && (bi < 0 || d2 < best)) {
                best = d2;
                bi = (int)j;
            }
        }
        if (bi < 0 || max_nn < 1) return 0;
        indices.resize(1);
        distance2.resize(1);
        indices[0] = bi;
        distance2[0] = best;
        return 1;
    }

private:
    const std::vector<Eigen::Vector3d>* pts_ = nullptr;
};
}  // namespace geometry
}  // namespace open3d
