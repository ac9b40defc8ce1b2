// ref_shim_ransac.cpp — TEST INFRASTRUCTURE.  Exports the reference's own RegistrationRANSACBasedOnCorrespondence
// (pipelines/registration/Registration.cpp), its checkers (CorrespondenceChecker.cpp) and UniformIntGenerator<int>
// (utility/Random.h, with utility/Random.cpp compiled beside it) through C, so that the library's generator and the
// CPU oracle (oracle/ransac/ransac_oracle.c) can be checked against them.  The two .cpp files are compiled unmodified
// as part of this translation unit against stubs/ (a minimal Eigen with the stated orders, a brute-force KDTreeFlann,
// the legacy PointCloud, a one-thread parallel_reduce).  No reference source is copied into this repository.
#include <cstdint>
#include <string>

#include "open3d/pipelines/registration/CorrespondenceChecker.cpp"
#include "open3d/pipelines/registration/Registration.cpp"
#include "open3d/utility/Random.h"

namespace open3d {
namespace utility {
// Only CorrespondenceCheckerBasedOnSourceRotation calls it, and the tests never run that checker.
Eigen::Vector6d TransformMatrix4dToVector6d(const Eigen::Matrix4d&) { throw std::runtime_error("not in the shim"); }
}  // namespace utility
namespace pipelines {
namespace registration {
// TransformationEstimationPointToPoint (TransformationEstimation.cpp:19-73): that file needs far more of Eigen than
// the stub provides, so its point-to-point members are restated; ComputeTransformation gathers the pairs into 3 x n
// matrices and calls Eigen::umeyama, which the stub states in the library's order.
double TransformationEstimationPointToPoint::ComputeRMSE(const geometry::PointCloud& source,
                                                         const geometry::PointCloud& target,
                                                         const CorrespondenceSet& corres) const {
    if (corres.empty()) return 0.0;
    double err = 0.0;
    for (const auto& c : corres) err += (source.points_[c[0]] - target.points_[c[1]]).squaredNorm();
    return std::sqrt(err / (double)corres.size());
}
Eigen::Matrix4d TransformationEstimationPointToPoint::ComputeTransformation(const geometry::PointCloud& source,
                                                                            const geometry::PointCloud& target,
                                                                            const CorrespondenceSet& corres) const {
    if (corres.empty()) return Eigen::Matrix4d::Identity();
    Eigen::MatrixXd source_mat(3, corres.size());
    Eigen::MatrixXd target_mat(3, corres.size());
    for (size_t i = 0; i < corres.size(); i++) {
        source_mat.block<3, 1>(0, i) = source.points_[corres[i][0]];
        target_mat.block<3, 1>(0, i) = target.points_[corres[i][1]];
    }
    return Eigen::umeyama(source_mat, target_mat, with_scaling_);
}
std::tuple<std::shared_ptr<const geometry::PointCloud>, std::shared_ptr<const geometry::PointCloud>>
TransformationEstimationPointToPoint::InitializePointCloudsForTransformation(const geometry::PointCloud& source,
                                                                            const geometry::PointCloud& target,
                                                                            double) const {
    return {std::shared_ptr<const geometry::PointCloud>(&source, [](const geometry::PointCloud*) {}),
            std::shared_ptr<const geometry::PointCloud>(&target, [](const geometry::PointCloud*) {})};
}
// RegistrationRANSACBasedOnFeatureMatching calls it; the tests call the correspondence function directly.
CorrespondenceSet CorrespondencesFromFeatures(const Feature&, const Feature&, bool, float) {
    throw std::runtime_error("not in the shim");
}
}  // namespace registration
}  // namespace pipelines
}  // namespace open3d

namespace {
std::string g_error;
open3d::geometry::PointCloud cloud(const float* p, const float* nrm, int64_t n) {
    open3d::geometry::PointCloud pc;
    pc.points_.resize((size_t)n);
    for (int64_t i = 0; i < n; ++i) pc.points_[i] = Eigen::Vector3d(p[3 * i], p[3 * i + 1], p[3 * i + 2]);
    if (nrm) {
        pc.normals_.resize((size_t)n);
        for (int64_t i = 0; i < n; ++i) pc.normals_[i] = Eigen::Vector3d(nrm[3 * i], nrm[3 * i + 1], nrm[3 * i + 2]);
    }
    return pc;
}
}  // namespace

extern "C" {

const char* ref_ransac_last_error() { return g_error.c_str(); }

void ref_ransac_seed(int seed) { open3d::utility::random::Seed(seed); }

// count draws of UniformIntGenerator<int>(low, high); returns -1 when it raised
int ref_uniform_ints(int low, int high, int64_t count, int* out) {
    try {
        open3d::utility::random::UniformIntGenerator<int> gen(low, high);
        for (int64_t k = 0; k < count; ++k) out[k] = gen();
        return 0;
    } catch (const std::exception& e) {
        g_error = e.what();
        return -1;
    }
}

// The reference's RegistrationRANSACBasedOnCorrespondence on f32 clouds converted to f64 as ToLegacy does, with the
// point-to-point estimate and the checkers whose use_* flag is set (normal_angle in radians: the checker takes its
// cosine).  T receives the transformation row-major, pairs [n][2] the correspondence set, fr {fitness, rmse},
// stats {validations from the summary line, warnings logged}.  Returns 0, or -1 when the reference raised.
int ref_ransac(const float* src, const float* src_nrm, int64_t n, const float* tgt, const float* tgt_nrm, int64_t m,
               const int64_t* corres, int64_t K, double max_dist, int ransac_n, int max_iteration, double confidence,
               int use_edge, double edge, int use_distance, double distance, int use_normal, double normal_angle,
               double* T, int64_t* pairs, int64_t* num_pairs, double* fr, int64_t* stats) {
    using namespace open3d::pipelines::registration;
    try {
        const auto s = cloud(src, src_nrm, n), t = cloud(tgt, tgt_nrm, m);
        CorrespondenceSet cs((size_t)K);
        for (int64_t k = 0; k < K; ++k) cs[k] = Eigen::Vector2i((int)corres[2 * k], (int)corres[2 * k + 1]);
        CorrespondenceCheckerBasedOnEdgeLength ce(edge);
        CorrespondenceCheckerBasedOnDistance cd(distance);
        CorrespondenceCheckerBasedOnNormal cn(normal_angle);
        std::vector<std::reference_wrapper<const CorrespondenceChecker>> checkers;
        if (use_edge) checkers.push_back(ce);
        if (use_distance) checkers.push_back(cd);
        if (use_normal) checkers.push_back(cn);
        open3d::utility::ransac_log() = {};
        const RegistrationResult r = RegistrationRANSACBasedOnCorrespondence(
                s, t, cs, max_dist, TransformationEstimationPointToPoint(false), ransac_n, checkers,
                RANSACConvergenceCriteria(max_iteration, confidence));
        for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 4; ++j) T[4 * i + j] = r.transformation_(i, j);
        for (size_t k = 0; k < r.correspondence_set_.size(); ++k) {
            pairs[2 * k] = r.correspondence_set_[k](0);
            pairs[2 * k + 1] = r.correspondence_set_[k](1);
        }
        *num_pairs = (int64_t)r.correspondence_set_.size();
        fr[0] = r.fitness_;
        fr[1] = r.inlier_rmse_;
        stats[0] = open3d::utility::ransac_log().validations;
        stats[1] = open3d::utility::ransac_log().warnings;
        return 0;
    } catch (const std::exception& e) {
        g_error = e.what();
        return -1;
    }
}

}  // extern "C"
