// ref_shim_fgr.cpp — TEST INFRASTRUCTURE.  Exports the reference's own FastGlobalRegistrationBasedOnCorrespondence
// and FastGlobalRegistrationBasedOnFeatureMatching (pipelines/registration/FastGlobalRegistration.cpp, with
// Registration.cpp's EvaluateRegistration) and UniformIntGenerator<int> (utility/Random.h, with utility/Random.cpp
// compiled beside it) through C, so that the CPU oracle (oracle/fgr/fgr_oracle.c) can be checked against them.  The
// two .cpp files are compiled unmodified as part of this translation unit against stubs/ (a minimal Eigen with the
// stated orders, a brute-force KDTreeFlann over points and over features, the legacy PointCloud, one-thread TBB).
// utility/Eigen.cpp needs Eigen's sparse module and far more of the dense one than the stub carries, so the two of
// its functions that FGR calls, SolveLinearSystemPSD and TransformVector6dToMatrix4d, are restated below as upstream
// writes them.  No reference source is copied into this repository.
#include <cstdint>
#include <string>

#include <Eigen/Geometry>

#include "open3d/pipelines/registration/FastGlobalRegistration.cpp"
#include "open3d/pipelines/registration/Registration.cpp"
#include "open3d/utility/Random.h"

namespace open3d {
namespace utility {
Eigen::Vector6d TransformMatrix4dToVector6d(const Eigen::Matrix4d&) { throw std::runtime_error("not in the shim"); }
// utility/Eigen.cpp:24-77 on the dense path FGR takes (prefer_sparse, check_symmetric, check_det, check_psd false)
std::tuple<bool, Eigen::VectorXd> SolveLinearSystemPSD(const Eigen::MatrixXd& A, const Eigen::VectorXd& b, bool, bool,
                                                       bool, bool) {
    Eigen::VectorXd x(b.size());
    x = A.ldlt().solve(b);
    return std::make_tuple(true, std::move(x));
}
// utility/Eigen.cpp:79-89
Eigen::Matrix4d TransformVector6dToMatrix4d(const Eigen::Vector6d& input) {
    Eigen::Matrix4d output;
    output.setIdentity();
    output.block<3, 3>(0, 0) = (Eigen::AngleAxisd(input(2), Eigen::Vector3d::UnitZ()) *
                                Eigen::AngleAxisd(input(1), Eigen::Vector3d::UnitY()) *
                                Eigen::AngleAxisd(input(0), Eigen::Vector3d::UnitX()))
                                       .matrix();
    output.block<3, 1>(0, 3) = input.block<3, 1>(3, 0);
    return output;
}
}  // namespace utility
namespace geometry {
KDTreeFlann::KDTreeFlann(const pipelines::registration::Feature& f) {
    dim_ = (int)f.data_.rows();
    cols_ = (int)f.data_.cols();
    feat_.resize((size_t)dim_ * cols_);
    for (int j = 0; j < cols_; ++j)
        for (int r = 0; r < dim_; ++r) feat_[(size_t)j * dim_ + r] = f.data_(r, j);
}
}  // namespace geometry
namespace pipelines {
namespace registration {
// As in ref_shim_ransac: TransformationEstimation.cpp needs far more of Eigen than the stub provides; Registration.cpp
// names these members, and FGR never calls them.
double TransformationEstimationPointToPoint::ComputeRMSE(const geometry::PointCloud&, const geometry::PointCloud&,
                                                         const CorrespondenceSet&) const {
    throw std::runtime_error("not in the shim");
}
Eigen::Matrix4d TransformationEstimationPointToPoint::ComputeTransformation(const geometry::PointCloud&,
                                                                            const geometry::PointCloud&,
                                                                            const CorrespondenceSet&) const {
    throw std::runtime_error("not in the shim");
}
std::tuple<std::shared_ptr<const geometry::PointCloud>, std::shared_ptr<const geometry::PointCloud>>
TransformationEstimationPointToPoint::InitializePointCloudsForTransformation(const geometry::PointCloud&,
                                                                            const geometry::PointCloud&,
                                                                            double) const {
    throw std::runtime_error("not in the shim");
}
CorrespondenceSet CorrespondencesFromFeatures(const Feature&, const Feature&, bool, float) {
    throw std::runtime_error("not in the shim");
}
}  // namespace registration
}  // namespace pipelines
}  // namespace open3d

namespace {
std::string g_error;
open3d::geometry::PointCloud cloud(const float* p, int64_t n) {
    open3d::geometry::PointCloud pc;
    pc.points_.resize((size_t)n);
    for (int64_t i = 0; i < n; ++i) pc.points_[i] = Eigen::Vector3d(p[3 * i], p[3 * i + 1], p[3 * i + 2]);
    return pc;
}
open3d::pipelines::registration::Feature feature(const float* f, int64_t n, int dim) {
    open3d::pipelines::registration::Feature out;
    out.data_.resize(dim, n);
    for (int64_t i = 0; i < n; ++i)
        for (int r = 0; r < dim; ++r) out.data_(r, i) = f[i * dim + r];
    return out;
}
struct Option {
    double division_factor;
    int use_absolute_scale, decrease_mu;
    double maximum_correspondence_distance;
    int iteration_number;
    double tuple_scale;
    int maximum_tuple_count, tuple_test;
};
}  // namespace

extern "C" {

const char* ref_fgr_last_error() { return g_error.c_str(); }

void ref_fgr_seed(int seed) { open3d::utility::random::Seed(seed); }

// The stub's stated operations on their own, through its Eigen types: x = A.ldlt().solve(b) for A [6][6] row-major;
// out = M.inverse() for M [4][4] row-major; TransformVector6dToMatrix4d(x) row-major; the stated sin / cos of x.
void ref_fgr_ldlt_solve6(const double* A, const double* b, double* x) {
    Eigen::MatrixXd M(6, 6);
    Eigen::VectorXd v(6);
    for (int r = 0; r < 6; ++r) {
        v(r) = b[r];
        for (int c = 0; c < 6; ++c) M(r, c) = A[6 * r + c];
    }
    const Eigen::VectorXd y = M.ldlt().solve(v);
    for (int r = 0; r < 6; ++r) x[r] = y(r);
}
void ref_fgr_inverse4(const double* A, double* out) {
    Eigen::Matrix4d M;
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) M(r, c) = A[4 * r + c];
    const Eigen::Matrix4d I = M.inverse();
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) out[4 * r + c] = I(r, c);
}
void ref_fgr_vec6_to_mat4(const double* x, double* out) {
    Eigen::Vector6d v;
    for (int k = 0; k < 6; ++k) v(k) = x[k];
    const Eigen::Matrix4d D = open3d::utility::TransformVector6dToMatrix4d(v);
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) out[4 * r + c] = D(r, c);
}
double ref_fgr_sincos(double x, int want_cos) { return Eigen::stated::sincos(x, want_cos); }

int ref_fgr_uniform_ints(int low, int high, int64_t count, int* out) {
    try {
        open3d::utility::random::UniformIntGenerator<int> gen(low, high);
        for (int64_t k = 0; k < count; ++k) out[k] = gen();
        return 0;
    } catch (const std::exception& e) {
        g_error = e.what();
        return -1;
    }
}

// The reference's FastGlobalRegistrationBasedOnCorrespondence (corres non-null) or ...BasedOnFeatureMatching
// (features [n][dim], [m][dim]) on f32 clouds converted to f64 as ToLegacy does.  T receives the transformation
// row-major, pairs [n][2] the correspondence set, fr {fitness, rmse}, stats {cross, tuples, trials consumed, warnings,
// -1}: cross and tuples from upstream's debug lines (-1 where it printed none), trials from its "actual" count.
// Returns 0, or -1 when the reference raised.
int ref_fgr(const float* src, int64_t n, const float* tgt, int64_t m, const int64_t* corres, int64_t K,
            const float* src_feat, const float* tgt_feat, int dim, const Option* o, double* T, int64_t* pairs,
            int64_t* num_pairs, double* fr, int64_t* stats) {
    using namespace open3d::pipelines::registration;
    try {
        const auto s = cloud(src, n), t = cloud(tgt, m);
        const FastGlobalRegistrationOption opt(o->division_factor, o->use_absolute_scale != 0, o->decrease_mu != 0,
                                               o->maximum_correspondence_distance, o->iteration_number,
                                               o->tuple_scale, o->maximum_tuple_count, o->tuple_test != 0);
        open3d::utility::ransac_log() = {};
        RegistrationResult r;
        if (corres) {
            CorrespondenceSet cs((size_t)K);
            for (int64_t k = 0; k < K; ++k) cs[k] = Eigen::Vector2i((int)corres[2 * k], (int)corres[2 * k + 1]);
            r = FastGlobalRegistrationBasedOnCorrespondence(s, t, cs, opt);
        } else {
            r = FastGlobalRegistrationBasedOnFeatureMatching(s, t, feature(src_feat, n, dim),
                                                             feature(tgt_feat, m, dim), opt);
        }
        for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 4; ++j) T[4 * i + j] = r.transformation_(i, j);
        for (size_t k = 0; k < r.correspondence_set_.size(); ++k) {
            pairs[2 * k] = r.correspondence_set_[k](0);
            pairs[2 * k + 1] = r.correspondence_set_[k](1);
        }
        *num_pairs = (int64_t)r.correspondence_set_.size();
        fr[0] = r.fitness_;
        fr[1] = r.inlier_rmse_;
        const auto& L = open3d::utility::ransac_log();
        // upstream's i: the index of the breaking trial, or number_of_trial when the loop ran out
        const long long trials = L.tuples < 0 ? 0 : (L.actual < L.trials ? L.actual + 1 : L.trials);
        stats[0] = L.cross;
        stats[1] = L.tuples;
        stats[2] = trials;
        stats[3] = L.warnings;
        stats[4] = -1;
        return 0;
    } catch (const std::exception& e) {
        g_error = e.what();
        return -1;
    }
}

}  // extern "C"
