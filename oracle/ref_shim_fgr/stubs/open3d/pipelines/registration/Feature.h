// ref_shim_fgr stub (test infrastructure): the Feature type and the CorrespondencesFromFeatures declaration that
// RegistrationRANSACBasedOnFeatureMatching calls (defined in the shim so that the file links).
#pragma once
#include <Eigen/Core>
#include "open3d/pipelines/registration/TransformationEstimation.h"
namespace open3d {
namespace pipelines {
namespace registration {
class Feature {
public:
    Eigen::MatrixXd data_;
};
CorrespondenceSet CorrespondencesFromFeatures(const Feature& source_features, const Feature& target_features,
                                              bool mutual_filter = false, float mutual_consistency_ratio = 0.1);
}  // namespace registration
}  // namespace pipelines
}  // namespace open3d
