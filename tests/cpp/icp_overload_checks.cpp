// Argument checks of the five registration::ICP overloads (include/open3d_b200.hpp): each rejects bad input on the
// host with its own exact message, in its order (empty clouds first, the estimator's own attributes, then the
// correspondence distance and the voxel size); without a device, valid calls fail loudly.  Exit code 0 = pass.
#include <cuda_runtime.h>

#include <array>
#include <cstdio>
#include <cstring>

#include "open3d_b200.hpp"

namespace reg = open3d_b200::t::pipelines::registration;
namespace geo = open3d_b200::t::geometry;

#define EXPECT(c)                                                      \
    do {                                                               \
        if (!(c)) {                                                    \
            std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); \
            return 1;                                                  \
        }                                                              \
    } while (0)

template <class F>
static bool throws_exactly(F&& f, const char* message) {
    try {
        f();
    } catch (const std::runtime_error& e) {
        return std::strcmp(e.what(), message) == 0;
    }
    return false;
}

template <class F>
static bool throws_with(F&& f, const char* needle) {
    try {
        f();
    } catch (const std::runtime_error& e) {
        return std::strstr(e.what(), needle) != nullptr;
    }
    return false;
}

static const char* kEmpty = "Source and/or Target pointcloud is empty.";
static const char* kDistance0 = " Max correspondence distance must be greater than 0, but got 0.000000 in scale: 0.";
static const char* kVoxel = "voxel_size > 0: apply PointCloud::VoxelDownSample first (o3db_voxel_down_sample)";

int main() {
    float dummy[3] = {0, 0, 0};
    const std::array<double, 16> eye{{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}};
    geo::PointCloud empty, src{dummy, nullptr, 1}, tgt_no_normals{dummy, nullptr, 1}, tgt{dummy, dummy, 1};

    reg::TransformationEstimationPointToPlane plane;
    EXPECT(throws_exactly([&] { reg::ICP(empty, tgt_no_normals, 0.0, eye, plane); }, kEmpty));
    EXPECT(throws_exactly([&] { reg::ICP(src, tgt_no_normals, 0.0, eye, plane); },
                          "TransformationEstimationPointToPlane require pre-computed normal vectors for target PointCloud."));
    EXPECT(throws_exactly([&] { reg::ICP(src, tgt, 0.0, eye, plane, {}, 0.02); }, kDistance0));
    EXPECT(throws_exactly([&] { reg::ICP(src, tgt, 0.1, eye, plane, {}, 0.02); },
                          "voxel_size > 0: apply PointCloud::VoxelDownSample first (o3db_voxel_down_sample); this "
                          "header-only wrapper owns no device memory for the pyramid"));

    reg::TransformationEstimationForColoredICP colored;
    geo::PointCloud csrc{dummy, nullptr, 1, dummy}, ctgt{dummy, dummy, 1, dummy},
            cgtgt{dummy, dummy, 1, dummy, nullptr, nullptr, dummy};
    EXPECT(throws_exactly([&] { reg::ICP(empty, tgt_no_normals, 0.0, eye, colored); }, kEmpty));
    EXPECT(throws_exactly([&] { reg::ICP(csrc, tgt_no_normals, 0.0, eye, colored); },
                          "ColoredICP requires target pointcloud to have normals."));
    EXPECT(throws_exactly([&] { reg::ICP(src, tgt, 0.0, eye, colored); },
                          "ColoredICP requires target pointcloud to have colors."));
    EXPECT(throws_exactly([&] { reg::ICP(src, ctgt, 0.0, eye, colored); },
                          "ColoredICP requires source pointcloud to have colors."));
    EXPECT(throws_exactly([&] { reg::ICP(csrc, ctgt, 0.0, eye, colored); },
                          "Target pointcloud missing color_gradients attribute."));
    EXPECT(throws_exactly([&] { reg::ICP(csrc, cgtgt, 0.0, eye, colored, {}, 0.02); }, kDistance0));
    EXPECT(throws_exactly([&] { reg::ICP(csrc, cgtgt, 0.1, eye, colored, {}, 0.02); },
                          "voxel_size > 0: apply PointCloud::VoxelDownSample first (o3db_voxel_down_sample_attrs)"));

    reg::TransformationEstimationPointToPoint p2p;
    EXPECT(throws_exactly([&] { reg::ICP(empty, src, 0.0, eye, p2p); }, kEmpty));
    EXPECT(throws_exactly([&] { reg::ICP(src, empty, 0.0, eye, p2p); }, kEmpty));
    EXPECT(throws_exactly([&] { reg::ICP(src, src, 0.0, eye, p2p, {}, 0.02); }, kDistance0));
    EXPECT(throws_exactly([&] { reg::ICP(src, src, 0.1, eye, p2p, {}, 0.02); }, kVoxel));

    reg::TransformationEstimationSymmetric sym;
    const char* kSymNormals = "SymmetricICP requires both source and target pointclouds to have normals.";
    geo::PointCloud nsrc{dummy, dummy, 1};
    EXPECT(throws_exactly([&] { reg::ICP(empty, tgt_no_normals, 0.0, eye, sym); }, kEmpty));
    EXPECT(throws_exactly([&] { reg::ICP(src, tgt, 0.0, eye, sym); }, kSymNormals));
    EXPECT(throws_exactly([&] { reg::ICP(nsrc, tgt_no_normals, 0.0, eye, sym); }, kSymNormals));
    EXPECT(throws_exactly([&] { reg::ICP(nsrc, tgt, 0.0, eye, sym, {}, 0.02); }, kDistance0));
    EXPECT(throws_exactly([&] { reg::ICP(nsrc, tgt, 0.1, eye, sym, {}, 0.02); }, kVoxel));

    reg::TransformationEstimationForDopplerICP dop;
    geo::PointCloud dsrc{dummy, nullptr, 1, nullptr, dummy, dummy}, no_dopplers{dummy, nullptr, 1, nullptr, nullptr, dummy},
            no_directions{dummy, nullptr, 1, nullptr, dummy, nullptr};
    EXPECT(throws_exactly([&] { reg::ICP(empty, tgt_no_normals, 0.0, eye, dop); }, kEmpty));
    EXPECT(throws_exactly([&] { reg::ICP(no_dopplers, tgt_no_normals, 0.0, eye, dop); },
                          "DopplerICP requires target pointcloud to have normals."));
    EXPECT(throws_exactly([&] { reg::ICP(no_dopplers, tgt, 0.0, eye, dop); },
                          "DopplerICP requires source pointcloud to have Doppler velocities."));
    EXPECT(throws_exactly([&] { reg::ICP(no_directions, tgt, 0.0, eye, dop); },
                          "DopplerICP requires source pointcloud to have pre-computed direction vectors."));
    EXPECT(throws_exactly([&] { reg::ICP(dsrc, tgt, 0.0, eye, dop, {}, 0.02); }, kDistance0));
    EXPECT(throws_exactly([&] { reg::ICP(dsrc, tgt, 0.1, eye, dop, {}, 0.02); }, kVoxel));

    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {   // no CPU fallback: valid calls must fail loudly
        EXPECT(throws_with([&] { reg::ICP(src, tgt, 0.1, eye, plane); }, "CUDA"));
        EXPECT(throws_with([&] { reg::ICP(src, src, 0.1, eye, p2p); }, "CUDA"));
        EXPECT(throws_with([&] { reg::ICP(nsrc, tgt, 0.1, eye, sym); }, "CUDA"));
        EXPECT(throws_with([&] { reg::ICP(dsrc, tgt, 0.1, eye, dop); }, "CUDA"));
    }
    std::printf("icp overload checks ok\n");
    return 0;
}
