// integration/o3d_forwarders.cpp — the bodies a maintainer drops into Open3D's `*CUDA` translation units so that the
// reference's OWN dispatch layer (`if (x.IsCUDA()) CUDA_CALL(FooCUDA, ...)`, core/CUDAUtils.h) lands in libo3db200.so.
//
// Every function below is a DEFINITION of a function the reference DECLARES, compiled against the reference's own
// headers (this file includes them from the reference tree; a signature drift is a compile error):
//   t/pipelines/kernel/RegistrationImpl.h:93-102, 118-131   ComputePosePointToPlaneCUDA, ComputePoseColoredICPCUDA
//   t/geometry/kernel/Transform.h:42-47                      TransformPointsCUDA, TransformNormalsCUDA
//   t/geometry/kernel/VoxelBlockGrid.h:345-381               DepthTouchCUDA, IntegrateCUDA<...> (all 4 instantiations)
//   core/nns/FixedRadiusIndex.h:227, 364                     BuildSpatialHashTableCUDA<float>, HybridSearchCUDA<float,int32_t>
//
// Two build modes:
//   * inside Open3D (BUILD_CUDA_MODULE build): add this file to the CUDA module instead of the bodies it replaces;
//     core::Tensor etc. are the real classes, the stream is core::cuda::GetStream().
//   * stand-alone check (oracle/ref_shim/Makefile, -DO3DB_FORWARDERS_STANDALONE): the same source against the reference
//     headers with the ref-shim's stub core::Tensor (oracle/ref_shim/stubs — a non-owning pointer/shape/dtype view),
//     linked with libo3db200.so and exercised on the GPU by tests/test_forwarders_gpu.py through forwarder_hooks.cpp.
// Float64 point clouds are outside this library's scope (north_star: fp32): those calls raise, exactly like any other
// unsupported dtype in the reference (utility::LogError -> std::runtime_error -> Python RuntimeError).
#ifndef BUILD_CUDA_MODULE
#define BUILD_CUDA_MODULE
#endif

#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "open3d/core/Tensor.h"
#include "open3d/core/nns/FixedRadiusIndex.h"
#include "open3d/t/geometry/kernel/Transform.h"
#include "open3d/t/geometry/kernel/VoxelBlockGrid.h"
#include "open3d/t/pipelines/kernel/RegistrationImpl.h"
#include "open3d/utility/Logging.h"
#include "open3d_b200.h"

namespace {

inline void Check(int rc) {
    if (rc < 0) open3d::utility::LogError("{}", o3db_last_error());
}

inline void* Stream() {
#ifdef O3DB_FORWARDERS_STANDALONE
    return nullptr;   // the legacy default stream
#else
    return (void*)open3d::core::cuda::GetStream();   // core/CUDAUtils.h:149-172
#endif
}

inline void RequireFloat32(const open3d::core::Dtype& dtype, const char* what) {
    if (dtype != open3d::core::Float32)
        open3d::utility::LogError("{}: open3d_b200 implements the Float32 path only", what);
}

// n doubles out of a small Float32 / Float64 tensor that may live on the host or on the device (intrinsics,
// extrinsics, 4x4 transformations): cudaMemcpyDefault resolves either through unified addressing.
inline void HostF64(const open3d::core::Tensor& t, int n, double* out) {
    if (t.NumElements() != n) open3d::utility::LogError("open3d_b200 forwarder: expected {} elements", n);
    if (t.GetDtype() == open3d::core::Float64) {
        if (cudaMemcpy(out, t.GetDataPtr(), sizeof(double) * n, cudaMemcpyDefault) != cudaSuccess)
            open3d::utility::LogError("open3d_b200 forwarder: copy to host failed");
    } else if (t.GetDtype() == open3d::core::Float32) {
        float tmp[16];
        if (n > 16 || cudaMemcpy(tmp, t.GetDataPtr(), sizeof(float) * n, cudaMemcpyDefault) != cudaSuccess)
            open3d::utility::LogError("open3d_b200 forwarder: copy to host failed");
        for (int i = 0; i < n; ++i) out[i] = tmp[i];
    } else {
        open3d::utility::LogError("open3d_b200 forwarder: Float32 / Float64 tensor expected");
    }
}

// the {6} Float64 pose the reference returns on the host (DecodeAndSolve6x6, TransformationConverter.cpp:189-226)
inline open3d::core::Tensor PoseToHost(const double* pose_dev) {
    std::vector<double> h(6);
    if (cudaMemcpy(h.data(), pose_dev, 6 * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess)
        open3d::utility::LogError("open3d_b200 forwarder: pose read-back failed");
    return open3d::core::Tensor(h, {6}, open3d::core::Float64);
}

struct DeviceScratch {   // small device buffer for the lifetime of one forwarder call
    void* p = nullptr;
    explicit DeviceScratch(size_t bytes) {
        if (cudaMalloc(&p, bytes) != cudaSuccess) open3d::utility::LogError("open3d_b200 forwarder: cudaMalloc failed");
    }
    ~DeviceScratch() { cudaFree(p); }
};

inline o3db_robust_kernel Robust(const open3d::t::pipelines::registration::RobustKernel& k) {
    // RobustKernelMethod (registration/RobustKernel.h:15-23) and o3db_robust_method share their numbering
    return o3db_robust_kernel{(int)k.type_, k.scaling_parameter_, k.shape_parameter_};
}

}  // namespace

namespace open3d {
namespace t {
namespace pipelines {
namespace kernel {

// replaces RegistrationCUDA.cu:81-117
void ComputePosePointToPlaneCUDA(const core::Tensor& source_points,
                                 const core::Tensor& target_points,
                                 const core::Tensor& target_normals,
                                 const core::Tensor& correspondence_indices,
                                 core::Tensor& pose,
                                 float& residual,
                                 int& inlier_count,
                                 const core::Dtype& dtype,
                                 const core::Device& device,
                                 const registration::RobustKernel& kernel) {
    (void)device;
    RequireFloat32(dtype, "ComputePosePointToPlaneCUDA");
    const o3db_robust_kernel rk = Robust(kernel);
    DeviceScratch pose_dev(6 * sizeof(double));
    // the 29 sums stay on the device; the 6x6 f64 solve runs there too (singular -> the reference's message)
    Check(o3db_compute_pose_point_to_plane(source_points.GetDataPtr<float>(), target_points.GetDataPtr<float>(),
                                           target_normals.GetDataPtr<float>(),
                                           correspondence_indices.GetDataPtr<int64_t>(), source_points.GetLength(), &rk,
                                           nullptr, (double*)pose_dev.p, &residual, &inlier_count, Stream()));
    pose = PoseToHost((const double*)pose_dev.p);
}

// replaces RegistrationCUDA.cu:183-230
void ComputePoseColoredICPCUDA(const core::Tensor& source_points,
                               const core::Tensor& source_colors,
                               const core::Tensor& target_points,
                               const core::Tensor& target_normals,
                               const core::Tensor& target_colors,
                               const core::Tensor& target_color_gradients,
                               const core::Tensor& correspondence_indices,
                               core::Tensor& pose,
                               float& residual,
                               int& inlier_count,
                               const core::Dtype& dtype,
                               const core::Device& device,
                               const registration::RobustKernel& kernel,
                               const double& lambda_geometric) {
    (void)device;
    RequireFloat32(dtype, "ComputePoseColoredICPCUDA");
    const o3db_robust_kernel rk = Robust(kernel);
    DeviceScratch pose_dev(6 * sizeof(double));
    Check(o3db_compute_pose_colored_icp(source_points.GetDataPtr<float>(), source_colors.GetDataPtr<float>(),
                                        target_points.GetDataPtr<float>(), target_normals.GetDataPtr<float>(),
                                        target_colors.GetDataPtr<float>(), target_color_gradients.GetDataPtr<float>(),
                                        correspondence_indices.GetDataPtr<int64_t>(), source_points.GetLength(), &rk,
                                        lambda_geometric, nullptr, (double*)pose_dev.p, &residual, &inlier_count, Stream()));
    pose = PoseToHost((const double*)pose_dev.p);
}

}  // namespace kernel
}  // namespace pipelines

namespace geometry {
namespace kernel {
namespace transform {

// replaces TransformCUDA.cu (declared Transform.h:42-47); `transformation` is 4x4 in the points' dtype on their device
void TransformPointsCUDA(const core::Tensor& transformation, core::Tensor& points) {
    RequireFloat32(points.GetDtype(), "TransformPointsCUDA");
    double T[16];
    HostF64(transformation, 16, T);
    Check(o3db_transform_points(T, points.GetDataPtr<float>(), points.GetLength(), Stream()));
}

void TransformNormalsCUDA(const core::Tensor& transformation, core::Tensor& normals) {
    RequireFloat32(normals.GetDtype(), "TransformNormalsCUDA");
    double T[16];
    HostF64(transformation, 16, T);
    Check(o3db_transform_normals(T, normals.GetDataPtr<float>(), normals.GetLength(), Stream()));
}

}  // namespace transform

namespace voxel_grid {

// replaces VoxelBlockGridCUDA.cu:106-227.  The frustum hash map the reference passes in only de-duplicates inside
// the call (VoxelBlockGrid.cpp:233-236 clears it first); the library de-duplicates in its own scratch table.
void DepthTouchCUDA(std::shared_ptr<core::HashMap>& hashmap,
                    const core::Tensor& depth,
                    const core::Tensor& intrinsic,
                    const core::Tensor& extrinsic,
                    core::Tensor& voxel_block_coords,
                    index_t voxel_grid_resolution,
                    float voxel_size,
                    float sdf_trunc,
                    float depth_scale,
                    float depth_max,
                    index_t stride) {
    (void)hashmap;
    const int rows = (int)depth.GetShape(0), cols = (int)depth.GetShape(1);
    const int dtype = depth.GetDtype() == core::UInt16 ? O3DB_DEPTH_U16 : O3DB_DEPTH_F32;
    if (depth.GetDtype() != core::UInt16 && depth.GetDtype() != core::Float32)
        utility::LogError("Unsupported depth image dtype {}", depth.GetDtype().ToString());
    double K[9], E[16];
    HostF64(intrinsic, 9, K);
    HostF64(extrinsic, 16, E);
    // VoxelBlockGridCUDA.cu:129-132: capacity of the per-frame candidate set
    const int64_t cap = (int64_t)(rows / stride) * (cols / stride) * 4;
    core::Tensor out({cap, 3}, core::Int32, depth.GetDevice());
    int64_t n = 0;
    Check(o3db_depth_touch(depth.GetDataPtr(), dtype, rows, cols, K, E, voxel_grid_resolution, voxel_size, sdf_trunc,
                           depth_scale, depth_max, stride, out.GetDataPtr<int32_t>(), cap, &n, Stream()));
    voxel_block_coords = out.Slice(0, 0, n);
}

namespace {
template <typename T>
struct ColorDtypeOf;
template <>
struct ColorDtypeOf<uint8_t> { static constexpr int value = O3DB_COLOR_U8; };
template <>
struct ColorDtypeOf<float> { static constexpr int value = O3DB_COLOR_F32; };
}  // namespace

// replaces VoxelBlockGridImpl.h:151-308 as instantiated by VoxelBlockGridCUDA.cu:238-244: block_indices, block_keys and
// the value tensors are the reference hash map's own buffers.
template <typename input_depth_t, typename input_color_t, typename tsdf_t, typename weight_t, typename color_t>
void IntegrateCUDA(const core::Tensor& depth,
                   const core::Tensor& color,
                   const core::Tensor& block_indices,
                   const core::Tensor& block_keys,
                   TensorMap& block_value_map,
                   const core::Tensor& depth_intrinsic,
                   const core::Tensor& color_intrinsic,
                   const core::Tensor& extrinsic,
                   index_t resolution,
                   float voxel_size,
                   float sdf_trunc,
                   float depth_scale,
                   float depth_max) {
    static_assert(sizeof(tsdf_t) == 4, "tsdf is Float32 in every reference instantiation");
    if (!block_value_map.Contains("tsdf") || !block_value_map.Contains("weight"))
        utility::LogError("TSDF and/or weight not allocated in blocks, please implement customized integration.");
    const bool integrate_color = block_value_map.Contains("color") && color.NumElements() > 0;   // VoxelBlockGridImpl.h:202-203
    const int rows = (int)depth.GetShape(0), cols = (int)depth.GetShape(1);
    double dK[9], cK[9], E[16];
    HostF64(depth_intrinsic, 9, dK);
    HostF64(color_intrinsic, 9, cK);
    HostF64(extrinsic, 16, E);
    Check(o3db_integrate_blocks(depth.GetDataPtr(), sizeof(input_depth_t) == 2 ? O3DB_DEPTH_U16 : O3DB_DEPTH_F32,
                                integrate_color ? color.GetDataPtr() : nullptr, ColorDtypeOf<input_color_t>::value, rows, cols,
                                block_indices.GetDataPtr<int32_t>(), block_indices.GetLength(),
                                block_keys.GetDataPtr<int32_t>(), block_value_map.at("tsdf").GetDataPtr<float>(),
                                block_value_map.at("weight").GetDataPtr(),
                                integrate_color ? block_value_map.at("color").GetDataPtr() : nullptr,
                                sizeof(weight_t) == 2 ? O3DB_VALUES_U16 : O3DB_VALUES_F32, dK, cK, E, resolution, voxel_size,
                                sdf_trunc, depth_scale, depth_max, Stream()));
}

#define O3DB_FN_ARGUMENTS                                                                                             \
    const core::Tensor &depth, const core::Tensor &color, const core::Tensor &indices, const core::Tensor &block_keys, \
            TensorMap &block_values, const core::Tensor &depth_intrinsic, const core::Tensor &color_intrinsic,        \
            const core::Tensor &extrinsic, index_t resolution, float voxel_size, float sdf_trunc, float depth_scale,  \
            float depth_max
template void IntegrateCUDA<uint16_t, uint8_t, float, uint16_t, uint16_t>(O3DB_FN_ARGUMENTS);
template void IntegrateCUDA<uint16_t, uint8_t, float, float, float>(O3DB_FN_ARGUMENTS);
template void IntegrateCUDA<float, float, float, uint16_t, uint16_t>(O3DB_FN_ARGUMENTS);
template void IntegrateCUDA<float, float, float, float, float>(O3DB_FN_ARGUMENTS);
#undef O3DB_FN_ARGUMENTS

}  // namespace voxel_grid
}  // namespace kernel
}  // namespace geometry
}  // namespace t

namespace core {
namespace nns {

// replaces FixedRadiusSearchOps.cu:20-58: the reference-layout tables (SpatialHash(floor(p / 2r)) % H, exclusive splits).
// Single batch item, as every caller on the ICP path uses it (FixedRadiusIndex.cpp:58-136).
template <class T>
void BuildSpatialHashTableCUDA(const Tensor& points,
                               double radius,
                               const Tensor& points_row_splits,
                               const Tensor& hash_table_splits,
                               Tensor& hash_table_index,
                               Tensor& hash_table_cell_splits) {
    static_assert(sizeof(T) == 4, "Float32 point clouds only");
    if (points_row_splits.GetLength() != 2 || hash_table_splits.GetLength() != 2)
        utility::LogError("open3d_b200: BuildSpatialHashTableCUDA supports one batch item");
    Check(o3db_build_spatial_hash_table(points.GetDataPtr<float>(), points.GetLength(), radius,
                                        (uint32_t)(hash_table_cell_splits.GetLength() - 1),
                                        hash_table_index.GetDataPtr<uint32_t>(), hash_table_cell_splits.GetDataPtr<uint32_t>(),
                                        Stream()));
}
template void BuildSpatialHashTableCUDA<float>(const Tensor&, double, const Tensor&, const Tensor&, Tensor&, Tensor&);

// replaces FixedRadiusSearchOps.cu:134-196.  The library searches its own index (a dense cell-sorted grid, DESIGN.md
// §3) built from `points` for this call; the reference-layout tables passed in are not read.  (The zero-rebuild cut is
// one level up, in FixedRadiusIndex::SetTensorData / SearchHybrid — INTEGRATION.md §2.)  Outputs have the reference's
// shapes: index / distance [num_queries, max_knn] (-1 / 0 padded), count [num_queries].
template <class T, class TIndex>
void HybridSearchCUDA(const Tensor& points,
                      const Tensor& queries,
                      double radius,
                      int max_knn,
                      const Tensor& points_row_splits,
                      const Tensor& queries_row_splits,
                      const Tensor& hash_table_splits,
                      const Tensor& hash_table_index,
                      const Tensor& hash_table_cell_splits,
                      const Metric metric,
                      Tensor& neighbors_index,
                      Tensor& neighbors_count,
                      Tensor& neighbors_distance) {
    static_assert(sizeof(T) == 4 && sizeof(TIndex) == 4, "Float32 points, Int32 indices");
    (void)hash_table_splits;
    (void)hash_table_index;
    (void)hash_table_cell_splits;
    if (metric != L2) utility::LogError("open3d_b200: HybridSearchCUDA implements the L2 metric");
    if (points_row_splits.GetLength() != 2 || queries_row_splits.GetLength() != 2)
        utility::LogError("open3d_b200: HybridSearchCUDA supports one batch item");
    const int64_t nq = queries.GetLength();
    neighbors_index = Tensor::Empty({nq, (int64_t)max_knn}, Int32, points.GetDevice());
    neighbors_distance = Tensor::Empty({nq, (int64_t)max_knn}, Float32, points.GetDevice());
    neighbors_count = Tensor::Empty({nq}, Int32, points.GetDevice());
    o3db_nns* index = nullptr;
    Check(o3db_nns_create(points.GetDataPtr<float>(), points.GetLength(), radius, Stream(), &index));
    const int rc = o3db_nns_hybrid_search(index, queries.GetDataPtr<float>(), nq, radius, max_knn,
                                          neighbors_index.GetDataPtr<int32_t>(), neighbors_distance.GetDataPtr<float>(),
                                          neighbors_count.GetDataPtr<int32_t>(), Stream());
    cudaStreamSynchronize((cudaStream_t)Stream());
    o3db_nns_destroy(index);
    Check(rc);
}
template void HybridSearchCUDA<float, int32_t>(const Tensor&, const Tensor&, double, int, const Tensor&, const Tensor&,
                                               const Tensor&, const Tensor&, const Tensor&, const Metric, Tensor&, Tensor&,
                                               Tensor&);

}  // namespace nns
}  // namespace core
}  // namespace open3d
