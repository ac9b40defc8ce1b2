// ref_shim_extract.cpp — TEST INFRASTRUCTURE.  Compiles the reference's own t/geometry/kernel/VoxelBlockGridCPU.cpp
// unmodified (it explicitly instantiates ExtractPointCloudCPU<float, uint16_t, uint16_t>), from where the file lies in
// the reference tree, against the stub core::Tensor / HashMap / TBB headers of ../ref_shim/stubs, and exports the
// point-cloud extraction through a C function so that the CPU oracle (oracle/extract/extract_oracle.c) can be checked
// against the real thing.  A library of its own (oracle/_ref/libo3dref_extract.so): the same translation unit is in
// libo3dref.so, and one library cannot hold it twice.  No reference source is copied into this repository.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <unordered_map>

using std::abs;
using std::max;
using std::min;

#include "open3d/t/geometry/kernel/VoxelBlockGridCPU.cpp"   // from -I <reference>/cpp

namespace o3c = open3d::core;
namespace o3v = open3d::t::geometry::kernel::voxel_grid;
using open3d::t::geometry::TensorMap;

namespace {
using Key = open3d::utility::MiniVec<int, 3>;
using Hash = open3d::utility::MiniVecHash<int, 3>;
using Eq = open3d::utility::MiniVecEq<int, 3>;
}  // namespace

extern "C" {

// ExtractPointCloudCPU<float, uint16_t, uint16_t> (VoxelBlockGridImpl.h:1122-1381) over every block of the map, with
// the 27-block neighbour tables BufferRadiusNeighbors (VoxelBlockGrid.cpp:22-51) builds, laid out [27][n] as its
// HashMap::Find returns them, and valid_size = -1 (the counting pass).  Rows come in upstream's atomic-counter order;
// the first min(total, max_points) are copied out and the total is returned.
int64_t ref_extract_point_cloud(const int32_t* table_keys, int64_t size, const float* tsdf, const uint16_t* weight,
                                const uint16_t* color_buf, int resolution, float voxel_size, float weight_threshold,
                                int64_t max_points, float* points_out, float* normals_out, float* colors_out) {
    const int64_t r3 = (int64_t)resolution * resolution * resolution;
    std::unordered_map<Key, int32_t, Hash, Eq> slot_of;
    for (int64_t s = 0; s < size; ++s)
        slot_of[Key(table_keys[3 * s], table_keys[3 * s + 1], table_keys[3 * s + 2])] = (int32_t)s;
    o3c::Tensor indices({size}, o3c::Int32), nb_indices({27, size, 1}, o3c::Int32), nb_masks({27, size, 1}, o3c::Bool);
    for (int64_t s = 0; s < size; ++s) {
        indices.GetDataPtr<int32_t>()[s] = (int32_t)s;
        for (int nb = 0; nb < 27; ++nb) {
            const int* k = table_keys + 3 * s;
            auto it = slot_of.find(Key(k[0] + nb % 3 - 1, k[1] + (nb % 9) / 3 - 1, k[2] + nb / 9 - 1));
            nb_indices.GetDataPtr<int32_t>()[nb * size + s] = it == slot_of.end() ? 0 : it->second;
            nb_masks.GetDataPtr<bool>()[nb * size + s] = it != slot_of.end();
        }
    }
    o3c::Tensor keys((void*)table_keys, {size, 3}, o3c::Int32);
    TensorMap vm("tsdf");
    vm["tsdf"] = o3c::Tensor((void*)tsdf, {size * r3, 1}, o3c::Float32);
    vm["weight"] = o3c::Tensor((void*)weight, {size * r3, 1}, o3c::UInt16);
    if (color_buf) vm["color"] = o3c::Tensor((void*)color_buf, {size * r3, 3}, o3c::UInt16);
    o3c::Tensor points, normals, colors;
    int valid_size = -1;
    o3v::ExtractPointCloudCPU<float, uint16_t, uint16_t>(indices, nb_indices, nb_masks, keys, vm, points, normals,
                                                         colors, resolution, voxel_size, weight_threshold, valid_size);
    const size_t n = (size_t)std::min<int64_t>(valid_size, max_points);
    if (n > 0) {
        memcpy(points_out, points.GetDataPtr<float>(), n * 3 * sizeof(float));
        memcpy(normals_out, normals.GetDataPtr<float>(), n * 3 * sizeof(float));
        if (color_buf && colors_out) memcpy(colors_out, colors.GetDataPtr<float>(), n * 3 * sizeof(float));
    }
    return valid_size;
}

}  // extern "C"
