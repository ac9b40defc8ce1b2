// ref_shim_mesh.cpp — TEST INFRASTRUCTURE.  Compiles the reference's own t/geometry/kernel/VoxelBlockGridCPU.cpp
// unmodified (it explicitly instantiates ExtractTriangleMeshCPU<float, uint16_t, uint16_t>) against the stub headers
// of ../ref_shim/stubs, and exports the triangle-mesh extraction and one row of the marching-cubes tables it was
// compiled with, so that the CPU oracle (oracle/mesh/mesh_oracle.c) and its case table can be checked against the
// real thing.  A library of its own (oracle/_ref/libo3dref_mesh.so), like ../ref_shim_extract, because one library
// cannot hold the translation unit twice.  No reference source is copied into this repository.
#include <omp.h>

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

// ExtractTriangleMeshCPU<float, uint16_t, uint16_t> (VoxelBlockGridImpl.h:1385-1780) over every block of the map, as
// VoxelBlockGrid::ExtractTriangleMesh (VoxelBlockGrid.cpp:436-472) calls it: active indices 0..size-1, the identity
// inverse map, the 27-block neighbour tables of BufferRadiusNeighbors laid out [27][n], estimated_vertex_number = -1.
// On `threads` OpenMP threads (<= 0: all); on one thread upstream's atomic counters give the sequential order (block,
// voxel, axis for vertices; block, voxel, table for triangles).  Copies the first min(count, max) rows of each array
// out; returns the vertex count and stores the triangle count in *num_triangles.
int64_t ref_extract_triangle_mesh(const int32_t* table_keys, int64_t size, const float* tsdf, const uint16_t* weight,
                                  const uint16_t* color_buf, int resolution, float voxel_size, float weight_threshold,
                                  int threads, int64_t max_vertices, int64_t max_triangles, float* vertices_out,
                                  float* normals_out, float* colors_out, int32_t* triangles_out,
                                  int64_t* num_triangles) {
    const int64_t r3 = (int64_t)resolution * resolution * resolution;
    std::unordered_map<Key, int32_t, Hash, Eq> slot_of;
    for (int64_t s = 0; s < size; ++s)
        slot_of[Key(table_keys[3 * s], table_keys[3 * s + 1], table_keys[3 * s + 2])] = (int32_t)s;
    o3c::Tensor indices({size}, o3c::Int32), inv_indices({size}, o3c::Int32);
    o3c::Tensor nb_indices({27, size, 1}, o3c::Int32), nb_masks({27, size, 1}, o3c::Bool);
    for (int64_t s = 0; s < size; ++s) {
        indices.GetDataPtr<int32_t>()[s] = (int32_t)s;
        inv_indices.GetDataPtr<int32_t>()[s] = (int32_t)s;
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
    o3c::Tensor vertices, triangles, normals, colors;
    int vertex_count = -1;
    const int saved = omp_get_max_threads();
    omp_set_num_threads(threads > 0 ? threads : omp_get_num_procs());
    o3v::ExtractTriangleMeshCPU<float, uint16_t, uint16_t>(indices, inv_indices, nb_indices, nb_masks, keys, vm,
                                                           vertices, triangles, normals, colors, resolution,
                                                           voxel_size, weight_threshold, vertex_count);
    omp_set_num_threads(saved);
    const int64_t nt = triangles.GetLength();
    *num_triangles = nt;
    const size_t nv = (size_t)std::min<int64_t>(vertex_count, max_vertices);
    if (nv > 0) {
        memcpy(vertices_out, vertices.GetDataPtr<float>(), nv * 3 * sizeof(float));
        memcpy(normals_out, normals.GetDataPtr<float>(), nv * 3 * sizeof(float));
        if (color_buf && colors_out) memcpy(colors_out, colors.GetDataPtr<float>(), nv * 3 * sizeof(float));
    }
    const size_t ntc = (size_t)std::min<int64_t>(nt, max_triangles);
    if (ntc > 0) memcpy(triangles_out, triangles.GetDataPtr<int32_t>(), ntc * 3 * sizeof(int32_t));
    return vertex_count;
}

// Row c of the compiled marching-cubes tables: tri_table[c][0..15] into row, edge_table[c], tri_count[c].
void ref_mc_table_row(int c, int32_t* row, int32_t* edge_mask, int32_t* triangle_count) {
    for (int i = 0; i < 16; ++i) row[i] = tri_table[c][i];
    *edge_mask = edge_table[c];
    *triangle_count = tri_count[c];
}

}  // extern "C"
