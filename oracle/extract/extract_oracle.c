/*
 * extract_oracle.c — CPU restatement of Open3D's VoxelBlockGrid::ExtractPointCloud
 * (t/geometry/VoxelBlockGrid.cpp:404-434 -> kernel::voxel_grid::ExtractPointCloud,
 * t/geometry/kernel/VoxelBlockGridImpl.h:1122-1381) for the slam::Model value layout
 * (tsdf f32, weight u16, colour u16 x 3).
 *
 * TEST INFRASTRUCTURE ONLY, like the rest of oracle/: the checker of the CUDA extraction
 * (tests/test_extract_gpu.py), itself pinned bit for bit, as a set of rows, against the
 * reference's own ExtractPointCloudCPU<float, uint16_t, uint16_t> compiled from the reference
 * (oracle/ref_shim_extract; tests/test_oracle_vs_ref_extract.py).
 * Compile with -ffp-contract=off: every f32 expression is evaluated operation by operation
 * in the reference's source order.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

/* Slot lookup of int32x3 block keys: chained hash over slots 0..size-1 (any hash will do). */
typedef struct {
    const int32_t* keys;
    int64_t* head;
    int64_t* next;
    int64_t nb;
} block_lookup;

static inline uint64_t key_hash(int32_t x, int32_t y, int32_t z) {
    uint64_t h = 14695981039346656037ull;
    h = (h ^ (uint64_t)(int64_t)x) * 1099511628211ull;
    h = (h ^ (uint64_t)(int64_t)y) * 1099511628211ull;
    h = (h ^ (uint64_t)(int64_t)z) * 1099511628211ull;
    return h;
}

static int lookup_build(block_lookup* m, const int32_t* keys, int64_t size) {
    m->keys = keys;
    m->nb = 16;
    while (m->nb < 2 * size) m->nb <<= 1;
    m->head = (int64_t*)malloc((size_t)m->nb * sizeof(int64_t));
    m->next = (int64_t*)malloc((size_t)(size > 0 ? size : 1) * sizeof(int64_t));
    if (!m->head || !m->next) return -1;
    for (int64_t i = 0; i < m->nb; ++i) m->head[i] = -1;
    for (int64_t s = 0; s < size; ++s) {
        const int32_t* k = keys + 3 * s;
        const uint64_t h = key_hash(k[0], k[1], k[2]) & (uint64_t)(m->nb - 1);
        m->next[s] = m->head[h];
        m->head[h] = s;
    }
    return 0;
}

static inline int64_t lookup_find(const block_lookup* m, int x, int y, int z) {
    const uint64_t h = key_hash(x, y, z) & (uint64_t)(m->nb - 1);
    for (int64_t s = m->head[h]; s >= 0; s = m->next[s]) {
        const int32_t* k = m->keys + 3 * s;
        if (k[0] == x && k[1] == y && k[2] == z) return s;
    }
    return -1;
}

static inline int isign(int x) { return (x > 0) ? 1 : ((x < 0) ? -1 : 0); } /* GeometryMacros.h:92-94 */


/* t/geometry/kernel/VoxelBlockGridImpl.h:94-121 DeviceGetLinearIdx, with the 27-block neighbourhood of
 * BufferRadiusNeighbors (t/geometry/VoxelBlockGrid.cpp:22-51) as `nb` (slot or -1, index (dx+1)+(dy+1)*3+(dz+1)*9).
 * Coordinates are in [-1, R+1]; with R == 1 a coordinate two blocks away maps into the adjacent block, as upstream. */
static inline int64_t ext_linear_idx(const int64_t nb[27], int xo, int yo, int zo, int R) {
    const int xn = (xo + R) % R, yn = (yo + R) % R, zn = (zo + R) % R;
    const int64_t blk = nb[(isign(xo - xn) + 1) + (isign(yo - yn) + 1) * 3 + (isign(zo - zn) + 1) * 9];
    if (blk < 0) return -1;
    return ((blk * R + zn) * R + yn) * R + xn;
}

/* :123-149 DeviceGetNormal: a component is written only when both of its neighbours exist. */
static inline void ext_normal(const float* tsdf, const int64_t nb[27], int xo, int yo, int zo, int R, float n[3]) {
    const int64_t vxp = ext_linear_idx(nb, xo + 1, yo, zo, R), vxn = ext_linear_idx(nb, xo - 1, yo, zo, R);
    const int64_t vyp = ext_linear_idx(nb, xo, yo + 1, zo, R), vyn = ext_linear_idx(nb, xo, yo - 1, zo, R);
    const int64_t vzp = ext_linear_idx(nb, xo, yo, zo + 1, R), vzn = ext_linear_idx(nb, xo, yo, zo - 1, R);
    if (vxp >= 0 && vxn >= 0) n[0] = tsdf[vxp] - tsdf[vxn];
    if (vyp >= 0 && vyn >= 0) n[1] = tsdf[vyp] - tsdf[vyn];
    if (vzp >= 0 && vzn >= 0) n[2] = tsdf[vzp] - tsdf[vzn];
}

/* t/geometry/kernel/VoxelBlockGridImpl.h:1122-1381 ExtractPointCloudCPU<float, uint16_t, uint16_t> for every block
 * of the map (VoxelBlockGrid::ExtractPointCloud, VoxelBlockGrid.cpp:404-434), in a deterministic order: ascending
 * slot, then the linear voxel index (z*R + y)*R + x, then axis 0, 1, 2.  Upstream's order comes from an atomic
 * counter; the set of rows is the same (tests/test_oracle_vs_ref_extract.py).  The first min(total, max_points) rows
 * are written; the return value is the total. */
int64_t orc_extract_point_cloud(const int32_t* table_keys, int64_t size, const float* tsdf,
                                const uint16_t* weight, const uint16_t* color, int resolution,
                                float voxel_size, float weight_threshold, int64_t max_points,
                                float* points, float* normals, float* colors) {
    block_lookup map;
    if (lookup_build(&map, table_keys, size) != 0) abort();
    const int R = resolution;
    const int64_t R3 = (int64_t)R * R * R;
    int64_t count = 0;
    for (int64_t b = 0; b < size; ++b) {
        int64_t nb[27];
        const int32_t* key = table_keys + 3 * b;
        for (int k = 0; k < 27; ++k)
            nb[k] = lookup_find(&map, key[0] + k % 3 - 1, key[1] + (k % 9) / 3 - 1, key[2] + k / 9 - 1);
        for (int64_t v = 0; v < R3; ++v) {
            const int xv = (int)(v % R), yv = (int)((v / R) % R), zv = (int)(v / ((int64_t)R * R));
            const int64_t lin = b * R3 + v;
            const float tsdf_o = tsdf[lin];
            const float weight_o = weight[lin];
            if (weight_o <= weight_threshold) continue;
            float no[3] = {0, 0, 0}, ne[3] = {0, 0, 0};   /* ne is NOT reset between the axes (:1283) */
            int have_no = 0;
            const int x = key[0] * R + xv, y = key[1] * R + yv, z = key[2] * R + zv;
            for (int i = 0; i < 3; ++i) {
                const int64_t lin_i = ext_linear_idx(nb, xv + (i == 0), yv + (i == 1), zv + (i == 2), R);
                if (lin_i < 0) continue;
                const float tsdf_i = tsdf[lin_i];
                const float weight_i = weight[lin_i];
                if (!(weight_i > weight_threshold && tsdf_i * tsdf_o < 0)) continue;
                const int64_t idx = count++;
                if (idx >= max_points) continue;
                if (!have_no) {
                    ext_normal(tsdf, nb, xv, yv, zv, R, no);
                    have_no = 1;
                }
                const float ratio = (0 - tsdf_o) / (tsdf_i - tsdf_o);
                float* p = points + 3 * idx;
                p[0] = voxel_size * (x + ratio * (int)(i == 0));
                p[1] = voxel_size * (y + ratio * (int)(i == 1));
                p[2] = voxel_size * (z + ratio * (int)(i == 2));
                ext_normal(tsdf, nb, xv + (i == 0), yv + (i == 1), zv + (i == 2), R, ne);
                const float nx = (1 - ratio) * no[0] + ratio * ne[0];
                const float ny = (1 - ratio) * no[1] + ratio * ne[1];
                const float nz = (1 - ratio) * no[2] + ratio * ne[2];
                /* (float)(sqrt(n.n) + 1e-5) (:1341-1342): the unqualified sqrt of a float resolves to the double
                 * overload in the reference's CPU build (pinned by tests/test_oracle_vs_ref_extract.py) */
                const float norm = (float)(sqrt(nx * nx + ny * ny + nz * nz) + 1e-5);
                float* n = normals + 3 * idx;
                n[0] = nx / norm;
                n[1] = ny / norm;
                n[2] = nz / norm;
                if (color && colors) {
                    const uint16_t* co = color + 3 * lin;
                    const uint16_t* ci = color + 3 * lin_i;
                    float* c = colors + 3 * idx;
                    for (int k = 0; k < 3; ++k) {
                        const float f_o = co[k], f_i = ci[k];
                        c[k] = ((1 - ratio) * f_o + ratio * f_i) / 255.0f;
                    }
                }
            }
        }
    }
    free(map.head);
    free(map.next);
    return count;
}
