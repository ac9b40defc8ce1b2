/*
 * mesh_oracle.c — CPU restatement of Open3D's VoxelBlockGrid::ExtractTriangleMesh
 * (t/geometry/VoxelBlockGrid.cpp:436-472 -> kernel::voxel_grid::ExtractTriangleMesh,
 * t/geometry/kernel/VoxelBlockGridImpl.h:1385-1780) for the slam::Model value layout, with its own
 * marching-cubes case table generated from the face rule.
 *
 * TEST INFRASTRUCTURE ONLY, like the rest of oracle/: the checker of the CUDA extraction
 * (tests/test_mesh_gpu.py), itself pinned against the reference's own ExtractTriangleMeshCPU and tri_table
 * (oracle/ref_shim_mesh; tests/test_oracle_vs_ref_mesh.py).  It reuses the point-cloud oracle's block lookup and
 * DeviceGetLinearIdx / DeviceGetNormal restatements.  Compile with -ffp-contract=off.
 */
#include "../extract/extract_oracle.c"

#include <string.h>

/* Corners in the standard marching-cubes numbering (GeometryMacros.h vtx_shifts), edges as corner pairs, lower
 * corner first (edge_to_vert). */
static const int mc_corner[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0}, {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};
static const int mc_edge[12][2] = {{0, 1}, {1, 2}, {3, 2}, {0, 3}, {4, 5}, {5, 6}, {7, 6}, {4, 7}, {0, 4}, {1, 5}, {2, 6}, {3, 7}};
/* The six faces' corners, counter-clockwise seen from outside the cube. */
static const int mc_face[6][4] = {{0, 3, 2, 1}, {4, 5, 6, 7}, {0, 1, 5, 4}, {3, 7, 6, 2}, {0, 4, 7, 3}, {1, 2, 6, 5}};

static int orc_ntri[256];
static int orc_tri[256][15];
static int orc_edges[256];
static int orc_table_ready = 0;

static int edge_of(int a, int b) {
    for (int e = 0; e < 12; ++e)
        if ((mc_edge[e][0] == a && mc_edge[e][1] == b) || (mc_edge[e][0] == b && mc_edge[e][1] == a)) return e;
    abort();
}

/* The case table from the face rule.  Walking a face's corners counter-clockwise seen from outside, every run of
 * set (tsdf < 0) corners is cut off by one segment, from the edge where the walk leaves the run to the edge where it
 * enters it; on a face whose diagonal corners share their bit the two set corners are two runs.  The segments chain
 * into cycles; each cycle, from its lowest edge, is capped by the fan from that edge. */
static void build_table(void) {
    for (int c = 0; c < 256; ++c) {
        int next[12];
        for (int e = 0; e < 12; ++e) next[e] = -1;
        int edges = 0;
        for (int f = 0; f < 6; ++f) {
            for (int k = 0; k < 4; ++k) {
                const int p = mc_face[f][k], q = mc_face[f][(k + 1) & 3];
                const int sp = (c >> p) & 1, sq = (c >> q) & 1;
                if (sp && !sq) {   /* the walk leaves a run at edge (p, q): find where it entered */
                    int j = k;
                    while ((c >> mc_face[f][j]) & 1) j = (j + 3) & 3;   /* the clear corner before the run */
                    const int enter = edge_of(mc_face[f][j], mc_face[f][(j + 1) & 3]);
                    next[edge_of(p, q)] = enter;
                }
            }
        }
        for (int e = 0; e < 12; ++e)
            if (next[e] >= 0) edges |= 1 << e;
        int n = 0, seen = 0;
        for (int e0 = 0; e0 < 12; ++e0) {
            if (!((edges >> e0) & 1) || ((seen >> e0) & 1)) continue;
            int cyc[12], len = 0;
            for (int e = e0; !((seen >> e) & 1); e = next[e]) {
                seen |= 1 << e;
                cyc[len++] = e;
            }
            for (int i = 1; i + 1 < len; ++i) {
                if (n >= 5) abort();
                orc_tri[c][3 * n] = cyc[0];
                orc_tri[c][3 * n + 1] = cyc[i];
                orc_tri[c][3 * n + 2] = cyc[i + 1];
                ++n;
            }
        }
        orc_ntri[c] = n;
        orc_edges[c] = edges;
    }
    orc_table_ready = 1;
}

/* Row c of the oracle's table: triangles (edge triples, before the reversal) into tri[0..15), returns their count. */
int orc_mc_table_row(int c, int32_t* tri, int32_t* edge_mask) {
    if (!orc_table_ready) build_table();
    for (int i = 0; i < 3 * orc_ntri[c]; ++i) tri[i] = orc_tri[c][i];
    *edge_mask = orc_edges[c];
    return orc_ntri[c];
}

/* ExtractTriangleMeshCPU<float, uint16_t, uint16_t> over every block of the map, in the sequential order: vertices by
 * slot, voxel (z*R + y)*R + x and axis; triangles by slot, voxel and table, each written reversed (triangle[2 - k]).
 * The first min(count, max) rows of each array are written; returns the vertex count, *num_triangles the triangle
 * count. */
int64_t orc_extract_triangle_mesh(const int32_t* table_keys, int64_t size, const float* tsdf, const uint16_t* weight,
                                  const uint16_t* color, int resolution, float voxel_size, float weight_threshold,
                                  int64_t max_vertices, int64_t max_triangles, float* vertices, float* normals,
                                  float* colors, int32_t* triangles, int64_t* num_triangles) {
    if (!orc_table_ready) build_table();
    block_lookup map;
    if (lookup_build(&map, table_keys, size) != 0) abort();
    const int R = resolution;
    const int64_t R3 = (int64_t)R * R * R, n = size * R3;
    int64_t* nbs = (int64_t*)malloc((size_t)(size > 0 ? size : 1) * 27 * sizeof(int64_t));
    int16_t* cases = (int16_t*)malloc((size_t)(n > 0 ? n : 1) * sizeof(int16_t));   /* -1: cube does not contribute */
    int64_t* vidx = (int64_t*)malloc((size_t)(n > 0 ? n : 1) * 3 * sizeof(int64_t));   /* -2: no vertex, -1: marked */
    if (!nbs || !cases || !vidx) abort();
    for (int64_t b = 0; b < size; ++b) {
        const int32_t* key = table_keys + 3 * b;
        for (int k = 0; k < 27; ++k)
            nbs[27 * b + k] = lookup_find(&map, key[0] + k % 3 - 1, key[1] + (k % 9) / 3 - 1, key[2] + k / 9 - 1);
    }
    for (int64_t i = 0; i < 3 * n; ++i) vidx[i] = -2;
    /* pass 0 (:1460-1530): cases, and the edges of contributing cubes marked on their owning voxels */
    for (int64_t b = 0; b < size; ++b) {
        const int64_t* nb = nbs + 27 * b;
        for (int64_t v = 0; v < R3; ++v) {
            const int xv = (int)(v % R), yv = (int)((v / R) % R), zv = (int)(v / ((int64_t)R * R));
            int c = 0, ok = 1;
            for (int k = 0; k < 8 && ok; ++k) {
                const int64_t li = ext_linear_idx(nb, xv + mc_corner[k][0], yv + mc_corner[k][1], zv + mc_corner[k][2], R);
                if (li < 0) { ok = 0; break; }
                const float w = weight[li];
                if (w <= weight_threshold) { ok = 0; break; }
                if (tsdf[li] < 0) c |= 1 << k;
            }
            cases[b * R3 + v] = (int16_t)(ok ? c : -1);
            if (!ok) continue;
            for (int e = 0; e < 12; ++e) {
                if (!((orc_edges[c] >> e) & 1)) continue;
                const int* p = mc_corner[mc_edge[e][0]];
                const int* q = mc_corner[mc_edge[e][1]];
                const int axis = q[0] != p[0] ? 0 : q[1] != p[1] ? 1 : 2;
                const int64_t lo = ext_linear_idx(nb, xv + p[0], yv + p[1], zv + p[2], R);
                vidx[3 * lo + axis] = -1;
            }
        }
    }
    /* pass 2 (:1590-1690): vertices in order */
    int64_t nv = 0;
    for (int64_t b = 0; b < size; ++b) {
        const int64_t* nb = nbs + 27 * b;
        const int32_t* key = table_keys + 3 * b;
        for (int64_t v = 0; v < R3; ++v) {
            const int64_t lin = b * R3 + v;
            if (vidx[3 * lin] != -1 && vidx[3 * lin + 1] != -1 && vidx[3 * lin + 2] != -1) continue;
            const int xv = (int)(v % R), yv = (int)((v / R) % R), zv = (int)(v / ((int64_t)R * R));
            const int x = key[0] * R + xv, y = key[1] * R + yv, z = key[2] * R + zv;
            const float tsdf_o = tsdf[lin];
            float no[3] = {0, 0, 0}, ne[3] = {0, 0, 0};   /* ne is NOT reset between the axes */
            ext_normal(tsdf, nb, xv, yv, zv, R, no);
            for (int e = 0; e < 3; ++e) {
                if (vidx[3 * lin + e] != -1) continue;
                const int64_t lin_e = ext_linear_idx(nb, xv + (e == 0), yv + (e == 1), zv + (e == 2), R);
                const float tsdf_e = tsdf[lin_e];
                const float ratio = (0 - tsdf_o) / (tsdf_e - tsdf_o);
                const int64_t idx = nv++;
                vidx[3 * lin + e] = idx;
                if (idx >= max_vertices) continue;
                float* p = vertices + 3 * idx;
                p[0] = voxel_size * (x + ratio * (int)(e == 0));
                p[1] = voxel_size * (y + ratio * (int)(e == 1));
                p[2] = voxel_size * (z + ratio * (int)(e == 2));
                ext_normal(tsdf, nb, xv + (e == 0), yv + (e == 1), zv + (e == 2), R, ne);
                const float nx = (1 - ratio) * no[0] + ratio * ne[0];
                const float ny = (1 - ratio) * no[1] + ratio * ne[1];
                const float nz = (1 - ratio) * no[2] + ratio * ne[2];
                const float norm = (float)(sqrt(nx * nx + ny * ny + nz * nz) + 1e-5);
                float* nn = normals + 3 * idx;
                nn[0] = nx / norm;
                nn[1] = ny / norm;
                nn[2] = nz / norm;
                if (color && colors) {
                    const uint16_t* co = color + 3 * lin;
                    const uint16_t* ce = color + 3 * lin_e;
                    float* cc = colors + 3 * idx;
                    for (int k = 0; k < 3; ++k) {
                        const float f_o = co[k], f_e = ce[k];
                        cc[k] = ((1 - ratio) * f_o + ratio * f_e) / 255.0f;
                    }
                }
            }
        }
    }
    /* pass 3 (:1700-1760): triangles in order */
    int64_t nt = 0;
    for (int64_t b = 0; b < size; ++b) {
        const int64_t* nb = nbs + 27 * b;
        for (int64_t v = 0; v < R3; ++v) {
            const int c = cases[b * R3 + v];
            if (c < 0) continue;
            const int xv = (int)(v % R), yv = (int)((v / R) % R), zv = (int)(v / ((int64_t)R * R));
            for (int t = 0; t < orc_ntri[c]; ++t) {
                const int64_t idx = nt++;
                if (idx >= max_triangles) continue;
                for (int k = 0; k < 3; ++k) {
                    const int e = orc_tri[c][3 * t + k];
                    const int* p = mc_corner[mc_edge[e][0]];
                    const int* q = mc_corner[mc_edge[e][1]];
                    const int axis = q[0] != p[0] ? 0 : q[1] != p[1] ? 1 : 2;
                    const int64_t lo = ext_linear_idx(nb, xv + p[0], yv + p[1], zv + p[2], R);
                    triangles[3 * idx + 2 - k] = (int32_t)vidx[3 * lo + axis];
                }
            }
        }
    }
    free(nbs);
    free(cases);
    free(vidx);
    free(map.head);
    free(map.next);
    *num_triangles = nt;
    return nv;
}
