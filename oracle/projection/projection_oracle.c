/*
 * projection_oracle.c — TEST INFRASTRUCTURE.  A C restatement of the reference's point-cloud <-> image projection, the
 * checker of open3d_b200/csrc/projection.cu:
 *   orc_unproject  kernel::pointcloud::Unproject (t/geometry/kernel/PointCloudImpl.h:43-144), rows row-major over the
 *                  strided grid instead of upstream's atomic-counter order;
 *   orc_project    kernel::pointcloud::Project with the CUDA kernel's per-pixel rule (PointCloudCUDA.cu:26-162): the
 *                  least (float bits of the depth, point index) wins, depth-only images included.
 * Camera geometry from ../geometry_indexer.h; f32 expressions op by op (-ffp-contract=off).  Pinned against the
 * reference's own UnprojectCPU / ProjectCPU by tests/test_oracle_vs_ref_projection.py.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../geometry_indexer.h"

/* depth: [rows][cols] u16 (depth_f32 == 0) or f32; color: NULL or [rows][cols][3] u8 (color_f32 == 0) or f32.
 * pose = InverseTransformation(extrinsics) (PointCloudImpl.h:63).  points / colors need room for
 * (rows / stride) * (cols / stride) rows; returns the number written. */
int64_t orc_unproject(const void* depth, int depth_f32, int rows, int cols, const void* color, int color_f32,
                      const double K[9], const double pose[16], float depth_scale, float depth_max, int stride,
                      float* points, float* colors) {
    xform_indexer t;
    xi_init(&t, K, pose, 1.0f);
    const int64_t rs = rows / stride, cs = cols / stride;
    int64_t n = 0;
    for (int64_t i = 0; i < rs; ++i) {
        for (int64_t j = 0; j < cs; ++j) {
            const int64_t y = i * stride, x = j * stride, p = y * cols + x;
            const float raw = depth_f32 ? ((const float*)depth)[p] : (float)((const uint16_t*)depth)[p];
            const float d = raw / depth_scale;
            if (!(d > 0 && d < depth_max)) continue;
            float xc, yc, zc;
            xi_unproject(&t, (float)x, (float)y, d, &xc, &yc, &zc);
            xi_rigid(&t, xc, yc, zc, points + 3 * n, points + 3 * n + 1, points + 3 * n + 2);
            if (color) {
                for (int k = 0; k < 3; ++k)
                    colors[3 * n + k] = color_f32 ? ((const float*)color)[3 * p + k]
                                                  : (float)((const uint8_t*)color)[3 * p + k];
            }
            ++n;
        }
    }
    return n;
}

/* points [n][3], colors NULL or [n][3]; depth [rows][cols] and color NULL or [rows][cols][3] are overwritten, 0 where
 * no point lands.  Returns -1 when out of memory. */
int orc_project(const float* points, const float* colors, int64_t n, const double K[9], const double E[16],
                float depth_scale, float depth_max, int rows, int cols, float* depth, float* color) {
    xform_indexer t;
    xi_init(&t, K, E, 1.0f);
    const int64_t npix = (int64_t)rows * cols;
    uint64_t* key = (uint64_t*)malloc((size_t)(npix > 0 ? npix : 1) * sizeof(uint64_t));
    if (!key) return -1;
    memset(key, 0xff, (size_t)npix * sizeof(uint64_t));
    for (int64_t i = 0; i < n; ++i) {
        float xc, yc, zc, u, v;
        xi_rigid(&t, points[3 * i], points[3 * i + 1], points[3 * i + 2], &xc, &yc, &zc);
        xi_project(&t, xc, yc, zc, &u, &v);
        u = roundf(u);
        v = roundf(v);
        if (!in_boundary(u, v, rows, cols) || zc <= 0 || zc > depth_max) continue;
        const float d = zc * depth_scale;
        uint32_t bits;
        memcpy(&bits, &d, 4);
        const uint64_t k = ((uint64_t)bits << 32) | (uint32_t)i;
        uint64_t* slot = key + (int64_t)v * cols + (int64_t)u;
        if (k < *slot) *slot = k;
    }
    for (int64_t p = 0; p < npix; ++p) {
        const int hit = key[p] != UINT64_MAX;
        const uint32_t bits = (uint32_t)(key[p] >> 32);
        float d = 0.0f;
        if (hit) memcpy(&d, &bits, 4);
        depth[p] = d;
        if (color) {
            const int64_t w = (int64_t)(uint32_t)key[p];
            for (int k = 0; k < 3; ++k) color[3 * p + k] = hit ? colors[3 * w + k] : 0.0f;
        }
    }
    free(key);
    return 0;
}
