/* fps_oracle.c — CPU oracle of farthest-point down-sampling (o3db_farthest_point_down_sample), restating
 * upstream's t::geometry::PointCloud::FarthestPointDownSample (t/geometry/PointCloud.cpp:612-648) as DESIGN.md §4.20
 * writes it out.
 *
 * TEST INFRASTRUCTURE ONLY.
 *   distance  e = ((dx*dx + dy*dy) + dz*dz), dx = x_j - x_f, in f32, each op rounded (-ffp-contract=off): upstream
 *             computes diff = positions - selected and diff * diff in the positions' dtype (:637-638) and its CPU
 *             Sum({1}) adds the three terms in order;
 *   minimum   d[j] = min(d[j], e), d starting at +inf (:628-630, :639-640);
 *   next      the largest d[j] over the points not yet selected, ties to the lowest index: the strict > of the legacy
 *             geometry::PointCloud::FarthestPointDownSample (geometry/PointCloud.cpp:543-554).  Excluding selected
 *             points changes nothing while the largest d is positive, since a selected point has d = 0.
 * selected[r] receives the r-th selected index (selection order).  The points must be finite (the device rejects other
 * clouds).
 */
#include <math.h>
#include <omp.h>
#include <stdint.h>
#include <stdlib.h>

int orc_fps(const float* pts, int64_t n, int64_t num_samples, int64_t start_index, int32_t* selected) {
    if (n <= 0 || num_samples < 1 || num_samples > n || start_index < 0 || start_index >= n) return -1;
    float* d = (float*)malloc((size_t)n * sizeof(float));
    unsigned char* taken = (unsigned char*)calloc((size_t)n, 1);
    const int nt = omp_get_max_threads();
    float* tbest = (float*)malloc((size_t)nt * sizeof(float));
    int64_t* tidx = (int64_t*)malloc((size_t)nt * sizeof(int64_t));
    if (!d || !taken || !tbest || !tidx) {
        free(d);
        free(taken);
        free(tbest);
        free(tidx);
        return -2;
    }
    for (int64_t j = 0; j < n; ++j) d[j] = INFINITY;
    int64_t f = start_index;
    for (int64_t r = 0; r < num_samples; ++r) {
        selected[r] = (int32_t)f;
        taken[f] = 1;
        if (r + 1 == num_samples) break;
        const float fx = pts[3 * f], fy = pts[3 * f + 1], fz = pts[3 * f + 2];
        for (int t = 0; t < nt; ++t) tidx[t] = -1;
#pragma omp parallel num_threads(nt)
        {
            const int t = omp_get_thread_num();
            float best = -1.0f;
            int64_t bi = -1;
            /* static schedule: each thread a contiguous ascending block, so strict > keeps its lowest index */
#pragma omp for schedule(static)
            for (int64_t j = 0; j < n; ++j) {
                const float dx = pts[3 * j] - fx;
                const float dy = pts[3 * j + 1] - fy;
                const float dz = pts[3 * j + 2] - fz;
                const float xx = dx * dx, yy = dy * dy, zz = dz * dz;
                const float e = (xx + yy) + zz;
                if (e < d[j]) d[j] = e;
                if (!taken[j] && d[j] > best) {
                    best = d[j];
                    bi = j;
                }
            }
            tbest[t] = best;
            tidx[t] = bi;
        }
        /* the blocks are in thread order, so the first thread with the largest value holds the lowest index */
        float best = -1.0f;
        for (int t = 0; t < nt; ++t)
            if (tidx[t] >= 0 && tbest[t] > best) {
                best = tbest[t];
                f = tidx[t];
            }
    }
    free(d);
    free(taken);
    free(tbest);
    free(tidx);
    return 0;
}
