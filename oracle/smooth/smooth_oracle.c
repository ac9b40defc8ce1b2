/* smooth_oracle.c — CPU restatement of t::geometry::PointCloud::SmoothLaplacian / SmoothTaubin (one pass),
 * SmoothMLS and SmoothBilateral (per point) on given neighbour lists, Float32 clouds
 * (t/geometry/kernel/PointCloudImpl.h:1357-1406, 1559-1655, 1697-1749).
 *
 * TEST INFRASTRUCTURE ONLY, like the rest of oracle/: the product never links or calls it.
 *
 * Precision follows the reference's CPU build (g++ -ffp-contract=off): every sum in f32 in neighbour-list order.  The
 * transcendental functions are chosen per call by `device_math`:
 *   0: libm's expf, acosf and cosf, as the reference's object code calls them;
 *   1: exp, acos and cos in f64, rounded to f32, as the device evaluates them.
 * The eigen solve is normals_oracle.c's, compiled in below with its acosf / cosf routed through that choice.  The
 * neighbour lists come from oracle/knn's brute force and oracle.hybrid_search(bruteforce=True).  Not reentrant: the
 * choice is a file-scope flag set by each entry point.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

static int g_device_math;

static float orc_acosf(float x) { return g_device_math ? (float)acos((double)x) : acosf(x); }
static float orc_cosf(float x) { return g_device_math ? (float)cos((double)x) : cosf(x); }
static float orc_expf(float x) { return g_device_math ? (float)exp((double)x) : expf(x); }

#define acosf orc_acosf
#define cosf orc_cosf
#include "../normals/normals_oracle.c"
#undef acosf
#undef cosf

/* ApplyLaplacianPass for the rows `rows` (NULL: rows 0 .. nrows-1) of a cloud; idx [nrows, kp] holds each row's
 * neighbours (-1 = none), out [nrows, 3] the moved points. */
void orc_laplacian_pass_f32(const float* pts, const int64_t* rows, int64_t nrows, const int32_t* idx, int kp,
                            double factor, float* out) {
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < nrows; ++r) {
        const int64_t i = rows ? rows[r] : r;
        float mean[3] = {0, 0, 0};
        int32_t count = 0;
        for (int s = 0; s < kp; ++s) {
            const int32_t j = idx[r * kp + s];
            if (j < 0 || j == i) continue;
            mean[0] += pts[3 * (int64_t)j];
            mean[1] += pts[3 * (int64_t)j + 1];
            mean[2] += pts[3 * (int64_t)j + 2];
            ++count;
        }
        const float* p = pts + 3 * i;
        float* o = out + 3 * r;
        if (count == 0) {
            memcpy(o, p, 3 * sizeof(float));
            continue;
        }
        const float inv_count = (float)(1.0 / count);
        const float alpha = (float)factor;
        for (int k = 0; k < 3; ++k) o[k] = p[k] + alpha * (mean[k] * inv_count - p[k]);
    }
}

/* SmoothMLS's per-point body.  Point i's list is idx[i * stride, + count), count = cnt[i] or, with cnt NULL, stride;
 * d2 NULL means every distance is 0 (the KNN branch).  out holds the positions on entry; normals (NULL: none) is
 * updated in place. */
void orc_mls_f32(const float* pts, int64_t n, const int32_t* idx, const float* d2, const int32_t* cnt, int stride,
                 double radius, float* normals, float* out, int device_math) {
    g_device_math = device_math;
    const float inv_radius2 = radius > 0.0 ? (float)(1.0 / (radius * radius)) : 0.0f;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        const int64_t o = i * stride;
        const int32_t count = cnt ? cnt[i] : stride;
        const float* p = pts + 3 * i;
        if (count < 3) {
            if (normals) {
                float* v = normals + 3 * i;
                const float norm = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
                if (norm > 0) {
                    v[0] /= norm;
                    v[1] /= norm;
                    v[2] /= norm;
                }
            }
            continue;
        }
        float c[3] = {0, 0, 0}, wsum = 0;
        for (int s = 0; s < count; ++s) {
            const int32_t j = idx[o + s];
            if (j < 0) continue;
            const float w = orc_expf(-(d2 ? d2[o + s] : 0.0f) * inv_radius2);
            c[0] += w * pts[3 * (int64_t)j];
            c[1] += w * pts[3 * (int64_t)j + 1];
            c[2] += w * pts[3 * (int64_t)j + 2];
            wsum += w;
        }
        if (wsum <= 0) continue;
        c[0] /= wsum;
        c[1] /= wsum;
        c[2] /= wsum;
        float C[9] = {0};
        for (int s = 0; s < count; ++s) {
            const int32_t j = idx[o + s];
            if (j < 0) continue;
            const float w = orc_expf(-(d2 ? d2[o + s] : 0.0f) * inv_radius2);
            const float x = pts[3 * (int64_t)j] - c[0], y = pts[3 * (int64_t)j + 1] - c[1],
                        z = pts[3 * (int64_t)j + 2] - c[2];
            C[0] += w * x * x;
            C[1] += w * x * y;
            C[2] += w * x * z;
            C[4] += w * y * y;
            C[5] += w * y * z;
            C[8] += w * z * z;
        }
        C[3] = C[1];
        C[6] = C[2];
        C[7] = C[5];
        float v[3];
        orc_normal_from_covariance_f32(C, v);
        const float proj = (p[0] - c[0]) * v[0] + (p[1] - c[1]) * v[1] + (p[2] - c[2]) * v[2];
        for (int k = 0; k < 3; ++k) out[3 * i + k] = p[k] - proj * v[k];
        if (normals) memcpy(normals + 3 * i, v, sizeof(v));
    }
}

/* SmoothBilateral's per-point body on hybrid-search lists idx, d2 [n, max_nn], cnt [n]; out holds the positions on
 * entry. */
void orc_bilateral_f32(const float* pts, const float* normals, int64_t n, const int32_t* idx, const float* d2,
                       const int32_t* cnt, int max_nn, double sigma_s, double sigma_r, float* out, int device_math) {
    g_device_math = device_math;
    const float inv_s2 = (float)(1.0 / (2.0 * sigma_s * sigma_s));
    const float inv_r2 = (float)(1.0 / (2.0 * sigma_r * sigma_r));
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        const int32_t count = cnt[i];
        if (count <= 1) continue;
        const float* p = pts + 3 * i;
        float nx = normals[3 * i], ny = normals[3 * i + 1], nz = normals[3 * i + 2];
        const float norm = sqrtf(nx * nx + ny * ny + nz * nz);
        if (norm <= 0) continue;
        nx /= norm;
        ny /= norm;
        nz /= norm;
        float ws[3] = {0, 0, 0}, wsum = 0;
        const int64_t o = i * max_nn;
        for (int s = 0; s < count; ++s) {
            const int32_t j = idx[o + s];
            if (j < 0) continue;
            const float* q = pts + 3 * (int64_t)j;
            const float r = (p[0] - q[0]) * nx + (p[1] - q[1]) * ny + (p[2] - q[2]) * nz;
            const float w = orc_expf(-d2[o + s] * inv_s2 - r * r * inv_r2);
            ws[0] += w * q[0];
            ws[1] += w * q[1];
            ws[2] += w * q[2];
            wsum += w;
        }
        if (wsum > 0)
            for (int k = 0; k < 3; ++k) out[3 * i + k] = ws[k] / wsum;
    }
}
