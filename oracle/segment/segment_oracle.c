// segment_oracle.c — CPU oracle of RANSAC plane segmentation, geometry::PointCloud::SegmentPlane
// (geometry/PointCloudSegmentation.cpp:157-279) run on one thread, restated in C from the contract of
// include/open3d_b200.h (o3db_segment_plane) and DESIGN.md §4.21.  TEST INFRASTRUCTURE.
//
// It takes the samples as input (the library's sampler is checked on its own).  Every sum over points runs
// sequentially over the points of each tile of `tile` points in index order, from 0, and then over the tiles in
// order, from 0; tile >= n gives upstream's single sequential sum.  f64 throughout, each op rounded (-ffp-contract=off).
// The hypotheses of a wave of 128 are scored in parallel (OpenMP); the serial rule then walks them in index order.
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define WAVE 128

typedef struct {
    double fitness, rmse;
} score_t;

// Eigen's Vector3d::dot order, (a0*b0 + a1*b1) + a2*b2
static double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

// Eigen's Vector4d::dot order for plane . (x, y, z, 1): (a*x + c*z) + (b*y + d)
static double dist(const double* pl, const float* p) {
    return fabs((pl[0] * (double)p[0] + pl[2] * (double)p[2]) + (pl[1] * (double)p[1] + pl[3]));
}

// abc / |abc|, d = -abc . c; zero when |abc| == 0 (TriangleMesh.cpp:1254-1261, PointCloudSegmentation.cpp:147-154)
static void finish_plane(double* abc, const double* c, double* out) {
    const double norm = sqrt(dot3(abc, abc));
    if (norm == 0) {
        out[0] = out[1] = out[2] = out[3] = 0;
        return;
    }
    for (int k = 0; k < 3; ++k) out[k] = abc[k] / norm;
    out[3] = -dot3(out, c);
}

// GetPlaneFromPoints (PointCloudSegmentation.cpp:131-154) from the centroid and the second moments
static void plane_from_moments(const double* c, const double* m, double* out) {
    const double xx = m[0], xy = m[1], xz = m[2], yy = m[3], yz = m[4], zz = m[5];
    const double det_x = yy * zz - yz * yz, det_y = xx * zz - xz * xz, det_z = xx * yy - xy * xy;
    double abc[3];
    if (det_x > det_y && det_x > det_z) {
        abc[0] = det_x;
        abc[1] = xz * yz - xy * zz;
        abc[2] = xy * yz - xz * yy;
    } else if (det_y > det_z) {
        abc[0] = xz * yz - xy * zz;
        abc[1] = det_y;
        abc[2] = xy * xz - yz * xx;
    } else {
        abc[0] = xy * yz - xz * yy;
        abc[1] = xy * xz - yz * xx;
        abc[2] = det_z;
    }
    finish_plane(abc, c, out);
}

static void moments_add(double* m, const double* r) {
    m[0] += r[0] * r[0];
    m[1] += r[0] * r[1];
    m[2] += r[0] * r[2];
    m[3] += r[1] * r[1];
    m[4] += r[1] * r[2];
    m[5] += r[2] * r[2];
}

static void hypothesis(const float* pts, const int64_t* s, int ransac_n, double* out) {
    double c[3] = {0, 0, 0};
    if (ransac_n == 3) {   // ComputeTrianglePlane (TriangleMesh.cpp:1248-1262)
        double p[3][3];
        for (int i = 0; i < 3; ++i)
            for (int k = 0; k < 3; ++k) p[i][k] = (double)pts[3 * s[i] + k];
        const double e0[3] = {p[1][0] - p[0][0], p[1][1] - p[0][1], p[1][2] - p[0][2]};
        const double e1[3] = {p[2][0] - p[0][0], p[2][1] - p[0][1], p[2][2] - p[0][2]};
        double abc[3] = {e0[1] * e1[2] - e0[2] * e1[1], e0[2] * e1[0] - e0[0] * e1[2], e0[0] * e1[1] - e0[1] * e1[0]};
        finish_plane(abc, p[0], out);
        return;
    }
    for (int i = 0; i < ransac_n; ++i)
        for (int k = 0; k < 3; ++k) c[k] += (double)pts[3 * s[i] + k];
    for (int k = 0; k < 3; ++k) c[k] /= (double)ransac_n;
    double m[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < ransac_n; ++i) {
        double r[3];
        for (int k = 0; k < 3; ++k) r[k] = (double)pts[3 * s[i] + k] - c[k];
        moments_add(m, r);
    }
    plane_from_moments(c, m, out);
}

static int is_zero(const double* pl) { return pl[0] == 0 && pl[1] == 0 && pl[2] == 0 && pl[3] == 0; }

// EvaluateRANSACBasedOnDistance (PointCloudSegmentation.cpp:78-107), the error summed in tile order
static score_t score(const float* pts, int64_t n, const double* pl, double thr, int64_t tile) {
    int64_t cnt = 0;
    double err = 0;
    for (int64_t lo = 0; lo < n; lo += tile) {
        const int64_t hi = lo + tile < n ? lo + tile : n;
        double e = 0;
        for (int64_t i = lo; i < hi; ++i) {
            const double d = dist(pl, pts + 3 * i);
            if (d < thr) {
                e += d * d;
                ++cnt;
            }
        }
        err += e;
    }
    score_t r = {0, 0};
    if (cnt) {
        r.fitness = (double)cnt / (double)n;
        r.rmse = sqrt(err / (double)cnt);
    }
    return r;
}

// samples [num_iterations][ransac_n].  plane [4]; inliers [n] receives the final inliers, *num_inliers their count;
// stats: best index (-1 for none), evaluated count; fit_rmse: the best fitness and rmse.  Returns 0, -1 on bad
// arguments, -2 when out of memory.
int orc_segment_plane(const float* pts, int64_t n, const int64_t* samples, int num_iterations, int ransac_n,
                      double thr, double probability, int64_t tile, double* plane, int64_t* inliers,
                      int64_t* num_inliers, int64_t* stats, double* fit_rmse) {
    if (n < 0 || ransac_n < 3 || n < ransac_n || tile < 1 || !(probability > 0 && probability <= 1)) return -1;
    const int H = num_iterations > 0 ? num_iterations : 0;
    double* planes = malloc(sizeof(double) * 4 * (H ? H : 1));
    score_t* sc = malloc(sizeof(score_t) * WAVE);
    if (!planes || !sc) {
        free(planes);
        free(sc);
        return -2;
    }
#pragma omp parallel for schedule(static)
    for (int h = 0; h < H; ++h) hypothesis(pts, samples + (int64_t)h * ransac_n, ransac_n, planes + 4 * (int64_t)h);

    // the serial rule of PointCloudSegmentation.cpp:200-253
    double best_fit = 0, best_rmse = 0;
    size_t brk = SIZE_MAX, count = 0;
    int64_t best = -1;
    for (int w = 0; w < H && count <= brk; w += WAVE) {
        const int hw = H - w < WAVE ? H - w : WAVE;
#pragma omp parallel for schedule(dynamic, 1)
        for (int k = 0; k < hw; ++k) sc[k] = score(pts, n, planes + 4 * (int64_t)(w + k), thr, tile);
        for (int k = 0; k < hw; ++k) {
            if (count > brk) break;
            if (is_zero(planes + 4 * (int64_t)(w + k))) continue;
            if (sc[k].fitness > best_fit || (sc[k].fitness == best_fit && sc[k].rmse < best_rmse)) {
                best_fit = sc[k].fitness;
                best_rmse = sc[k].rmse;
                best = w + k;
                if (best_fit < 1.0) {
                    const double q = log(1 - probability) / log(1 - pow(best_fit, ransac_n));
                    const double v = (double)num_iterations < q ? (double)num_iterations : q;   // std::min(q, N)
                    // size_t(v) as gcc compiles it for x86-64: -inf and NaN give 2^63
                    brk = v >= 0 ? (size_t)v : (size_t)1 << 63;
                } else {
                    brk = 0;
                }
            }
            ++count;
        }
    }

    // final inliers and the refit, sums in tile order (PointCloudSegmentation.cpp:255-271)
    int64_t K = 0;
    if (best >= 0) {
        const double* pl = planes + 4 * best;
        for (int64_t i = 0; i < n; ++i)
            if (dist(pl, pts + 3 * i) < thr) inliers[K++] = i;
    }
    double c[3] = {0, 0, 0}, m[6] = {0, 0, 0, 0, 0, 0};
    int64_t j = 0;
    for (int64_t lo = 0; lo < n; lo += tile) {
        const int64_t hi = lo + tile < n ? lo + tile : n;
        double t[3] = {0, 0, 0};
        for (; j < K && inliers[j] < hi; ++j)
            for (int k = 0; k < 3; ++k) t[k] += (double)pts[3 * inliers[j] + k];
        for (int k = 0; k < 3; ++k) c[k] += t[k];
    }
    for (int k = 0; k < 3; ++k) c[k] /= (double)K;
    j = 0;
    for (int64_t lo = 0; lo < n; lo += tile) {
        const int64_t hi = lo + tile < n ? lo + tile : n;
        double t[6] = {0, 0, 0, 0, 0, 0};
        for (; j < K && inliers[j] < hi; ++j) {
            double r[3];
            for (int k = 0; k < 3; ++k) r[k] = (double)pts[3 * inliers[j] + k] - c[k];
            moments_add(t, r);
        }
        for (int k = 0; k < 6; ++k) m[k] += t[k];
    }
    plane_from_moments(c, m, plane);
    *num_inliers = K;
    stats[0] = best;
    stats[1] = (int64_t)count;
    fit_rmse[0] = best_fit;
    fit_rmse[1] = best_rmse;
    free(planes);
    free(sc);
    return 0;
}
