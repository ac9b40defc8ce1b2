/* normals_oracle.c — CPU restatement of t::geometry::PointCloud::EstimateNormals (hybrid search) and the two
 * OrientNormals* calls (t/geometry/PointCloud.cpp:856-1040, t/geometry/kernel/PointCloudImpl.h), Float32 clouds.
 *
 * TEST INFRASTRUCTURE ONLY, like the rest of oracle/: the product never links or calls it.
 *
 * Precision follows the reference's CPU build (g++ -ffp-contract=off):
 *   covariance (PointCloudImpl.h:512-586): centroid and cumulants in f64, in neighbour-list order, Bessel's
 *     correction, stored as f32; fewer than 3 neighbours give the identity;
 *   normal (PointCloudImpl.h:746-1009, EstimatePointWiseNormalsWithFastEigen3x3<float>): f32, except where the
 *     expression holds a double literal — q, p (an f64 sqrt) and the angle are evaluated in f64 and rounded to f32;
 *     acos and cos are libm's f32 acosf / cosf, as the reference's object code calls them;
 *   orientation (PointCloudImpl.h:1011-1065): without prior normals a zero normal becomes (0,0,1); with prior
 *     normals the new normal is flipped where its dot with the prior is negative, and a zero normal stays zero.
 * Every function is checked bit for bit against the reference's own, compiled from its headers into
 * oracle/_ref/libo3dref_normals.so (tests/test_oracle_vs_ref_normals.py).  The neighbour lists come from the
 * oracle's hybrid search (oracle/icp_oracle.c), which orders them as the product does.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

/* PointCloudImpl.h:512-586 EstimatePointWiseRobustNormalizedCovarianceKernel<float>: centroid and the six cumulants
 * in f64, in neighbour-list order, Bessel's correction, stored as f32; fewer than 3 neighbours give the identity. */
void orc_covariance_point_f32(const float* pts, const int32_t* idx, int count, float cov[9]) {
    if (count < 3) {
        for (int k = 0; k < 9; ++k) cov[k] = (k % 4 == 0) ? 1.0f : 0.0f;
        return;
    }
    double c[3] = {0, 0, 0};
    for (int i = 0; i < count; ++i) {
        const int64_t a = 3 * (int64_t)idx[i];
        c[0] += pts[a];
        c[1] += pts[a + 1];
        c[2] += pts[a + 2];
    }
    c[0] /= count;
    c[1] /= count;
    c[2] /= count;
    double m[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < count; ++i) {
        const int64_t a = 3 * (int64_t)idx[i];
        const double x = (double)pts[a] - c[0], y = (double)pts[a + 1] - c[1], z = (double)pts[a + 2] - c[2];
        m[0] += x * x;
        m[1] += y * y;
        m[2] += z * z;
        m[3] += x * y;
        m[4] += x * z;
        m[5] += y * z;
    }
    const double f = (double)(count - 1);
    for (int k = 0; k < 6; ++k) m[k] /= f;
    cov[0] = (float)m[0];
    cov[4] = (float)m[1];
    cov[8] = (float)m[2];
    cov[1] = cov[3] = (float)m[3];
    cov[2] = cov[6] = (float)m[4];
    cov[5] = cov[7] = (float)m[5];
}

static inline void cross3f(const float* a, const float* b, float* c) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

static inline float dot3f(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

/* PointCloudImpl.h:746-796 ComputeEigenvector0<float> */
static void eigenvector0_f32(const float* A, float eval0, float* v) {
    const float r0[3] = {A[0] - eval0, A[1], A[2]};
    const float r1[3] = {A[1], A[4] - eval0, A[5]};
    const float r2[3] = {A[2], A[5], A[8] - eval0};
    float c[3][3];
    cross3f(r0, r1, c[0]);
    cross3f(r0, r2, c[1]);
    cross3f(r1, r2, c[2]);
    const float d[3] = {dot3f(c[0], c[0]), dot3f(c[1], c[1]), dot3f(c[2], c[2])};
    float dmax = d[0];
    int imax = 0;
    if (d[1] > dmax) {
        dmax = d[1];
        imax = 1;
    }
    if (d[2] > dmax) imax = 2;
    const float s = sqrtf(d[imax]);
    v[0] = c[imax][0] / s;
    v[1] = c[imax][1] / s;
    v[2] = c[imax][2] / s;
}

/* PointCloudImpl.h:798-873 ComputeEigenvector1<float> (1.0 / sqrtf in f64 rounds as the f32 division does) */
static void eigenvector1_f32(const float* A, const float* e0, float eval1, float* v) {
    float U[3];
    if (fabsf(e0[0]) > fabsf(e0[1])) {
        const float inv = (float)(1.0 / sqrtf(e0[0] * e0[0] + e0[2] * e0[2]));
        U[0] = -e0[2] * inv;
        U[1] = 0.0f;
        U[2] = e0[0] * inv;
    } else {
        const float inv = (float)(1.0 / sqrtf(e0[1] * e0[1] + e0[2] * e0[2]));
        U[0] = 0.0f;
        U[1] = e0[2] * inv;
        U[2] = -e0[1] * inv;
    }
    float V[3], AU[3], AV[3];
    cross3f(e0, U, V);
    for (int r = 0; r < 3; ++r) {
        AU[r] = A[3 * r] * U[0] + A[3 * r + 1] * U[1] + A[3 * r + 2] * U[2];
        AV[r] = A[3 * r] * V[0] + A[3 * r + 1] * V[1] + A[3 * r + 2] * V[2];
    }
    float m00 = dot3f(U, AU) - eval1, m01 = dot3f(U, AV), m11 = dot3f(V, AV) - eval1;
    const float a00 = fabsf(m00), a01 = fabsf(m01), a11 = fabsf(m11);
    if (a00 >= a11) {
        const float mx = a00 < a01 ? a01 : a00; /* std::max */
        if (mx > 0) {
            if (a00 >= a01) {
                m01 /= m00;
                m00 = 1 / sqrtf(1 + m01 * m01);
                m01 *= m00;
            } else {
                m00 /= m01;
                m01 = 1 / sqrtf(1 + m00 * m00);
                m00 *= m01;
            }
            for (int k = 0; k < 3; ++k) v[k] = m01 * U[k] - m00 * V[k];
            return;
        }
    } else {
        const float mx = a11 < a01 ? a01 : a11;
        if (mx > 0) {
            if (a11 >= a01) {
                m01 /= m11;
                m11 = 1 / sqrtf(1 + m01 * m01);
                m01 *= m11;
            } else {
                m11 /= m01;
                m01 = 1 / sqrtf(1 + m11 * m11);
                m11 *= m01;
            }
            for (int k = 0; k < 3; ++k) v[k] = m11 * U[k] - m01 * V[k];
            return;
        }
    }
    v[0] = U[0];
    v[1] = U[1];
    v[2] = U[2];
}

/* PointCloudImpl.h:875-1009 EstimatePointWiseNormalsWithFastEigen3x3<float>.  Where upstream's expression holds a
 * double literal it is evaluated in f64 and rounded to f32 (q, p, angle); acos and cos are libm's f32 acosf / cosf. */
void orc_normal_from_covariance_f32(const float cov[9], float out[3]) {
    float max_coeff = cov[0];
    for (int i = 1; i < 9; ++i)
        if (max_coeff < cov[i]) max_coeff = cov[i];
    if (max_coeff == 0) {
        out[0] = out[1] = out[2] = 0.0f;
        return;
    }
    float A[9];
    for (int i = 0; i < 9; ++i) A[i] = cov[i] / max_coeff;
    const float norm = A[1] * A[1] + A[2] * A[2] + A[5] * A[5];
    if (!(norm > 0)) {
        out[0] = out[1] = out[2] = 0.0f;
        if (cov[0] < cov[4] && cov[0] < cov[8])
            out[0] = 1.0f;
        else if (cov[4] < cov[0] && cov[4] < cov[8])
            out[1] = 1.0f;
        else
            out[2] = 1.0f;
        return;
    }
    const float q = (float)((A[0] + A[4] + A[8]) / 3.0);
    const float b00 = A[0] - q, b11 = A[4] - q, b22 = A[8] - q;
    const float p = (float)sqrt((b00 * b00 + b11 * b11 + b22 * b22 + norm * 2.0) / 6.0);
    const float c00 = b11 * b22 - A[5] * A[5];
    const float c01 = A[1] * b22 - A[5] * A[2];
    const float c02 = A[1] * A[5] - b11 * A[2];
    const float det = (b00 * c00 - A[1] * c01 + A[2] * c02) / (p * p * p);
    float half_det = (float)(det * 0.5);
    half_det = half_det < -1.0f ? -1.0f : half_det; /* std::max, then std::min */
    half_det = 1.0f < half_det ? 1.0f : half_det;
    const float angle = (float)(acosf(half_det) / 3.0);
    const float two_thirds_pi = (float)2.09439510239319549;
    const float beta2 = (float)(cosf(angle) * 2.0);
    const float beta0 = (float)(cosf(angle + two_thirds_pi) * 2.0);
    const float beta1 = -(beta0 + beta2);
    const float eval[3] = {q + p * beta0, q + p * beta1, q + p * beta2};
    float e0[3], e1[3];
    if (half_det >= 0) {
        eigenvector0_f32(A, eval[2], e0); /* evec2 */
        if (eval[2] < eval[0] && eval[2] < eval[1]) {
            memcpy(out, e0, sizeof(e0));
            return;
        }
        eigenvector1_f32(A, e0, eval[1], e1);
        if (eval[1] < eval[0] && eval[1] < eval[2]) {
            memcpy(out, e1, sizeof(e1));
            return;
        }
        cross3f(e1, e0, out);
    } else {
        eigenvector0_f32(A, eval[0], e0);
        if (eval[0] < eval[1] && eval[0] < eval[2]) {
            memcpy(out, e0, sizeof(e0));
            return;
        }
        eigenvector1_f32(A, e0, eval[1], e1);
        if (eval[1] < eval[0] && eval[1] < eval[2]) {
            memcpy(out, e1, sizeof(e1));
            return;
        }
        cross3f(e0, e1, out);
    }
}

/* PointCloudImpl.h:1011-1065 EstimateNormalsFromCovariances<float>, one point: without prior normals a zero normal
 * becomes (0,0,1); with them the normal is flipped where its dot with the prior is negative (a zero normal stays). */
static void normal_oriented_f32(const float cov[9], int has_normals, float* nrm) {
    float v[3];
    orc_normal_from_covariance_f32(cov, v);
    if (v[0] * v[0] + v[1] * v[1] + v[2] * v[2] == 0.0 && !has_normals) {
        v[0] = 0.0f;
        v[1] = 0.0f;
        v[2] = 1.0f;
    }
    if (has_normals && nrm[0] * v[0] + nrm[1] * v[1] + nrm[2] * v[2] < 0.0) {
        v[0] *= -1;
        v[1] *= -1;
        v[2] *= -1;
    }
    nrm[0] = v[0];
    nrm[1] = v[1];
    nrm[2] = v[2];
}

void orc_normals_from_covariances_f32(const float* cov, int64_t n, int has_normals, float* normals) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) normal_oriented_f32(cov + 9 * i, has_normals, normals + 3 * i);
}

/* EstimateCovariancesUsingHybridSearch + EstimateNormalsFromCovariances (PointCloud.cpp:856-984) on given neighbour
 * lists: idx [n, max_nn] (the point's hybrid-search neighbours, ascending distance), cnt [n].  normals holds the prior
 * normals on entry when has_normals; covariances [n, 9] may be NULL. */
void orc_estimate_normals_f32(const float* pts, int64_t n, const int32_t* idx, int max_nn, const int32_t* cnt,
                              int has_normals, float* normals, float* covariances) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        float cov[9];
        orc_covariance_point_f32(pts, idx + i * max_nn, cnt[i], cov);
        if (covariances) memcpy(covariances + 9 * i, cov, sizeof(cov));
        normal_oriented_f32(cov, has_normals, normals + 3 * i);
    }
}

/* PointCloudImpl.h:261-294 OrientNormalsToAlignWithDirection<float> */
void orc_orient_normals_to_align_with_direction_f32(float* nrm, int64_t n, const float dir[3]) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        float* v = nrm + 3 * i;
        const float norm = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
        if (norm == 0.0) {
            v[0] = dir[0];
            v[1] = dir[1];
            v[2] = dir[2];
        } else if (dot3f(v, dir) < 0) {
            v[0] *= -1;
            v[1] *= -1;
            v[2] *= -1;
        }
    }
}

/* PointCloudImpl.h:296-351 OrientNormalsTowardsCameraLocation<float> */
void orc_orient_normals_towards_camera_location_f32(const float* pts, float* nrm, int64_t n, const float cam[3]) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        float* v = nrm + 3 * i;
        const float* p = pts + 3 * i;
        const float r[3] = {cam[0] - p[0], cam[1] - p[1], cam[2] - p[2]};
        const float norm = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
        if (norm == 0.0) {
            v[0] = r[0];
            v[1] = r[1];
            v[2] = r[2];
            const float norm_new = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
            if (norm_new == 0.0) {
                v[0] = 0.0f;
                v[1] = 0.0f;
                v[2] = 1.0f;
            } else {
                v[0] /= norm_new;
                v[1] /= norm_new;
                v[2] /= norm_new;
            }
        } else if (dot3f(v, r) < 0) {
            v[0] *= -1;
            v[1] *= -1;
            v[2] *= -1;
        }
    }
}
