/* CPU oracle of TransformationEstimationPointToPoint and the ICP loop around it (test infrastructure).
 *
 * A restatement of the reference's CPU semantics, written from its description:
 *   - Get3x3SxyLinearSystem (t/pipelines/kernel/RegistrationCPU.cpp:497-617): pass 1 sums the matched source and
 *     target points and their count, pass 2 sums (s_k - mean s_k)(t_j - mean t_j); Sxy[j][k] is target row j, source
 *     column k, divided by the count.  All in the cloud's dtype, in index order (a serial reduction).
 *   - ComputeRtPointToPointCPU (:619-653): R = U diag(1, 1, sign(det U det V)) V^T of the SVD of Sxy,
 *     t = mean t - R mean s.  The SVD here is f64 and this file's own (the reference calls LAPACK in the cloud's
 *     dtype): the rotation is unique for rank >= 2, so only rounding differs.
 *   - TransformationEstimationPointToPoint::ComputeRMSE (registration/TransformationEstimation.cpp:101-130).
 *   - the loop of DoSingleScaleICPIterations / MultiScaleICP (registration/Registration.cpp:293-358, 398-431) with the
 *     rules of orc_icp_p2plane_f32 (../icp_oracle.c), whose search and transform it calls. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle.h"

#define P2P_SXY(NAME, T)                                                                                        \
    int64_t NAME(const T* src, const T* tgt, const int64_t* corr, int64_t n, T sxy[9], T mean_t[3], T mean_s[3]) { \
        T m[7] = {0, 0, 0, 0, 0, 0, 0};                                                                         \
        for (int64_t i = 0; i < n; ++i) {                                                                       \
            if (corr[i] == -1) continue;                                                                        \
            const int64_t t = 3 * corr[i];                                                                      \
            for (int k = 0; k < 3; ++k) {                                                                       \
                m[k] += src[3 * i + k];                                                                         \
                m[3 + k] += tgt[t + k];                                                                         \
            }                                                                                                   \
            m[6] += 1;                                                                                          \
        }                                                                                                       \
        if (m[6] == 0) return 0;                                                                                \
        for (int k = 0; k < 6; ++k) m[k] = m[k] / m[6];                                                         \
        T s[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};                                                                   \
        for (int64_t i = 0; i < n; ++i) {                                                                       \
            if (corr[i] == -1) continue;                                                                        \
            const int64_t t = 3 * corr[i];                                                                      \
            for (int q = 0; q < 9; ++q) s[q] += (src[3 * i + q % 3] - m[q % 3]) * (tgt[t + q / 3] - m[3 + q / 3]); \
        }                                                                                                       \
        for (int q = 0; q < 9; ++q) sxy[q] = s[q] / m[6];                                                       \
        for (int k = 0; k < 3; ++k) {                                                                           \
            mean_s[k] = m[k];                                                                                   \
            mean_t[k] = m[3 + k];                                                                               \
        }                                                                                                       \
        return (int64_t)m[6];                                                                                   \
    }
P2P_SXY(orc_p2p_sxy_f32, float)
P2P_SXY(orc_p2p_sxy_f64, double)

/* sqrt(sum |s - t|^2 / #valid): the squares in the cloud's dtype, their sum in f64 */
double orc_rmse_p2p_f32(const float* src, const float* tgt, const int64_t* corr, int64_t n) {
    double err = 0.0;
    int64_t cnt = 0;
    for (int64_t i = 0; i < n; ++i) {
        if (corr[i] == -1) continue;
        for (int c = 0; c < 3; ++c) {
            float e = src[3 * i + c] - tgt[3 * corr[i] + c];
            e = e * e;
            err += e;
        }
        ++cnt;
    }
    return sqrt(err / (double)cnt);
}

double orc_rmse_p2p_f64(const double* src, const double* tgt, const int64_t* corr, int64_t n) {
    double err = 0.0;
    int64_t cnt = 0;
    for (int64_t i = 0; i < n; ++i) {
        if (corr[i] == -1) continue;
        for (int c = 0; c < 3; ++c) {
            const double e = src[3 * i + c] - tgt[3 * corr[i] + c];
            err += e * e;
        }
        ++cnt;
    }
    return sqrt(err / (double)cnt);
}

/* Eigenvectors of the symmetric 3x3 A (cyclic two-sided Jacobi), as the columns of V; A becomes diagonal. */
static void eig_sym3(double A[3][3], double V[3][3]) {
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) V[r][c] = r == c;
    for (int sweep = 0; sweep < 60; ++sweep) {
        const double off = fabs(A[0][1]) + fabs(A[0][2]) + fabs(A[1][2]);
        if (off <= 1e-300 || off <= 1e-20 * (fabs(A[0][0]) + fabs(A[1][1]) + fabs(A[2][2]))) break;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                if (A[p][q] == 0.0) continue;
                const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 3; ++k) {   /* A <- A J */
                    const double akp = A[k][p], akq = A[k][q];
                    A[k][p] = c * akp - s * akq;
                    A[k][q] = s * akp + c * akq;
                }
                for (int k = 0; k < 3; ++k) {   /* A <- J^T A */
                    const double apk = A[p][k], aqk = A[q][k];
                    A[p][k] = c * apk - s * aqk;
                    A[q][k] = s * apk + c * aqk;
                }
                for (int k = 0; k < 3; ++k) {
                    const double vkp = V[k][p], vkq = V[k][q];
                    V[k][p] = c * vkp - s * vkq;
                    V[k][q] = s * vkp + c * vkq;
                }
            }
    }
}

static void cross3(const double a[3], const double b[3], double c[3]) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

/* [R t; 0 1] from Sxy (row-major, target rows) and the two means.  V from the eigenvectors of Sxy^T Sxy, ordered by
 * eigenvalue; u_1, u_2 = Sxy v / |Sxy v| (u_2 made orthogonal to u_1); the third pair of R = U S V^T enters as
 * (u_1 x u_2)(v_1 x v_2)^T, which is what the reflection fix S = diag(1, 1, sign(det U det V)) evaluates to.  Needs
 * rank >= 2; returns 0 otherwise and leaves T alone. */
int orc_p2p_kabsch_f64(const double sxy[9], const double mean_t[3], const double mean_s[3], double T[16]) {
    double A[3][3], V[3][3];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            A[r][c] = 0;
            for (int k = 0; k < 3; ++k) A[r][c] += sxy[3 * k + r] * sxy[3 * k + c];
        }
    eig_sym3(A, V);
    int o[3] = {0, 1, 2};
    for (int a = 0; a < 2; ++a)
        for (int b = a + 1; b < 3; ++b)
            if (A[o[b]][o[b]] > A[o[a]][o[a]]) {
                const int t = o[a];
                o[a] = o[b];
                o[b] = t;
            }
    double v[2][3], u[2][3], u3[3], v3[3];
    for (int i = 0; i < 2; ++i) {
        for (int r = 0; r < 3; ++r) v[i][r] = V[r][o[i]];
        for (int r = 0; r < 3; ++r) u[i][r] = sxy[3 * r] * v[i][0] + sxy[3 * r + 1] * v[i][1] + sxy[3 * r + 2] * v[i][2];
    }
    const double n1 = sqrt(u[0][0] * u[0][0] + u[0][1] * u[0][1] + u[0][2] * u[0][2]);
    if (!(n1 > 0)) return 0;
    for (int r = 0; r < 3; ++r) u[0][r] /= n1;
    const double d = u[1][0] * u[0][0] + u[1][1] * u[0][1] + u[1][2] * u[0][2];
    for (int r = 0; r < 3; ++r) u[1][r] -= d * u[0][r];
    const double n2 = sqrt(u[1][0] * u[1][0] + u[1][1] * u[1][1] + u[1][2] * u[1][2]);
    if (!(n2 > 1e-13 * n1)) return 0;
    for (int r = 0; r < 3; ++r) u[1][r] /= n2;
    cross3(u[0], u[1], u3);
    cross3(v[0], v[1], v3);
    for (int r = 0; r < 3; ++r) {
        double t = mean_t[r];
        for (int c = 0; c < 3; ++c) {
            const double R = u[0][r] * v[0][c] + u[1][r] * v[1][c] + u3[r] * v3[c];
            T[4 * r + c] = R;
            t -= R * mean_s[c];
        }
        T[4 * r + 3] = t;
    }
    T[12] = T[13] = T[14] = 0.0;
    T[15] = 1.0;
    return 1;
}

static void matmul4(const double A[16], const double B[16], double C[16]) {
    double R[16];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            double s = 0;
            for (int k = 0; k < 4; ++k) s += A[i * 4 + k] * B[k * 4 + j];
            R[i * 4 + j] = s;
        }
    memcpy(C, R, sizeof(R));
}

static void eye4(double T[16]) {
    for (int i = 0; i < 16; ++i) T[i] = (i % 5 == 0) ? 1.0 : 0.0;
}

/* Registration.cpp:24-62 ComputeRegistrationResult */
static void registration_result(const float* src, int64_t n, const float* tgt, int64_t m, double radius, int32_t* idx,
                                float* d2, int32_t* cnt, int64_t* corr, double* fitness, double* rmse, int64_t* count) {
    orc_hybrid_search_f32(tgt, m, src, n, radius, 1, idx, d2, cnt);
    double sq = 0.0;
    int64_t c = 0;
    for (int64_t i = 0; i < n; ++i) {
        corr[i] = cnt[i] ? (int64_t)idx[i] : -1;
        if (cnt[i]) {
            sq += (double)d2[i];
            c += 1;
        }
    }
    *count = c;
    *fitness = c ? (double)c / (double)n : 0.0;
    *rmse = c ? sqrt(sq / (double)c) : 0.0;
}

/* The loop of orc_icp_p2plane_f32 with the point-to-point estimator.  accumulate_f64 != 0: the two passes run in f64
 * over the f32 points (precise); 0: in f32, as the reference does for an f32 cloud.  Returns 0, or -1 without memory;
 * collinear matches (no unique rotation) end the loop as a singular system does there: return 1. */
int orc_icp_p2p_f32(const float* source, int64_t n, const float* target, int64_t m, double max_corr_dist,
                    const double init_T[16], int max_iteration, double rel_fitness, double rel_rmse, int accumulate_f64,
                    orc_icp_result* res, double* per_iter, int64_t* corr_out) {
    const size_t nn = (size_t)(n > 0 ? n : 1);
    float* src = (float*)malloc(nn * 3 * sizeof(float));
    double* src64 = accumulate_f64 ? (double*)malloc(nn * 3 * sizeof(double)) : NULL;
    double* tgt64 = accumulate_f64 ? (double*)malloc((size_t)(m > 0 ? m : 1) * 3 * sizeof(double)) : NULL;
    int64_t* corr = (int64_t*)malloc(nn * sizeof(int64_t));
    int32_t* idx = (int32_t*)malloc(nn * sizeof(int32_t));
    int32_t* cnt = (int32_t*)malloc(nn * sizeof(int32_t));
    float* d2 = (float*)malloc(nn * sizeof(float));
    int rc = 0;
    if (!src || !corr || !idx || !cnt || !d2 || (accumulate_f64 && (!src64 || !tgt64))) {
        rc = -1;
        goto done;
    }
    memcpy(src, source, (size_t)n * 3 * sizeof(float));
    if (accumulate_f64)
        for (int64_t i = 0; i < 3 * m; ++i) tgt64[i] = (double)target[i];
    double T[16];
    memcpy(T, init_T, sizeof(T));
    orc_transform_points_f32(T, src, n);   /* Registration.cpp:398-404 */

    double fitness = 0, rmse = 0, prev_fitness = 0, prev_rmse = 0;
    int64_t count = 0;
    int converged = 0, it = 0;
    for (it = 0; it < max_iteration; ++it) {
        registration_result(src, n, target, m, max_corr_dist, idx, d2, cnt, corr, &fitness, &rmse, &count);
        if (count == 0) eye4(T);                       /* :51-60 */
        if (fitness <= 2.2250738585072014e-308) break; /* :300-306 */
        double sxy[9], mt[3], ms[3], U[16];
        if (accumulate_f64) {
            for (int64_t i = 0; i < 3 * n; ++i) src64[i] = (double)src[i];
            orc_p2p_sxy_f64(src64, tgt64, corr, n, sxy, mt, ms);
        } else {
            float sxy32[9], mt32[3], ms32[3];
            orc_p2p_sxy_f32(src, target, corr, n, sxy32, mt32, ms32);
            for (int k = 0; k < 9; ++k) sxy[k] = (double)sxy32[k];
            for (int k = 0; k < 3; ++k) {
                mt[k] = (double)mt32[k];
                ms[k] = (double)ms32[k];
            }
        }
        if (!orc_p2p_kabsch_f64(sxy, mt, ms, U)) {
            rc = 1;
            goto done;
        }
        matmul4(U, T, T);                    /* :319 */
        orc_transform_points_f32(U, src, n); /* :322 */
        if (per_iter) {
            per_iter[2 * it + 0] = fitness;
            per_iter[2 * it + 1] = rmse;
        }
        if (it != 0 && fabs(prev_fitness - fitness) < rel_fitness && fabs(prev_rmse - rmse) < rel_rmse) { /* :348-355 */
            converged = 1;
            break;
        }
        prev_fitness = fitness;
        prev_rmse = rmse;
    }
    const int iterations = it;   /* :358: not incremented after a break */
    registration_result(src, n, target, m, max_corr_dist, idx, d2, cnt, corr, &fitness, &rmse, &count); /* :424-431 */
    if (count == 0) {
        eye4(T);
        converged = 0;
    }
    res->num_iterations = iterations;
    res->converged = converged;
    res->fitness = fitness;
    res->inlier_rmse = rmse;
    res->loop_seconds = res->build_seconds = 0.0;
    memcpy(res->transformation, T, sizeof(T));
    if (corr_out) memcpy(corr_out, corr, (size_t)n * sizeof(int64_t));
done:
    free(src);
    free(src64);
    free(tgt64);
    free(corr);
    free(idx);
    free(cnt);
    free(d2);
    return rc;
}
