/* CPU oracle of TransformationEstimationSymmetric and the ICP loop around it (test infrastructure).
 *
 * A restatement of the reference's CPU semantics, written from its description:
 *   - GetJacobianSymmetric (t/pipelines/kernel/RegistrationImpl.h:324-387): sign = (n_s . n_t < 0) ? -1 : 1,
 *     n = n_t + sign n_s, J = [(s - ms + t - mt) x n ; n], centred residual ((s - ms) - (t - mt)) . n, objective residual
 *     (s - t) . n; all in f32 in that order.
 *   - ComputePoseSymmetricKernelCPU (RegistrationCPU.cpp:124-180): weight of the objective residual, 21 + 6 slots of
 *     J^T w J and J^T w r_c, [27] sum of squared objective residuals, [28] count; a serial reduction in the cloud's
 *     dtype (the reference's TBB reduce with one range), or in f64 on request.
 *   - ComputeTransformationSymmetric (kernel/Registration.cpp:80-135): the means of the matched pairs (here in f64,
 *     then rounded to the cloud's dtype, which the kernel receives), DecodeAndSolve6x6 (../oracle.h) and
 *     PoseToSymmetricTransformation (SymmetricICPImpl.h:19-43): H = AngleAxis(atan|g|, g / |g|) by Rodrigues' formula,
 *     R = H H, t = mt + H (pose[3:6] cos(atan|g|)) - R ms; the identity with no valid correspondence.
 *   - TransformationEstimationSymmetric::ComputeRMSE (registration/TransformationEstimation.cpp:229-274).
 *   - the loop of DoSingleScaleICPIterations (registration/Registration.cpp:293-358): every iteration transforms the
 *     source's points AND normals by the update in f32 (PointCloud::Transform), with the rules of
 *     orc_icp_p2plane_f32 (../icp_oracle.c), whose search and transforms it calls. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle.h"

/* 1 when an entry lies outside [-1, m) (AssertValidSymmetricCorrespondences, TransformationEstimation.cpp:85-99) */
static int bad_corr(const int64_t* corr, int64_t n, int64_t m) {
    for (int64_t i = 0; i < n; ++i)
        if (corr[i] < -1 || corr[i] >= m) return 1;
    return 0;
}

/* The 29 sums about the given means.  accumulate_f64 = 0: float accumulators (the reference for an f32 cloud). */
void orc_sym_sums_f32(const float* src, const float* tgt, const float* sn, const float* tn, const int64_t* corr,
                      int64_t n, const float ms[3], const float mt[3], int method, double scale, double shape,
                      int accumulate_f64, double sums29[29]) {
    float a32[29];
    double a64[29];
    memset(a32, 0, sizeof(a32));
    memset(a64, 0, sizeof(a64));
    for (int64_t i = 0; i < n; ++i) {
        if (corr[i] == -1) continue;
        const float* s = src + 3 * i;
        const float* t = tgt + 3 * corr[i];
        const float* ns = sn + 3 * i;
        const float* nt = tn + 3 * corr[i];
        const float dot = ns[0] * nt[0] + ns[1] * nt[1] + ns[2] * nt[2];
        const float sg = dot < 0.f ? -1.f : 1.f;
        const float nx = nt[0] + sg * ns[0], ny = nt[1] + sg * ns[1], nz = nt[2] + sg * ns[2];
        const float sxc = s[0] - ms[0], syc = s[1] - ms[1], szc = s[2] - ms[2];
        const float txc = t[0] - mt[0], tyc = t[1] - mt[1], tzc = t[2] - mt[2];
        const float ux = sxc + txc, uy = syc + tyc, uz = szc + tzc;
        const float J[6] = {uy * nz - uz * ny, uz * nx - ux * nz, ux * ny - uy * nx, nx, ny, nz};
        const float rc = (sxc - txc) * nx + (syc - tyc) * ny + (szc - tzc) * nz;
        const float ro = (s[0] - t[0]) * nx + (s[1] - t[1]) * ny + (s[2] - t[2]) * nz;
        const float w = orc_robust_weight_f32(method, scale, shape, ro);
        int q = 0;
        for (int j = 0; j < 6; ++j) {
            for (int k = 0; k <= j; ++k, ++q) {
                if (accumulate_f64) a64[q] += (double)(J[j] * w * J[k]);
                else a32[q] += J[j] * w * J[k];
            }
            if (accumulate_f64) a64[21 + j] += (double)(J[j] * w * rc);
            else a32[21 + j] += J[j] * w * rc;
        }
        if (accumulate_f64) {
            a64[27] += (double)(ro * ro);
            a64[28] += 1;
        } else {
            a32[27] += ro * ro;
            a32[28] += 1;
        }
    }
    for (int k = 0; k < 29; ++k) sums29[k] = accumulate_f64 ? a64[k] : (double)a32[k];
}

/* Means of the matched pairs, rounded to f32; returns the count. */
int64_t orc_sym_means_f32(const float* src, const float* tgt, const int64_t* corr, int64_t n, float ms[3], float mt[3]) {
    double a[6] = {0, 0, 0, 0, 0, 0};
    int64_t c = 0;
    for (int64_t i = 0; i < n; ++i) {
        if (corr[i] == -1) continue;
        for (int k = 0; k < 3; ++k) {
            a[k] += src[3 * i + k];
            a[3 + k] += tgt[3 * corr[i] + k];
        }
        c += 1;
    }
    for (int k = 0; k < 3; ++k) {
        ms[k] = c ? (float)(a[k] / (double)c) : 0.f;
        mt[k] = c ? (float)(a[3 + k] / (double)c) : 0.f;
    }
    return c;
}

void orc_pose_to_symmetric_transformation(const double pose[6], const double ms[3], const double mt[3], double T[16]) {
    const double gn = sqrt(pose[0] * pose[0] + pose[1] * pose[1] + pose[2] * pose[2]);
    const double theta = atan(gn);
    double H[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    if (gn > 0.0) {   /* Rodrigues: H = cos I + sin [k]x + (1 - cos) k k^T */
        const double k[3] = {pose[0] / gn, pose[1] / gn, pose[2] / gn};
        const double c = cos(theta), s = sin(theta);
        const double K[3][3] = {{0, -k[2], k[1]}, {k[2], 0, -k[0]}, {-k[1], k[0], 0}};
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) H[i][j] = (i == j ? c : 0.0) + s * K[i][j] + (1.0 - c) * k[i] * k[j];
    }
    const double ct = cos(theta);
    for (int i = 0; i < 3; ++i) {
        double t = mt[i];
        for (int j = 0; j < 3; ++j) {
            double r = 0;
            for (int l = 0; l < 3; ++l) r += H[i][l] * H[l][j];
            T[4 * i + j] = r;
            t += H[i][j] * pose[3 + j] * ct;
        }
        T[4 * i + 3] = t;
    }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) T[4 * i + 3] -= T[4 * i + j] * ms[j];
    T[12] = T[13] = T[14] = 0.0;
    T[15] = 1.0;
}

static void eye4(double T[16]) {
    for (int i = 0; i < 16; ++i) T[i] = (i % 5 == 0) ? 1.0 : 0.0;
}

/* ComputeTransformationSymmetric -> T.  Returns 0, 1 for a singular system, -2 for a correspondence outside [-1, m). */
int orc_sym_transformation_f32(const float* src, const float* tgt, const float* sn, const float* tn, const int64_t* corr,
                               int64_t n, int64_t m, int method, double scale, double shape, int accumulate_f64,
                               double T[16]) {
    if (bad_corr(corr, n, m)) return -2;
    float ms[3], mt[3];
    if (orc_sym_means_f32(src, tgt, corr, n, ms, mt) == 0) {
        eye4(T);
        return 0;
    }
    double sums[29], pose[6], residual;
    int count;
    orc_sym_sums_f32(src, tgt, sn, tn, corr, n, ms, mt, method, scale, shape, accumulate_f64, sums);
    if (orc_decode_and_solve_6x6(sums, pose, &residual, &count)) return 1;
    const double ms64[3] = {ms[0], ms[1], ms[2]}, mt64[3] = {mt[0], mt[1], mt[2]};
    orc_pose_to_symmetric_transformation(pose, ms64, mt64, T);
    return 0;
}

/* ComputeRMSE; -1.0 for a correspondence outside [-1, m). */
double orc_rmse_sym_f32(const float* src, const float* tgt, const float* sn, const float* tn, const int64_t* corr,
                        int64_t n, int64_t m) {
    if (bad_corr(corr, n, m)) return -1.0;
    double sq = 0;
    int64_t c = 0;
    for (int64_t i = 0; i < n; ++i) {
        if (corr[i] == -1) continue;
        const float* s = src + 3 * i;
        const float* t = tgt + 3 * corr[i];
        const float* ns = sn + 3 * i;
        const float* nt = tn + 3 * corr[i];
        const float dot = ns[0] * nt[0] + ns[1] * nt[1] + ns[2] * nt[2];
        const float d = dot < 0.f ? -1.f : 1.f;
        const float r = (s[0] - t[0]) * (ns[0] * d + nt[0]) + (s[1] - t[1]) * (ns[1] * d + nt[1]) +
                        (s[2] - t[2]) * (ns[2] * d + nt[2]);
        sq += (double)(r * r);
        c += 1;
    }
    return c ? sqrt(sq / (double)c) : 0.0;
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

/* The loop of orc_icp_p2plane_f32 with the symmetric estimator.  Returns 0, -1 without memory, 1 for a singular
 * system (the reference raises). */
int orc_icp_sym_f32(const float* source, const float* source_normals, int64_t n, const float* target,
                    const float* target_normals, int64_t m, double max_corr_dist, const double init_T[16],
                    int max_iteration, double rel_fitness, double rel_rmse, int method, double scale, double shape,
                    int accumulate_f64, orc_icp_result* res, double* per_iter, int64_t* corr_out) {
    const size_t nn = (size_t)(n > 0 ? n : 1);
    float* src = (float*)malloc(nn * 3 * sizeof(float));
    float* sn = (float*)malloc(nn * 3 * sizeof(float));
    int64_t* corr = (int64_t*)malloc(nn * sizeof(int64_t));
    int32_t* idx = (int32_t*)malloc(nn * sizeof(int32_t));
    int32_t* cnt = (int32_t*)malloc(nn * sizeof(int32_t));
    float* d2 = (float*)malloc(nn * sizeof(float));
    int rc = 0;
    if (!src || !sn || !corr || !idx || !cnt || !d2) {
        rc = -1;
        goto done;
    }
    memcpy(src, source, (size_t)n * 3 * sizeof(float));
    memcpy(sn, source_normals, (size_t)n * 3 * sizeof(float));
    double T[16];
    memcpy(T, init_T, sizeof(T));
    orc_transform_points_f32(T, src, n);   /* Registration.cpp:398-404: PointCloud::Transform */
    orc_transform_normals_f32(T, sn, n);

    double fitness = 0, rmse = 0, prev_fitness = 0, prev_rmse = 0;
    int64_t count = 0;
    int converged = 0, it = 0;
    for (it = 0; it < max_iteration; ++it) {
        registration_result(src, n, target, m, max_corr_dist, idx, d2, cnt, corr, &fitness, &rmse, &count);
        if (count == 0) eye4(T);                       /* :51-60 */
        if (fitness <= 2.2250738585072014e-308) break; /* :300-306 */
        double U[16];
        if (orc_sym_transformation_f32(src, target, sn, target_normals, corr, n, m, method, scale, shape,
                                       accumulate_f64, U)) {
            rc = 1;
            goto done;
        }
        matmul4(U, T, T);                     /* :319 */
        orc_transform_points_f32(U, src, n);  /* :322 */
        orc_transform_normals_f32(U, sn, n);
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
    const int iterations = it;
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
    free(sn);
    free(corr);
    free(idx);
    free(cnt);
    free(d2);
    return rc;
}
