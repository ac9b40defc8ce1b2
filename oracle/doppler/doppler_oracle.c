/* CPU oracle of TransformationEstimationForDopplerICP and the ICP loop around it (test infrastructure).
 *
 * A restatement of the reference's CPU semantics, written from its description:
 *   - the host part of ComputePoseDopplerICP (t/pipelines/kernel/Registration.cpp:193-265): the kernels in force and
 *     outlier rejection switch on at their iterations; the pose of the accumulated transformation T
 *     (TransformationToPose: atan2 of T's rotation block, T's translation) in f64, cast to f32; w = -pose[0:3] / period
 *     and v = -pose[3:6] / period in f32.  R_S_to_V and r_v_to_s_in_V arrive in f32 (the caller inverts in f64).
 *   - PreComputeForDopplerICP (RegistrationImpl.h:525-541): v_s_in_S = R_S_to_V (v + w x r_v_to_s_in_V) in f32.
 *   - GetJacobianDopplerICP (RegistrationImpl.h:557-643): the predicted Doppler -(R_S_to_V d) . v_s_in_S and the error
 *     in f32, widened to f64; a rejected point counts with zero J and r; J_D = sqrt_ld / period [d x r ; -d],
 *     r_D = (float)(sqrt_ld * error); J_G and r_G of point-to-plane scaled by sqrt(1 - lambda).
 *   - ComputePoseDopplerICPKernelCPU (RegistrationCPU.cpp:336-400): 21 + 6 slots of J_G w_G J_G + J_D w_D J_D and
 *     J_G w_G r_G + J_D w_D r_D, [27] r_G^2 + r_D^2, [28] count; a serial reduction in f32 (the reference's TBB reduce
 *     with one range), or in f64 on request.
 *   - the loop of DoSingleScaleICPIterations (registration/Registration.cpp:293-358), with the rules of
 *     orc_icp_p2plane_f32 (../icp_oracle.c): the source's points move every iteration, its directions never. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle.h"

typedef struct {
    float R[9];          /* R_S_to_V, row-major */
    float r[3];          /* r_v_to_s_in_V */
    double period, lambda_doppler, threshold;
    int reject;
    int64_t min_reject, min_geo, min_dop;
    int method_g;
    double scale_g, shape_g;
    int method_d;
    double scale_d, shape_d;
} orc_dop_params;

/* TransformationToPose in f64 (TransformationConverterImpl.h:47-60 and TransformationConverter.cpp:163-187) */
void orc_dop_transformation_to_pose(const double T[16], double pose[6]) {
    const double sy = sqrt(T[0] * T[0] + T[4] * T[4]);
    if (!(sy < 1e-6)) {
        pose[0] = atan2(T[9], T[10]);
        pose[1] = atan2(-T[8], sy);
        pose[2] = atan2(T[4], T[0]);
    } else {
        pose[0] = atan2(-T[6], T[5]);
        pose[1] = atan2(-T[8], sy);
        pose[2] = 0.0;
    }
    pose[3] = T[3];
    pose[4] = T[7];
    pose[5] = T[11];
}

/* w_v_in_V and v_v_in_V of T (f32) */
void orc_dop_state(const double T[16], double period, float w[3], float v[3]) {
    double pose[6];
    orc_dop_transformation_to_pose(T, pose);
    const float p = (float)period;
    for (int j = 0; j < 3; ++j) {
        w[j] = -(float)pose[j] / p;
        v[j] = -(float)pose[3 + j] / p;
    }
}

/* PreComputeForDopplerICP */
void orc_dop_precompute(const float R[9], const float r[3], const float w[3], const float v[3], float out[3]) {
    const float c[3] = {w[1] * r[2] - w[2] * r[1] + v[0], w[2] * r[0] - w[0] * r[2] + v[1],
                        w[0] * r[1] - w[1] * r[0] + v[2]};
    for (int j = 0; j < 3; ++j) out[j] = R[3 * j] * c[0] + R[3 * j + 1] * c[1] + R[3 * j + 2] * c[2];
}

/* v_s_in_S for the accumulated transformation T */
void orc_dop_velocity(const orc_dop_params* p, const double T[16], float out[3]) {
    float w[3], v[3];
    orc_dop_state(T, p->period, w, v);
    orc_dop_precompute(p->R, p->r, w, v, out);
}

/* The 29 sums of iteration `iter` at the accumulated transformation T.  accumulate_f64 = 0: float accumulators. */
void orc_dop_sums_f32(const float* src, const float* dops, const float* dirs, const float* tgt, const float* nrm,
                      const int64_t* corr, int64_t n, const orc_dop_params* p, const double T[16], int64_t iter,
                      int accumulate_f64, double sums29[29]) {
    float vs[3];
    orc_dop_velocity(p, T, vs);
    const int reject = p->reject && iter >= p->min_reject;
    const int mg = iter >= p->min_geo ? p->method_g : 0, md = iter >= p->min_dop ? p->method_d : 0;
    const float slg = (float)sqrt(1.0 - (double)(float)p->lambda_doppler);
    const float sld = (float)sqrt(p->lambda_doppler);
    const float sld_dt = sld / (float)p->period;
    const float thr = (float)p->threshold;
    const float* R = p->R;
    const float* r = p->r;
    float a32[29];
    double a64[29];
    memset(a32, 0, sizeof(a32));
    memset(a64, 0, sizeof(a64));
    for (int64_t i = 0; i < n; ++i) {
        if (corr[i] == -1) continue;
        const float* d = dirs + 3 * i;
        float JG[6] = {0, 0, 0, 0, 0, 0}, JD[6] = {0, 0, 0, 0, 0, 0}, rG = 0.f, rD = 0.f;
        const float ds[3] = {R[0] * d[0] + R[1] * d[1] + R[2] * d[2], R[3] * d[0] + R[4] * d[1] + R[5] * d[2],
                             R[6] * d[0] + R[7] * d[1] + R[8] * d[2]};
        const float pred = -(ds[0] * vs[0] + ds[1] * vs[1] + ds[2] * vs[2]);
        const double err = (double)(dops[i] - pred);
        if (!(reject && fabs(err) > (double)thr)) {
            JD[0] = sld_dt * (d[1] * r[2] - d[2] * r[1]);
            JD[1] = sld_dt * (d[2] * r[0] - d[0] * r[2]);
            JD[2] = sld_dt * (d[0] * r[1] - d[1] * r[0]);
            JD[3] = sld_dt * -d[0];
            JD[4] = sld_dt * -d[1];
            JD[5] = sld_dt * -d[2];
            rD = (float)((double)sld * err);
            const float* s = src + 3 * i;
            const float* t = tgt + 3 * corr[i];
            const float* nt = nrm + 3 * corr[i];
            const float e = (s[0] - t[0]) * nt[0] + (s[1] - t[1]) * nt[1] + (s[2] - t[2]) * nt[2];
            JG[0] = slg * (-s[2] * nt[1] + s[1] * nt[2]);
            JG[1] = slg * (s[2] * nt[0] - s[0] * nt[2]);
            JG[2] = slg * (-s[1] * nt[0] + s[0] * nt[1]);
            JG[3] = slg * nt[0];
            JG[4] = slg * nt[1];
            JG[5] = slg * nt[2];
            rG = slg * e;
        }
        const float wG = orc_robust_weight_f32(mg, p->scale_g, p->shape_g, rG);
        const float wD = orc_robust_weight_f32(md, p->scale_d, p->shape_d, rD);
        int q = 0;
        for (int j = 0; j < 6; ++j) {
            for (int k = 0; k <= j; ++k, ++q) {
                const float v = JG[j] * wG * JG[k] + JD[j] * wD * JD[k];
                if (accumulate_f64) a64[q] += (double)v;
                else a32[q] += v;
            }
            const float v = JG[j] * wG * rG + JD[j] * wD * rD;
            if (accumulate_f64) a64[21 + j] += (double)v;
            else a32[21 + j] += v;
        }
        const float sq = rG * rG + rD * rD;
        if (accumulate_f64) {
            a64[27] += (double)sq;
            a64[28] += 1;
        } else {
            a32[27] += sq;
            a32[28] += 1;
        }
    }
    for (int k = 0; k < 29; ++k) sums29[k] = accumulate_f64 ? a64[k] : (double)a32[k];
}

/* ComputePoseDopplerICP + PoseToTransformation -> the update U.  Returns 0, or 1 for a singular system. */
int orc_dop_transformation_f32(const float* src, const float* dops, const float* dirs, const float* tgt,
                               const float* nrm, const int64_t* corr, int64_t n, const orc_dop_params* p,
                               const double T[16], int64_t iter, int accumulate_f64, double U[16]) {
    double sums[29], pose[6], residual;
    int count;
    orc_dop_sums_f32(src, dops, dirs, tgt, nrm, corr, n, p, T, iter, accumulate_f64, sums);
    if (orc_decode_and_solve_6x6(sums, pose, &residual, &count)) return 1;
    orc_pose_to_transformation(pose, U);
    return 0;
}

static void eye4(double T[16]) {
    for (int i = 0; i < 16; ++i) T[i] = (i % 5 == 0) ? 1.0 : 0.0;
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

/* The loop of orc_icp_p2plane_f32 with the Doppler estimator.  Returns 0, -1 without memory, 1 for a singular system
 * (the reference raises). */
int orc_icp_dop_f32(const float* source, const float* dops, const float* dirs, int64_t n, const float* target,
                    const float* target_normals, int64_t m, double max_corr_dist, const double init_T[16],
                    int max_iteration, double rel_fitness, double rel_rmse, const orc_dop_params* p, int accumulate_f64,
                    orc_icp_result* res, double* per_iter, int64_t* corr_out) {
    const size_t nn = (size_t)(n > 0 ? n : 1);
    float* src = (float*)malloc(nn * 3 * sizeof(float));
    int64_t* corr = (int64_t*)malloc(nn * sizeof(int64_t));
    int32_t* idx = (int32_t*)malloc(nn * sizeof(int32_t));
    int32_t* cnt = (int32_t*)malloc(nn * sizeof(int32_t));
    float* d2 = (float*)malloc(nn * sizeof(float));
    int rc = 0;
    if (!src || !corr || !idx || !cnt || !d2) {
        rc = -1;
        goto done;
    }
    memcpy(src, source, (size_t)n * 3 * sizeof(float));
    double T[16];
    memcpy(T, init_T, sizeof(T));
    orc_transform_points_f32(T, src, n);   /* Registration.cpp:398-404: PointCloud::Transform */

    double fitness = 0, rmse = 0, prev_fitness = 0, prev_rmse = 0;
    int64_t count = 0;
    int converged = 0, it = 0;
    for (it = 0; it < max_iteration; ++it) {
        registration_result(src, n, target, m, max_corr_dist, idx, d2, cnt, corr, &fitness, &rmse, &count);
        if (count == 0) eye4(T);                       /* :51-60 */
        if (fitness <= 2.2250738585072014e-308) break; /* :300-306 */
        double U[16];
        if (orc_dop_transformation_f32(src, dops, dirs, target, target_normals, corr, n, p, T, it, accumulate_f64, U)) {
            rc = 1;
            goto done;
        }
        matmul4(U, T, T);                     /* :319 */
        orc_transform_points_f32(U, src, n);  /* :322, the directions stay */
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
    free(corr);
    free(idx);
    free(cnt);
    free(d2);
    return rc;
}
