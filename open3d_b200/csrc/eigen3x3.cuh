// eigen3x3.cuh — t::geometry::kernel::pointcloud's fast 3x3 symmetric eigen solve (PointCloudImpl.h:746-1009) in f32
// with no FMA contraction, in the reference CPU build's operation order (DESIGN.md §4.13).  pointcloud.cu's normals
// and smooth.cu's moving-least-squares projection share it.
#pragma once

#include <cmath>

namespace o3db {

#define MUL(a, b) __fmul_rn(a, b)
#define ADD(a, b) __fadd_rn(a, b)
#define SUB(a, b) __fsub_rn(a, b)
#define DIV(a, b) __fdiv_rn(a, b)

__device__ __forceinline__ float dot3_rn(const float* a, const float* b) {
    return ADD(ADD(MUL(a[0], b[0]), MUL(a[1], b[1])), MUL(a[2], b[2]));
}

__device__ __forceinline__ void cross3_rn(const float* a, const float* b, float* c) {
    c[0] = SUB(MUL(a[1], b[2]), MUL(a[2], b[1]));
    c[1] = SUB(MUL(a[2], b[0]), MUL(a[0], b[2]));
    c[2] = SUB(MUL(a[0], b[1]), MUL(a[1], b[0]));
}

// ComputeEigenvector0 (PointCloudImpl.h:746-796)
__device__ __forceinline__ void eigenvector0(const float* A, float eval0, float* v) {
    const float r0[3] = {SUB(A[0], eval0), A[1], A[2]};
    const float r1[3] = {A[1], SUB(A[4], eval0), A[5]};
    const float r2[3] = {A[2], A[5], SUB(A[8], eval0)};
    float c01[3], c02[3], c12[3];
    cross3_rn(r0, r1, c01);
    cross3_rn(r0, r2, c02);
    cross3_rn(r1, r2, c12);
    const float d0 = dot3_rn(c01, c01), d1 = dot3_rn(c02, c02), d2 = dot3_rn(c12, c12);
    float dmax = d0;
    int imax = 0;
    if (d1 > dmax) {
        dmax = d1;
        imax = 1;
    }
    if (d2 > dmax) imax = 2;
    // selects on values, not on the arrays: a pointer into one of three arrays would put them in local memory
    const float s = __fsqrt_rn(imax == 0 ? d0 : (imax == 1 ? d1 : d2));
#pragma unroll
    for (int k = 0; k < 3; ++k) v[k] = DIV(imax == 0 ? c01[k] : (imax == 1 ? c02[k] : c12[k]), s);
}

// ComputeEigenvector1 (PointCloudImpl.h:798-873); upstream's 1.0 / sqrt(f32) rounds as the f32 division does
__device__ __forceinline__ void eigenvector1(const float* A, const float* e0, float eval1, float* v) {
    float U[3];
    if (fabsf(e0[0]) > fabsf(e0[1])) {
        const float inv = DIV(1.0f, __fsqrt_rn(ADD(MUL(e0[0], e0[0]), MUL(e0[2], e0[2]))));
        U[0] = MUL(-e0[2], inv);
        U[1] = 0.0f;
        U[2] = MUL(e0[0], inv);
    } else {
        const float inv = DIV(1.0f, __fsqrt_rn(ADD(MUL(e0[1], e0[1]), MUL(e0[2], e0[2]))));
        U[0] = 0.0f;
        U[1] = MUL(e0[2], inv);
        U[2] = MUL(-e0[1], inv);
    }
    float V[3], AU[3], AV[3];
    cross3_rn(e0, U, V);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        AU[r] = dot3_rn(A + 3 * r, U);
        AV[r] = dot3_rn(A + 3 * r, V);
    }
    float m00 = SUB(dot3_rn(U, AU), eval1), m01 = dot3_rn(U, AV), m11 = SUB(dot3_rn(V, AV), eval1);
    const float a00 = fabsf(m00), a01 = fabsf(m01), a11 = fabsf(m11);
    // the pair (first, second) that weights (U, V): (m01, m00) or (m11, m01), as upstream's two branches
    float wu, wv;
    bool ok;
    if (a00 >= a11) {
        ok = (a00 < a01 ? a01 : a00) > 0;   // std::max
        if (a00 >= a01) {
            m01 = DIV(m01, m00);
            m00 = DIV(1.0f, __fsqrt_rn(ADD(1.0f, MUL(m01, m01))));
            m01 = MUL(m01, m00);
        } else {
            m00 = DIV(m00, m01);
            m01 = DIV(1.0f, __fsqrt_rn(ADD(1.0f, MUL(m00, m00))));
            m00 = MUL(m00, m01);
        }
        wu = m01;
        wv = m00;
    } else {
        ok = (a11 < a01 ? a01 : a11) > 0;
        if (a11 >= a01) {
            m01 = DIV(m01, m11);
            m11 = DIV(1.0f, __fsqrt_rn(ADD(1.0f, MUL(m01, m01))));
            m01 = MUL(m01, m11);
        } else {
            m11 = DIV(m11, m01);
            m01 = DIV(1.0f, __fsqrt_rn(ADD(1.0f, MUL(m11, m11))));
            m11 = MUL(m11, m01);
        }
        wu = m11;
        wv = m01;
    }
    if (!ok) {
        v[0] = U[0];
        v[1] = U[1];
        v[2] = U[2];
        return;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) v[k] = SUB(MUL(wu, U[k]), MUL(wv, V[k]));
}

// EstimatePointWiseNormalsWithFastEigen3x3<float> (PointCloudImpl.h:875-1009)
__device__ __forceinline__ void normal_from_covariance(const float* cov, float* out) {
    float max_coeff = cov[0];
#pragma unroll
    for (int i = 1; i < 9; ++i)
        if (max_coeff < cov[i]) max_coeff = cov[i];
    if (max_coeff == 0) {
        out[0] = out[1] = out[2] = 0.0f;
        return;
    }
    float A[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) A[i] = DIV(cov[i], max_coeff);
    const float norm = ADD(ADD(MUL(A[1], A[1]), MUL(A[2], A[2])), MUL(A[5], A[5]));
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
    const float q = (float)__ddiv_rn((double)ADD(ADD(A[0], A[4]), A[8]), 3.0);
    const float b00 = SUB(A[0], q), b11 = SUB(A[4], q), b22 = SUB(A[8], q);
    const double ss = (double)ADD(ADD(MUL(b00, b00), MUL(b11, b11)), MUL(b22, b22));
    const float p = (float)__dsqrt_rn(__ddiv_rn(__dadd_rn(ss, __dmul_rn((double)norm, 2.0)), 6.0));
    const float c00 = SUB(MUL(b11, b22), MUL(A[5], A[5]));
    const float c01 = SUB(MUL(A[1], b22), MUL(A[5], A[2]));
    const float c02 = SUB(MUL(A[1], A[5]), MUL(b11, A[2]));
    const float det = DIV(ADD(SUB(MUL(b00, c00), MUL(A[1], c01)), MUL(A[2], c02)), MUL(MUL(p, p), p));
    float half_det = MUL(det, 0.5f);                    // exact, as upstream's f64 product rounded to f32
    half_det = half_det < -1.0f ? -1.0f : half_det;     // std::max, then std::min: a NaN passes through
    half_det = 1.0f < half_det ? 1.0f : half_det;
    const float angle = (float)__ddiv_rn((double)(float)acos((double)half_det), 3.0);
    const float two_thirds_pi = (float)2.09439510239319549;   // upstream's double literal
    const float beta2 = MUL((float)cos((double)angle), 2.0f);
    const float beta0 = MUL((float)cos((double)ADD(angle, two_thirds_pi)), 2.0f);
    const float beta1 = -ADD(beta0, beta2);
    const float eval0 = ADD(q, MUL(p, beta0)), eval1 = ADD(q, MUL(p, beta1)), eval2 = ADD(q, MUL(p, beta2));
    float e0[3], e1[3];
    if (half_det >= 0) {
        eigenvector0(A, eval2, e0);   // upstream's evec2
        if (eval2 < eval0 && eval2 < eval1) {
            out[0] = e0[0];
            out[1] = e0[1];
            out[2] = e0[2];
            return;
        }
        eigenvector1(A, e0, eval1, e1);
        if (eval1 < eval0 && eval1 < eval2) {
            out[0] = e1[0];
            out[1] = e1[1];
            out[2] = e1[2];
            return;
        }
        cross3_rn(e1, e0, out);
    } else {
        eigenvector0(A, eval0, e0);
        if (eval0 < eval1 && eval0 < eval2) {
            out[0] = e0[0];
            out[1] = e0[1];
            out[2] = e0[2];
            return;
        }
        eigenvector1(A, e0, eval1, e1);
        if (eval1 < eval0 && eval1 < eval2) {
            out[0] = e1[0];
            out[1] = e1[1];
            out[2] = e1[2];
            return;
        }
        cross3_rn(e0, e1, out);
    }
}

#undef MUL
#undef ADD
#undef SUB
#undef DIV

}  // namespace o3db
