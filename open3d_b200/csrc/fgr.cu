// fgr.cu — Fast Global Registration on the device: pipelines::registration::
// FastGlobalRegistrationBasedOnCorrespondence and FastGlobalRegistrationBasedOnFeatureMatching
// (pipelines/registration/FastGlobalRegistration.cpp:68-395), run as upstream runs them on one thread.
// DESIGN.md §4.26.
//
// f64 throughout, every op rounded on its own (this file is compiled with -fmad=false), in the orders DESIGN.md §4.26
// states for Eigen's:
//   normalise   fgr_check_kernel: the input checks; fgr_mean_kernel: each cloud's mean, one thread per axis, the serial
//               sum in point order divided by n; fgr_scale_kernel: the largest norm of a centred point;
//   tuples      AdvancedMatching in batches of kFgrBatch trials drawn on the host: fgr_tuple_kernel flags each trial,
//               a scan counts the passing ones, fgr_stop_kernel finds the trial whose running count reaches
//               maximum_tuple_count, fgr_tuple_compact_kernel lists the passing trials' pairs in trial order;
//   optimise    fgr_optimize_kernel: OptimizePairwiseRegistration in one CTA, all iterations in one launch, then
//               GetTransformationOriginalScale and the 4x4 inverse;
//   evaluate    fgr_transform_kernel: EvaluateRegistration's transformed source; fgr_eval_kernel: the nearest target
//               point of each, the tile's count and sum of d^2; fgr_sum_kernel: the tiles in order.
// The call synchronises the stream 3 times (the checks and the normalisation, the target index, the result), once per
// batch of trials, and twice more in the feature matching.
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "common.cuh"
#include "grid.cuh"
#include "scan.cuh"

namespace o3db {

constexpr int kFgrT = 256;          // threads per CTA of the elementwise kernels and of the optimisation
constexpr int kFgrTile = 128;       // source points per tile of the evaluation sums
constexpr int kFgrBatch = 16384;    // tuple trials drawn per batch
constexpr size_t kFgrSmem = 220 * 1024;   // the optimisation's pair staging (7 doubles a pair), when it fits

// Device state: the result.
struct FgrState {
    double T[16];    // row-major
    double fitness, rmse;
};

struct FgrArgs {
    const float* src;        // [n,3]
    const float* tgt;        // [m,3]
    int64_t n, m;
    double mean_s[3], mean_t[3];
    double scale_global;
    const int64_t* pairs;    // [np,2] (source row, target row): the optimiser's input
    int np;
    int iterations;
    int decrease_mu;
    double max_dist, division;
    double* buf;             // [3 np] p, then [7 np] q, r, s when they do not fit in shared memory; SoA
    int staged;              // 1: q, r and s are in the dynamic shared memory
    double r2;
    RadiusView view;
    int tiles;
    int* part_cnt;           // [tiles]
    double* part_err;        // [tiles]
    FgrState* state;
    const double* xs;        // [n,3]: the transformed source
    int64_t* out;            // [n]
};

__device__ __forceinline__ void load3(const float* p, int64_t i, double& x, double& y, double& z) {
    x = (double)__ldg(p + 3 * i);
    y = (double)__ldg(p + 3 * i + 1);
    z = (double)__ldg(p + 3 * i + 2);
}

// Eigen's norm / dot / squaredNorm of three, in the stated order ((a0 b0 + a1 b1) + a2 b2).
__device__ __forceinline__ double sq3(double x, double y, double z) { return (x * x + y * y) + z * z; }

// Input checks: bad[0] |= 1 for a non-finite source coordinate, 2 for a non-finite target coordinate; bad[1] = 1 for a
// pair outside [0, n) x [0, m).
__global__ void __launch_bounds__(kFgrT) fgr_check_kernel(const float* src, int64_t n, const float* tgt, int64_t m,
                                                          const int64_t* corres, int64_t K, unsigned* bad) {
    const int64_t i = blockIdx.x * (int64_t)kFgrT + threadIdx.x;
    if (i < n) flag_nonfinite(src, i, bad);
    if (i < m && (!isfinite(tgt[3 * i]) || !isfinite(tgt[3 * i + 1]) || !isfinite(tgt[3 * i + 2]))) atomicOr(bad, 2u);
    if (corres && i < K) {
        const int64_t s = corres[2 * i], t = corres[2 * i + 1];
        if (s < 0 || s >= n || t < 0 || t >= m) atomicOr(bad + 1, 1u);
    }
}

// NormalizePointCloud's means (FastGlobalRegistration.cpp:157-162): thread c < 3 sums the source's axis c, thread
// 3 + c the target's, mean = mean + p in point order from 0, then mean / n.
__global__ void __launch_bounds__(32) fgr_mean_kernel(const float* src, int64_t n, const float* tgt, int64_t m,
                                                      double* mean /* [6] */) {
    const int c = threadIdx.x;
    if (c >= 6) return;
    const float* p = c < 3 ? src + c : tgt + (c - 3);
    const int64_t k = c < 3 ? n : m;
    double s = 0.0;
    for (int64_t i = 0; i < k; ++i) s = s + (double)__ldg(p + 3 * i);
    mean[c] = s / (double)(int)k;
}

// The largest (p - mean).norm() over both clouds (:167-173): the max is exact in any order.  scale holds the bits of a
// non-negative double, which order as unsigned integers.
__global__ void __launch_bounds__(kFgrT) fgr_scale_kernel(const float* src, int64_t n, const float* tgt, int64_t m,
                                                          const double* mean, unsigned long long* scale) {
    const int64_t i = blockIdx.x * (int64_t)kFgrT + threadIdx.x;
    double v = 0.0;
    if (i < n + m) {
        const bool s = i < n;
        double x, y, z;
        load3(s ? src : tgt, s ? i : i - n, x, y, z);
        const double* mu = mean + (s ? 0 : 3);
        v = sqrt(sq3(x - mu[0], y - mu[1], z - mu[2]));
    }
    for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0 && v > 0.0) atomicMax(scale, (unsigned long long)__double_as_longlong(v));
}

// AdvancedMatching's trial t of the batch (:99-137): three pairs of the draws, the three edge lengths of each cloud,
// pass = li*scale < lj < li/scale for all three.  a / b are the first and second cloud of the pairs (the target and
// the source in the swapped branch of the feature call).
__global__ void __launch_bounds__(kFgrT) fgr_tuple_kernel(const float* a, const float* b, const int64_t* corres,
                                                          const int* draws, int hb, double scale, unsigned* pass) {
    const int t = blockIdx.x * kFgrT + threadIdx.x;
    if (t >= hb) return;
    const int64_t r0 = draws[3 * t], r1 = draws[3 * t + 1], r2 = draws[3 * t + 2];
    double i0x, i0y, i0z, i1x, i1y, i1z, i2x, i2y, i2z, j0x, j0y, j0z, j1x, j1y, j1z, j2x, j2y, j2z;
    load3(a, corres[2 * r0], i0x, i0y, i0z);
    load3(a, corres[2 * r1], i1x, i1y, i1z);
    load3(a, corres[2 * r2], i2x, i2y, i2z);
    load3(b, corres[2 * r0 + 1], j0x, j0y, j0z);
    load3(b, corres[2 * r1 + 1], j1x, j1y, j1z);
    load3(b, corres[2 * r2 + 1], j2x, j2y, j2z);
    const double li0 = sqrt(sq3(i0x - i1x, i0y - i1y, i0z - i1z));
    const double li1 = sqrt(sq3(i1x - i2x, i1y - i2y, i1z - i2z));
    const double li2 = sqrt(sq3(i2x - i0x, i2y - i0y, i2z - i0z));
    const double lj0 = sqrt(sq3(j0x - j1x, j0y - j1y, j0z - j1z));
    const double lj1 = sqrt(sq3(j1x - j2x, j1y - j2y, j1z - j2z));
    const double lj2 = sqrt(sq3(j2x - j0x, j2y - j0y, j2z - j0z));
    pass[t] = (li0 * scale < lj0) && (lj0 < li0 / scale) && (li1 * scale < lj1) && (lj1 < li1 / scale) &&
              (li2 * scale < lj2) && (lj2 < li2 / scale);
}

// After the scan: stop[0] = the first trial t after which the running count cnt0 + scan[t + 1] has reached maxc (the
// break test runs after every trial, passing or not), stop[1] = scan[t + 1], the batch's passing trials up to it.
// The count is monotone in t, so exactly one thread writes.
__global__ void __launch_bounds__(kFgrT) fgr_stop_kernel(const unsigned* scan, int hb, long long cnt0, long long maxc,
                                                         int* stop) {
    const int t = blockIdx.x * kFgrT + threadIdx.x;
    if (t >= hb) return;
    if (cnt0 + (long long)scan[t + 1] >= maxc && (t == 0 || cnt0 + (long long)scan[t] < maxc)) {
        stop[0] = t;
        stop[1] = (int)scan[t + 1];
    }
}

// The passing trials up to and including stop[0] (all of them when it is hb): their three pairs at 3 (cnt0 + scan[t]),
// as (first, second) or swapped back to (source, target).
__global__ void __launch_bounds__(kFgrT) fgr_tuple_compact_kernel(const int64_t* corres, const int* draws,
                                                                  const unsigned* scan, int hb, const int* stop,
                                                                  long long cnt0, int swap, int64_t* out) {
    const int t = blockIdx.x * kFgrT + threadIdx.x;
    if (t >= hb || t > *stop || scan[t + 1] == scan[t]) return;
    int64_t* o = out + 6 * (cnt0 + (long long)scan[t]);
    for (int k = 0; k < 3; ++k) {
        const int64_t r = draws[3 * t + k];
        o[2 * k] = corres[2 * r + swap];
        o[2 * k + 1] = corres[2 * r + 1 - swap];
    }
}

// The 24 structurally non-zero entries of JTJ, (row, column), and for each its J factors per Jacobian row x, y, z of
// OptimizePairwiseRegistration (:226-251):
//   row x: J1 = -q2, J2 = q1, J3 = -1;   row y: J0 = q2, J2 = -q0, J4 = -1;   row z: J0 = -q1, J1 = q0, J5 = -1.
// A factor is coded as 1 + (axis of q, or 3 for the constant 1), negative for a negated factor, 0 where the entry of J
// is structurally zero.
__constant__ signed char c_jfac[3][6] = {{0, -3, 2, -4, 0, 0}, {3, 0, -1, 0, -4, 0}, {-2, 1, 0, 0, 0, -4}};
__constant__ unsigned char c_entry[24][2] = {{1, 1}, {1, 2}, {1, 3}, {2, 1}, {2, 2}, {2, 3}, {3, 1}, {3, 2},
                                             {3, 3}, {0, 0}, {0, 2}, {0, 4}, {2, 0}, {2, 4}, {4, 0}, {4, 2},
                                             {4, 4}, {0, 1}, {0, 5}, {1, 0}, {1, 5}, {5, 0}, {5, 1}, {5, 5}};

// Row j of M (4x4, row-major) times (x, y, z, 1): ((M_j0 x + M_j1 y) + M_j2 z) + M_j3 * 1.
__device__ __forceinline__ double row4(const double* M, int j, double x, double y, double z) {
    return ((M[4 * j] * x + M[4 * j + 1] * y) + M[4 * j + 2] * z) + M[4 * j + 3] * 1.0;
}

// Eigen's LDLT of A (6x6 in s_A, row-major, only the lower triangle read) with diagonal pivoting, then its solve of
// A x = b in place in s_b (DESIGN.md §4.26).  One thread; the arrays are shared memory, indexed by pivot.
__device__ void ldlt_solve6(double* A, double* b, int* tr, double* tmp) {
    for (int k = 0; k < 6; ++k) {
        int p = k;   // the largest |diagonal| of the trailing corner, the first of equal ones
        double big = fabs(A[7 * k]);
        for (int i = k + 1; i < 6; ++i)
            if (fabs(A[7 * i]) > big) {
                big = fabs(A[7 * i]);
                p = i;
            }
        tr[k] = p;
        if (p != k) {
            for (int j = 0; j < k; ++j) {   // row k and row p, columns < k
                const double t = A[6 * k + j];
                A[6 * k + j] = A[6 * p + j];
                A[6 * p + j] = t;
            }
            for (int i = p + 1; i < 6; ++i) {   // column k and column p, rows > p
                const double t = A[6 * i + k];
                A[6 * i + k] = A[6 * i + p];
                A[6 * i + p] = t;
            }
            const double t = A[7 * k];
            A[7 * k] = A[7 * p];
            A[7 * p] = t;
            for (int i = k + 1; i < p; ++i) {
                const double u = A[6 * i + k];
                A[6 * i + k] = A[6 * p + i];
                A[6 * p + i] = u;
            }
        }
        if (k > 0) {
            for (int j = 0; j < k; ++j) tmp[j] = A[7 * j] * A[6 * k + j];
            double d = A[6 * k] * tmp[0];
            for (int j = 1; j < k; ++j) d = d + A[6 * k + j] * tmp[j];
            A[7 * k] = A[7 * k] - d;
            for (int i = k + 1; i < 6; ++i) {
                double e = A[6 * i] * tmp[0];
                for (int j = 1; j < k; ++j) e = e + A[6 * i + j] * tmp[j];
                A[6 * i + k] = A[6 * i + k] - e;
            }
        }
        const double akk = A[7 * k];
        if (k == 0 && !(fabs(akk) > 0.0)) {   // an all-zero diagonal: nothing more to factor
            for (int j = 0; j < 6; ++j) tr[j] = j;
            break;
        }
        if (fabs(akk) > 0.0)
            for (int i = k + 1; i < 6; ++i) A[6 * i + k] = A[6 * i + k] / akk;
    }
    for (int k = 0; k < 6; ++k) {   // P b
        const int p = tr[k];
        const double t = b[k];
        b[k] = b[p];
        b[p] = t;
    }
    for (int i = 0; i < 6; ++i)   // L^-1, column by column
        for (int j = i + 1; j < 6; ++j) b[j] = b[j] - A[6 * j + i] * b[i];
    for (int i = 0; i < 6; ++i) {   // D^+: pivots not above 1 / DBL_MAX give 0
        const double d = A[7 * i];
        b[i] = fabs(d) > 1.0 / DBL_MAX ? b[i] / d : 0.0;
    }
    for (int i = 5; i >= 0; --i)   // L^-T, column by column from the last
        for (int j = 0; j < i; ++j) b[j] = b[j] - A[6 * i + j] * b[i];
    for (int k = 5; k >= 0; --k) {   // P^T
        const int p = tr[k];
        const double t = b[k];
        b[k] = b[p];
        b[p] = t;
    }
}

// The stated sine and cosine (DESIGN.md §4.26), the same ops in the C oracle and the shim's Eigen: k = rint(x 2/pi),
// r = (x - k P1) - k P2 with pi/2 = P1 + P2 (P1 has 33 bits, so k P1 is exact for |k| < 2^20), then the Taylor
// polynomials of sin and cos on [-pi/4, pi/4] to x^17 and x^18 by Horner, by the quadrant k mod 4.
__device__ __forceinline__ double fgr_sincos(double x, int want_cos) {
    const double P1 = 1.57079632673412561417e+00, P2 = 6.07710050650619224932e-11;
    const double k = rint(x * 0.63661977236758134308);
    const double r = (x - k * P1) - k * P2;
    const double z = r * r;
    const double ps = -1.0 / 6.0 + z * (1.0 / 120.0 + z * (-1.0 / 5040.0 + z * (1.0 / 362880.0 + z * (-1.0 / 39916800.0 +
                      z * (1.0 / 6227020800.0 + z * (-1.0 / 1307674368000.0 + z * (1.0 / 355687428096000.0)))))));
    const double pc = -0.5 + z * (1.0 / 24.0 + z * (-1.0 / 720.0 + z * (1.0 / 40320.0 + z * (-1.0 / 3628800.0 +
                      z * (1.0 / 479001600.0 + z * (-1.0 / 87178291200.0 + z * (1.0 / 20922789888000.0 +
                      z * (-1.0 / 6402373705728000.0))))))));
    const double sv = r + r * (z * ps), cv = 1.0 + z * pc;
    const int q = ((int)k + want_cos) & 3;
    return q == 0 ? sv : (q == 1 ? cv : (q == 2 ? -sv : -cv));
}
__device__ __forceinline__ double fgr_sin(double x) { return fgr_sincos(x, 0); }
__device__ __forceinline__ double fgr_cos(double x) { return fgr_sincos(x, 1); }

// Quaternion product a * b (w, x, y, z), Eigen's scalar formula left to right.
__device__ __forceinline__ void qmul(const double* a, const double* b, double* o) {
    o[0] = ((a[0] * b[0] - a[1] * b[1]) - a[2] * b[2]) - a[3] * b[3];
    o[1] = ((a[0] * b[1] + a[1] * b[0]) + a[2] * b[3]) - a[3] * b[2];
    o[2] = ((a[0] * b[2] + a[2] * b[0]) + a[3] * b[1]) - a[1] * b[3];
    o[3] = ((a[0] * b[3] + a[3] * b[0]) + a[1] * b[2]) - a[2] * b[1];
}

// TransformVector6dToMatrix4d (utility/Eigen.cpp:79-89): (AngleAxis(x2, Z) * AngleAxis(x1, Y)) * AngleAxis(x0, X) as
// quaternions (w = cos(a/2), v = sin(a/2) axis), then toRotationMatrix; t = x3..5; row 3 = (0, 0, 0, 1).
__device__ __forceinline__ void vec6_to_mat4(const double* x, double* D) {
    double qz[4], qy[4], qx[4], q1[4], q[4];
    const double hz = 0.5 * x[2], hy = 0.5 * x[1], hx = 0.5 * x[0];
    const double sz = fgr_sin(hz), sy = fgr_sin(hy), sx = fgr_sin(hx);
    qz[0] = fgr_cos(hz), qz[1] = sz * 0.0, qz[2] = sz * 0.0, qz[3] = sz * 1.0;
    qy[0] = fgr_cos(hy), qy[1] = sy * 0.0, qy[2] = sy * 1.0, qy[3] = sy * 0.0;
    qx[0] = fgr_cos(hx), qx[1] = sx * 1.0, qx[2] = sx * 0.0, qx[3] = sx * 0.0;
    qmul(qz, qy, q1);
    qmul(q1, qx, q);
    const double tx = 2.0 * q[1], ty = 2.0 * q[2], tz = 2.0 * q[3];
    const double twx = tx * q[0], twy = ty * q[0], twz = tz * q[0];
    const double txx = tx * q[1], txy = ty * q[1], txz = tz * q[1];
    const double tyy = ty * q[2], tyz = tz * q[2], tzz = tz * q[3];
    D[0] = 1.0 - (tyy + tzz), D[1] = txy - twz, D[2] = txz + twy, D[3] = x[3];
    D[4] = txy + twz, D[5] = 1.0 - (txx + tzz), D[6] = tyz - twx, D[7] = x[4];
    D[8] = txz - twy, D[9] = tyz + twx, D[10] = 1.0 - (txx + tyy), D[11] = x[5];
    D[12] = 0.0, D[13] = 0.0, D[14] = 0.0, D[15] = 1.0;
}

// det of the 3x3 minor of M (4x4 row-major) on rows r0 < r1 < r2 and columns c0 < c1 < c2:
// (a (e i - f h) - b (d i - f g)) + c (d h - e g).
__device__ __forceinline__ double det3(const double* M, int r0, int r1, int r2, int c0, int c1, int c2) {
    const double a = M[4 * r0 + c0], b = M[4 * r0 + c1], c = M[4 * r0 + c2];
    const double d = M[4 * r1 + c0], e = M[4 * r1 + c1], f = M[4 * r1 + c2];
    const double g = M[4 * r2 + c0], h = M[4 * r2 + c1], i = M[4 * r2 + c2];
    return (a * (e * i - f * h) - b * (d * i - f * g)) + c * (d * h - e * g);
}

// Matrix4d::inverse, as stated: cofactors C_ij = (-1)^(i+j) det3(M without row i, column j), det = ((M_00 C_00 +
// M_10 C_10) + M_20 C_20) + M_30 C_30, inv_ij = C_ji / det.  M and out are distinct shared arrays.
__device__ void inverse4(const double* M, double* out) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            const int r0 = i == 0 ? 1 : 0, r1 = i <= 1 ? 2 : 1, r2 = i <= 2 ? 3 : 2;
            const int c0 = j == 0 ? 1 : 0, c1 = j <= 1 ? 2 : 1, c2 = j <= 2 ? 3 : 2;
            const double m = det3(M, r0, r1, r2, c0, c1, c2);
            out[4 * j + i] = (i + j) & 1 ? -m : m;   // the transpose of the cofactors
        }
    const double det = ((M[0] * out[0] + M[4] * out[1]) + M[8] * out[2]) + M[12] * out[3];
    for (int k = 0; k < 16; ++k) out[k] = out[k] / det;
}

// OptimizePairwiseRegistration (:190-264), GetTransformationOriginalScale (:268-282) and the inverse, one CTA.
// Every iteration: the threads move each pair's target point by the last delta (dividing by w, which is 1) and compute
// rpq and s; warp 0 accumulates JTJ and JTr, each lane one entry, walking the pairs in order; thread 0 solves and
// updates trans and par.
__global__ void __launch_bounds__(kFgrT) fgr_optimize_kernel(FgrArgs a) {
    extern __shared__ double s_pairs[];
    __shared__ double s_A[36], s_b[6], s_ld[6], s_delta[16], s_trans[16], s_tmp[16], s_par, s_const[2];
    __shared__ int s_tr[6];
    const int tid = threadIdx.x, np = a.np;
    double* base = a.staged ? s_pairs : a.buf + 3 * (size_t)np;   // q, r, s: shared memory while they fit
    double *px = a.buf, *py = a.buf + np, *pz = a.buf + 2 * (size_t)np;
    double *qx = base, *qy = base + np, *qz = base + 2 * (size_t)np, *rx = base + 3 * (size_t)np,
           *ry = base + 4 * (size_t)np, *rz = base + 5 * (size_t)np, *sw = base + 6 * (size_t)np;
    const double sg = a.scale_global;
    const int iters = np < 10 ? 0 : a.iterations;   // fewer than 10 pairs: the identity
    for (int c = tid; c < (iters > 0 ? np : 0); c += kFgrT) {   // the normalised points: (p - mean) / scale_global
        double x, y, z;
        load3(a.src, a.pairs[2 * c], x, y, z);
        px[c] = (x - a.mean_s[0]) / sg;
        py[c] = (y - a.mean_s[1]) / sg;
        pz[c] = (z - a.mean_s[2]) / sg;
        load3(a.tgt, a.pairs[2 * c + 1], x, y, z);
        qx[c] = (x - a.mean_t[0]) / sg;
        qy[c] = (y - a.mean_t[1]) / sg;
        qz[c] = (z - a.mean_t[2]) / sg;
    }
    if (tid < 16) s_trans[tid] = tid % 5 == 0 ? 1.0 : 0.0;
    if (tid == 0) {
        s_par = sg;   // upstream starts par at scale_global, not at scale_start
        s_const[0] = 0.0;
        s_const[1] = 1.0;
    }
    // Lane l < 30 of warp 0 owns JTJ entry c_entry[l] (l < 24) or JTr entry l - 24.  For Jacobian row k its term is
    // (J_a J_b) s, or (J_a r_k) s, as upstream's dense update adds it; J_a = sign * |J_a| and the product's sign is
    // exact, so the lane reads |J_a| and |J_b| (or r_k) from the array each names, with stride 0 for the constants 0 and
    // 1, and multiplies by the sign.  A structurally zero term is +-0, and adding it changes no sum: an accumulator
    // that starts at +0 never becomes -0.
    const double* fa[3] = {s_const, s_const, s_const};
    const double* fb[3] = {s_const, s_const, s_const};
    int sa[3] = {0, 0, 0}, sb[3] = {0, 0, 0};
    double sgn[3] = {1.0, 1.0, 1.0};
    if (tid < 30) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int ca = c_jfac[k][tid < 24 ? c_entry[tid][0] : tid - 24];
            const int cb = tid < 24 ? c_jfac[k][c_entry[tid][1]] : 0;
            const int ia = ca < 0 ? -ca : ca, ib = cb < 0 ? -cb : cb;
            fa[k] = ia == 0 ? s_const : (ia == 1 ? qx : (ia == 2 ? qy : (ia == 3 ? qz : s_const + 1)));
            sa[k] = ia >= 1 && ia <= 3;
            if (tid < 24) {
                fb[k] = ib == 0 ? s_const : (ib == 1 ? qx : (ib == 2 ? qy : (ib == 3 ? qz : s_const + 1)));
                sb[k] = ib >= 1 && ib <= 3;
            } else {
                fb[k] = k == 0 ? rx : (k == 1 ? ry : rz);
                sb[k] = 1;
            }
            sgn[k] = (ca < 0) != (cb < 0) ? -1.0 : 1.0;
        }
    }
    for (int itr = 0; itr < iters; ++itr) {
        __syncthreads();
        const double par = s_par;
        for (int c = tid; c < np; c += kFgrT) {
            double x = qx[c], y = qy[c], z = qz[c];
            if (itr > 0) {   // point_cloud_copy_j.Transform(delta) of the last iteration
                const double w = row4(s_delta, 3, x, y, z);
                const double ox = row4(s_delta, 0, x, y, z), oy = row4(s_delta, 1, x, y, z),
                             oz = row4(s_delta, 2, x, y, z);
                x = ox / w, y = oy / w, z = oz / w;
                qx[c] = x, qy[c] = y, qz[c] = z;
            }
            const double dx = px[c] - x, dy = py[c] - y, dz = pz[c] - z;   // rpq = p - q
            rx[c] = dx, ry[c] = dy, rz[c] = dz;
            const double t = par / (sq3(dx, dy, dz) + par);
            sw[c] = t * t;
        }
        __syncthreads();
        if (tid < 32) {
            double acc = 0.0;
#pragma unroll 4
            for (int c = 0; c < np; ++c) {
                const double s = sw[c];
                acc = acc + ((fa[0][c * sa[0]] * fb[0][c * sb[0]]) * sgn[0]) * s;
                acc = acc + ((fa[1][c * sa[1]] * fb[1][c * sb[1]]) * sgn[1]) * s;
                acc = acc + ((fa[2][c * sa[2]] * fb[2][c * sb[2]]) * sgn[2]) * s;
            }
            if (tid < 24)
                s_A[6 * c_entry[tid][0] + c_entry[tid][1]] = acc;
            else if (tid < 30)
                s_b[tid - 24] = acc;
            for (int k = tid; k < 36; k += 32)   // the structurally zero entries stay +0
                if (!(c_jfac[0][k / 6] && c_jfac[0][k % 6]) && !(c_jfac[1][k / 6] && c_jfac[1][k % 6]) &&
                    !(c_jfac[2][k / 6] && c_jfac[2][k % 6]))
                    s_A[k] = 0.0;
        }
        __syncthreads();
        if (tid == 0) {   // x = (-JTJ).ldlt().solve(JTr); delta; trans = delta * trans; par
            for (int k = 0; k < 36; ++k) s_A[k] = -s_A[k];
            ldlt_solve6(s_A, s_b, s_tr, s_ld);
            vec6_to_mat4(s_b, s_delta);
            for (int r = 0; r < 4; ++r)
                for (int c = 0; c < 4; ++c)
                    s_tmp[4 * r + c] = ((s_delta[4 * r] * s_trans[c] + s_delta[4 * r + 1] * s_trans[4 + c]) +
                                        s_delta[4 * r + 2] * s_trans[8 + c]) +
                                       s_delta[4 * r + 3] * s_trans[12 + c];
            for (int k = 0; k < 16; ++k) s_trans[k] = s_tmp[k];
            if (a.decrease_mu && itr % 4 == 0 && s_par > a.max_dist) s_par = s_par / a.division;
        }
    }
    __syncthreads();
    if (tid != 0) return;
    // GetTransformationOriginalScale: [R, -R mean_t + t scale_global + mean_s; 0 0 0 1], then its inverse
    for (int k = 0; k < 16; ++k) s_tmp[k] = 0.0;
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) s_tmp[4 * r + c] = s_trans[4 * r + c];
        const double rm = ((-s_trans[4 * r] * a.mean_t[0] + -s_trans[4 * r + 1] * a.mean_t[1]) +
                           -s_trans[4 * r + 2] * a.mean_t[2]);
        s_tmp[4 * r + 3] = (rm + s_trans[4 * r + 3] * sg) + a.mean_s[r];
    }
    s_tmp[15] = 1.0;
    inverse4(s_tmp, a.state->T);
}

// Eigen's isIdentity() at its default precision 1e-12: |T_ii - 1| <= min(|T_ii|, 1) 1e-12, |T_ij| <= 1e-12.
__device__ __forceinline__ bool approx_identity(const double* T) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            const double v = T[4 * i + j];
            if (i == j ? !(fabs(v - 1.0) <= fmin(fabs(v), 1.0) * 1e-12) : !(fabs(v) <= 1e-12)) return false;
        }
    return true;
}

// EvaluateRegistration's source (Registration.cpp:134-137): xs[i] = source point i transformed unless T is the
// identity (Transform: p = (T (x, y, z, 1)).head<3>() / w).  Its own kernel: the division's slow path is a call, which
// would cost the search kernel a stack frame.
__global__ void __launch_bounds__(kFgrT) fgr_transform_kernel(const float* src, int64_t n, const FgrState* state,
                                                              double* xs) {
    const int64_t i = blockIdx.x * (int64_t)kFgrT + threadIdx.x;
    if (i >= n) return;
    const double* T = state->T;
    double px, py, pz;
    load3(src, i, px, py, pz);
    if (!approx_identity(T)) {
        const double w = row4(T, 3, px, py, pz);
        const double ox = row4(T, 0, px, py, pz), oy = row4(T, 1, px, py, pz), oz = row4(T, 2, px, py, pz);
        px = ox / w, py = oy / w, pz = oz / w;
    }
    xs[3 * i] = px;
    xs[3 * i + 1] = py;
    xs[3 * i + 2] = pz;
}

// The nearest target point of the transformed source point i: ((dx^2 + dy^2) + dz^2) in f64, a match when
// d^2 < r^2, ties to the lowest index; -1 for none.  The cells are binned from the query rounded to f32, as in
// ransac.cu.
__device__ __forceinline__ int nearest(const FgrArgs& a, int64_t i, double& best_d2) {
    const double px = a.xs[3 * i], py = a.xs[3 * i + 1], pz = a.xs[3 * i + 2];
    const float4 q = make_float4((float)px, (float)py, (float)pz, 0.f);
    double d2 = 0.0;
    int idx = -1, best = -1;
    best_d2 = INFINITY;
    if (!isfinite(q.x) || !isfinite(q.y) || !isfinite(q.z)) return -1;   // no d^2 is below r^2
    radius_visit(
            a.view, q, 0u,
            [&](const float4 p) {
                d2 = sq3(px - (double)p.x, py - (double)p.y, pz - (double)p.z);
                idx = __float_as_int(p.w);
                return d2 < a.r2;
            },
            [&](unsigned) {
                if (d2 < best_d2 || (d2 == best_d2 && idx < best)) {
                    best_d2 = d2;
                    best = idx;
                }
                return true;
            });
    return best;
}

// EvaluateRegistration (Registration.cpp:127-141) over one tile of kFgrTile source points: each point's nearest
// target point; thread 0 sums
// the tile's matches and d^2 in index order.
__global__ void __launch_bounds__(kFgrTile) fgr_eval_kernel(FgrArgs a) {
    __shared__ double s_d2[kFgrTile];
    __shared__ bool s_in[kFgrTile];
    const int64_t i = (int64_t)blockIdx.x * kFgrTile + threadIdx.x;
    double best_d2 = 0.0;
    int best = -1;
    if (i < a.n) {
        best = nearest(a, i, best_d2);
        a.out[i] = best;
    }
    s_d2[threadIdx.x] = best >= 0 ? best_d2 : 0.0;
    s_in[threadIdx.x] = best >= 0;
    __syncthreads();
    if (threadIdx.x != 0) return;
    const int cnt_max = (int)min((int64_t)kFgrTile, a.n - (int64_t)blockIdx.x * kFgrTile);
    int cnt = 0;
    double err = 0.0;
    for (int j = 0; j < cnt_max; ++j)
        if (s_in[j]) {
            ++cnt;
            err += s_d2[j];
        }
    a.part_cnt[blockIdx.x] = cnt;
    a.part_err[blockIdx.x] = err;
}

// The tiles' sums in tile order: fitness = matches / n, rmse = sqrt(sum d^2 / matches), both 0 without a match.
__global__ void __launch_bounds__(32) fgr_sum_kernel(FgrArgs a) {
    if (threadIdx.x != 0) return;
    long long cnt = 0;
    double err = 0.0;
    for (int t = 0; t < a.tiles; ++t) {
        cnt += a.part_cnt[t];
        err += a.part_err[t];
    }
    FgrState* s = a.state;
    s->fitness = cnt ? (double)cnt / (double)a.n : 0.0;
    s->rmse = cnt ? sqrt(err / (double)cnt) : 0.0;
}

// nonfinite = 1 when any target coordinate is NaN or infinite (grid_index_finite)
__global__ void __launch_bounds__(kThreads) fgr_finite_kernel(const float* __restrict__ pts, int64_t n,
                                                              unsigned* __restrict__ nonfinite) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) flag_nonfinite(pts, i, nonfinite);
}

}  // namespace o3db

using namespace o3db;

extern "C" {

int o3db_registration_fgr(const float* source_dev, int64_t n, const float* target_dev, int64_t m,
                          const int64_t* correspondences_dev, int64_t K, const float* source_feature_dev,
                          const float* target_feature_dev, int dim, const o3db_fgr_option* option,
                          double* transformation_host, int64_t* correspondence_set_dev, o3db_fgr_stats* stats,
                          void* stream) {
    O3DB_REQUIRE(transformation_host && option, "o3db_registration_fgr: null transformation or option");
    O3DB_REQUIRE(n >= 0 && n < INT_MAX && m >= 0 && m < INT_MAX && K >= 0 && K < INT_MAX,
                 "o3db_registration_fgr: point and correspondence counts must be below 2^31 - 1 (got n=%lld, m=%lld, "
                 "K=%lld)", (long long)n, (long long)m, (long long)K);
    const bool features = correspondences_dev == nullptr;
    O3DB_REQUIRE(!features || (source_feature_dev && target_feature_dev && dim >= 1) || (n == 0 || m == 0),
                 "o3db_registration_fgr: give either the correspondences or both feature matrices");
    O3DB_REQUIRE(n == 0 || (source_dev && correspondence_set_dev), "o3db_registration_fgr: null source or output");
    O3DB_REQUIRE(m == 0 || target_dev, "o3db_registration_fgr: null target");
    const o3db_fgr_option o = *option;
    O3DB_REQUIRE(!std::isnan(o.maximum_correspondence_distance) && !std::isinf(o.maximum_correspondence_distance),
                 "FastGlobalRegistration: maximum_correspondence_distance must be finite (got %g)",
                 o.maximum_correspondence_distance);
    cudaStream_t st = (cudaStream_t)stream;
    for (int k = 0; k < 16; ++k) transformation_host[k] = k % 5 == 0 ? 1.0 : 0.0;
    if (stats) *stats = o3db_fgr_stats{0, 0, 0, 0, 0.0, 0.0};
    configure_memory_pool();
    struct Readback {
        FgrState state;
        double mean[6];
        unsigned long long scale;
        unsigned bad[2];
        unsigned passed;
        int stop[2];
    };
    DevPtr<Readback> d;
    if (int rc = dev_alloc(d, 1, st)) return rc;
    PinnedPtr<Readback> h = pinned_block<Readback>();
    if (!h) {
        set_last_error("o3db_registration_fgr: out of pinned host memory");
        return O3DB_ERR_CUDA;
    }
    O3DB_CUDA_CHECK(cudaMemsetAsync(d.get(), 0, sizeof(Readback), st));
    const int64_t big = std::max(std::max(n, m), features ? (int64_t)0 : K);
    if (big > 0) {
        fgr_check_kernel<<<(unsigned)ceil_div(big, kFgrT), kFgrT, 0, st>>>(source_dev, n, target_dev, m,
                                                                           correspondences_dev, features ? 0 : K,
                                                                           d->bad);
        O3DB_LAUNCH_CHECK();
    }
    fgr_mean_kernel<<<1, 32, 0, st>>>(source_dev, n, target_dev, m, d->mean);
    O3DB_LAUNCH_CHECK();
    if (n + m > 0) {
        fgr_scale_kernel<<<(unsigned)ceil_div(n + m, kFgrT), kFgrT, 0, st>>>(source_dev, n, target_dev, m, d->mean,
                                                                             &d->scale);
        O3DB_LAUNCH_CHECK();
    }
    O3DB_CUDA_CHECK(cudaMemcpyAsync(h.get(), d.get(), sizeof(Readback), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));   // the checks, the means and the scale
    O3DB_REQUIRE(!(h->bad[0] & 1u), "FastGlobalRegistration: the source point cloud has non-finite coordinates; "
                                    "remove them first with remove_non_finite_points");
    O3DB_REQUIRE(!(h->bad[0] & 2u), "FastGlobalRegistration: the target point cloud has non-finite coordinates; "
                                    "remove them first with remove_non_finite_points");
    O3DB_REQUIRE(!h->bad[1], "FastGlobalRegistration: a correspondence lies outside [0, %lld) x [0, %lld)",
                 (long long)n, (long long)m);
    double scale;
    {
        const unsigned long long bits = h->scale;
        memcpy(&scale, &bits, sizeof(scale));
    }
    const double scale_global = o.use_absolute_scale ? 1.0 : scale;
    // NormalizePointCloud (:185-188), with fmt's {} of a double
    O3DB_REQUIRE(scale_global > 0, "Invalid scale_global: %g, it must be > 0.", scale_global);

    // The initial pairs: the given set, or InitialMatching's mutual nearest features (:27-81) with the smaller cloud's
    // rows as the queries when the tuple test runs (:354-365).  o3db_correspondences_from_features with a negative
    // ratio keeps exactly the mutual pairs, in ascending query row, and never falls back to all of them.
    DevPtr<int64_t> cross;
    const int64_t* pairs0 = correspondences_dev;
    int64_t ncross = K;
    int swapped = 0;
    if (features) {
        ncross = 0;
        if (n > 0 && m > 0) {
            swapped = o.tuple_test && n < m;
            const int64_t nq = swapped ? m : n;
            if (int rc = dev_alloc(cross, (size_t)nq * 2, st)) return rc;
            int64_t mutual = 0;
            if (int rc = swapped ? o3db_correspondences_from_features(target_feature_dev, m, source_feature_dev, n,
                                                                      dim, 1, -1.0f, cross.get(), &ncross, &mutual,
                                                                      stream)
                                 : o3db_correspondences_from_features(source_feature_dev, n, target_feature_dev, m,
                                                                      dim, 1, -1.0f, cross.get(), &ncross, &mutual,
                                                                      stream))
                return rc;
            pairs0 = cross.get();
        }
    }
    if (stats) stats->cross = ncross;

    // AdvancedMatching (:83-141) on the unnormalised clouds, kFgrBatch trials at a time
    DevPtr<int64_t> tuples;
    const int64_t* pairs = pairs0;
    int64_t np = ncross;
    long long cnt = 0, consumed = 0;
    if (o.tuple_test) {
        np = 0;
        if (ncross <= 2) {
            fprintf(stderr,
                    "[Open3D WARNING] Not enough correspondences for tuple test. At least 3 needed, got %lld.\n",
                    (long long)ncross);
        } else {
            O3DB_REQUIRE(ncross <= INT_MAX / 100, "FastGlobalRegistration: %lld correspondences give more than 2^31 - 1 "
                         "tuple trials", (long long)ncross);
            const int ntrial = (int)ncross * 100;
            const long long maxc = o.maximum_tuple_count;
            const long long cap = std::max(1LL, std::min<long long>(maxc, ntrial));
            if (int rc = dev_alloc(tuples, (size_t)cap * 6, st)) return rc;
            const int B = std::min(kFgrBatch, ntrial);
            DevPtr<int> draws, stop;
            DevPtr<unsigned> pass;
            if (int rc = dev_alloc(draws, (size_t)B * 3, st)) return rc;
            if (int rc = dev_alloc(stop, 2, st)) return rc;
            if (int rc = dev_alloc(pass, (size_t)B + 1 + ceil_div(B, kScanTile), st)) return rc;
            std::vector<int> hdraws((size_t)B * 3);
            const float* A = swapped ? target_dev : source_dev;
            const float* Bc = swapped ? source_dev : target_dev;
            std::uniform_int_distribution<int> dist(0, (int)ncross - 1);
            std::lock_guard<std::mutex> lock(random_mutex());
            std::mt19937& engine = random_engine();
            // a failure inside the loop returns with the engine where the call found it, not part-way into a batch
            struct EngineGuard {
                std::mt19937& engine;
                const std::mt19937 entry;
                bool keep = false;
                ~EngineGuard() {
                    if (!keep) engine = entry;
                }
            } guard{engine, engine};
            for (int base = 0; base < ntrial; base += B) {
                const int hb = std::min(B, ntrial - base);
                const std::mt19937 saved = engine;
                for (int64_t k = 0; k < (int64_t)hb * 3; ++k) hdraws[k] = dist(engine);
                O3DB_CUDA_CHECK(cudaMemcpyAsync(draws.get(), hdraws.data(), (size_t)hb * 3 * sizeof(int),
                                                cudaMemcpyHostToDevice, st));
                const unsigned grid = (unsigned)ceil_div(hb, kFgrT);
                fgr_tuple_kernel<<<grid, kFgrT, 0, st>>>(A, Bc, pairs0, draws.get(), hb, o.tuple_scale, pass.get());
                O3DB_LAUNCH_CHECK();
                if (int rc = exclusive_scan_u32(pass.get(), hb, pass.get() + B + 1, st)) return rc;
                h->stop[0] = hb;
                h->stop[1] = 0;
                O3DB_CUDA_CHECK(cudaMemcpyAsync(stop.get(), h->stop, 2 * sizeof(int), cudaMemcpyHostToDevice, st));
                fgr_stop_kernel<<<grid, kFgrT, 0, st>>>(pass.get(), hb, cnt, maxc, stop.get());
                O3DB_LAUNCH_CHECK();
                fgr_tuple_compact_kernel<<<grid, kFgrT, 0, st>>>(pairs0, draws.get(), pass.get(), hb, stop.get(), cnt,
                                                                 swapped, tuples.get());
                O3DB_LAUNCH_CHECK();
                O3DB_CUDA_CHECK(cudaMemcpyAsync(h->stop, stop.get(), 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
                O3DB_CUDA_CHECK(cudaMemcpyAsync(&h->passed, pass.get() + hb, sizeof(unsigned),
                                                cudaMemcpyDeviceToHost, st));
                O3DB_CUDA_CHECK(cudaStreamSynchronize(st));   // the batch's stop, if any
                if (h->stop[0] < hb) {   // stopped: restore the engine and redraw the consumed prefix
                    cnt += h->stop[1];
                    consumed = (long long)base + h->stop[0] + 1;
                    engine = saved;
                    for (int64_t k = 0; k < (int64_t)(h->stop[0] + 1) * 3; ++k) (void)dist(engine);
                    break;
                }
                cnt += h->passed;
                consumed = (long long)base + hb;
            }
            guard.keep = true;
        }
        pairs = tuples.get();
        np = 3 * cnt;
    }
    if (stats) {
        stats->tuples = cnt;
        stats->trials = consumed;
        stats->pairs = np;
    }

    // OptimizePairwiseRegistration and the de-normalisation, one CTA
    FgrArgs a{};
    a.src = source_dev;
    a.tgt = target_dev;
    a.n = n;
    a.m = m;
    for (int c = 0; c < 3; ++c) {
        a.mean_s[c] = h->mean[c];
        a.mean_t[c] = h->mean[3 + c];
    }
    a.scale_global = scale_global;
    a.pairs = pairs;
    a.np = (int)np;
    a.iterations = o.iteration_number;
    a.decrease_mu = o.decrease_mu;
    a.max_dist = o.maximum_correspondence_distance;
    a.division = o.division_factor;
    a.r2 = o.maximum_correspondence_distance * o.maximum_correspondence_distance;
    a.tiles = (int)ceil_div(n, kFgrTile);
    DevPtr<FgrState> state;
    DevPtr<double> buf, part_err, xs;
    DevPtr<int> part_cnt;
    if (int rc = dev_alloc(state, 1, st)) return rc;
    a.state = state.get();
    a.out = correspondence_set_dev;
    const bool iterate = np >= 10 && o.iteration_number > 0;
    const size_t smem = iterate ? (size_t)np * 7 * sizeof(double) : 0;
    a.staged = smem <= kFgrSmem;
    if (iterate) {   // p, and q, r, s when they do not fit in shared memory
        if (int rc = dev_alloc(buf, (size_t)np * (a.staged ? 3 : 10), st)) return rc;
        a.buf = buf.get();
    }
    const size_t dyn = a.staged ? smem : 0;
    if (dyn > 48 * 1024)
        O3DB_CUDA_CHECK(cudaFuncSetAttribute(fgr_optimize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)kFgrSmem));
    fgr_optimize_kernel<<<1, kFgrT, dyn, st>>>(a);
    O3DB_LAUNCH_CHECK();

    // EvaluateRegistration on the original clouds
    o3db_nns index;
    const bool search = n > 0 && m > 0 && o.maximum_correspondence_distance > 0.0;
    if (search) {
        if (int rc = dev_alloc(part_cnt, (size_t)a.tiles, st)) return rc;
        if (int rc = dev_alloc(part_err, (size_t)a.tiles, st)) return rc;
        a.part_cnt = part_cnt.get();
        a.part_err = part_err.get();
        if (int rc = grid_index_finite(&index, target_dev, m, o.maximum_correspondence_distance, fgr_finite_kernel,
                                       "FastGlobalRegistration: the target point cloud has non-finite coordinates",
                                       st))
            return rc;
        const double rr = o.maximum_correspondence_distance * (1.0 + 1e-5);
        a.view = RadiusView{index.g, index.pts4.get(), index.cell_start.get(),
                            rr < (double)FLT_MAX ? (float)rr : INFINITY};
        if (int rc = dev_alloc(xs, (size_t)n * 3, st)) return rc;
        a.xs = xs.get();
        fgr_transform_kernel<<<(unsigned)ceil_div(n, kFgrT), kFgrT, 0, st>>>(source_dev, n, state.get(), xs.get());
        O3DB_LAUNCH_CHECK();
        fgr_eval_kernel<<<(unsigned)a.tiles, kFgrTile, 0, st>>>(a);
        O3DB_LAUNCH_CHECK();
        fgr_sum_kernel<<<1, 32, 0, st>>>(a);
        O3DB_LAUNCH_CHECK();
    } else if (n > 0) {
        O3DB_CUDA_CHECK(cudaMemsetAsync(correspondence_set_dev, 0xff, (size_t)n * sizeof(int64_t), st));
    }
    O3DB_CUDA_CHECK(cudaMemcpyAsync(&h->state, state.get(), sizeof(FgrState), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));   // the result
    const FgrState& s = h->state;
    for (int k = 0; k < 16; ++k) transformation_host[k] = s.T[k];
    if (stats) {
        stats->fitness = search ? s.fitness : 0.0;
        stats->inlier_rmse = search ? s.rmse : 0.0;
    }
    return O3DB_OK;
}

}  // extern "C"
