// fgr_oracle.c — CPU oracle of Fast Global Registration, pipelines::registration::
// FastGlobalRegistrationBasedOnCorrespondence (pipelines/registration/FastGlobalRegistration.cpp:285-327) run on one
// thread, restated in C in the orders DESIGN.md §4.26 states.  TEST INFRASTRUCTURE.  With one tile for the whole cloud
// it equals the reference's own function, compiled unmodified into oracle/_ref/libo3dref_fgr.so (oracle/ref_shim_fgr),
// bit for bit (tests/test_oracle_fgr.py).  The feature call is this one on the mutual feature pairs the caller lists.
//
// It takes the tuple test's draws as input (the library's generator is checked on its own).  f64 throughout, each op
// rounded (-ffp-contract=off).  The nearest target point is found by brute force over all m target points (OpenMP
// over the source points).  The sum of d^2 runs over each tile of `tile` source points in index order, then over the
// tiles in order; tile >= n gives upstream's single sequential sum.
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    double division_factor;
    int use_absolute_scale;
    int decrease_mu;
    double maximum_correspondence_distance;
    int iteration_number;
    double tuple_scale;
    int maximum_tuple_count;
    int tuple_test;
} fgr_option_t;

static double sq3(double x, double y, double z) { return (x * x + y * y) + z * z; }

// The stated sine / cosine (fgr_sincos in open3d_b200/csrc/fgr.cu, op for op).
double orc_fgr_sincos(double x, int want_cos) {
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

// Eigen's LDLT of the 6x6 A (row-major; only the lower triangle is read; A is overwritten) with diagonal pivoting,
// then its solve of A x = b, b overwritten by x (ldlt_solve6 in fgr.cu, op for op).
void orc_fgr_ldlt_solve6(double* A, double* b) {
    int tr[6];
    double tmp[6];
    for (int k = 0; k < 6; ++k) {
        int p = k;
        double big = fabs(A[7 * k]);
        for (int i = k + 1; i < 6; ++i)
            if (fabs(A[7 * i]) > big) {
                big = fabs(A[7 * i]);
                p = i;
            }
        tr[k] = p;
        if (p != k) {
            for (int j = 0; j < k; ++j) {
                const double t = A[6 * k + j];
                A[6 * k + j] = A[6 * p + j];
                A[6 * p + j] = t;
            }
            for (int i = p + 1; i < 6; ++i) {
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
        if (k == 0 && !(fabs(akk) > 0.0)) {
            for (int j = 0; j < 6; ++j) tr[j] = j;
            break;
        }
        if (fabs(akk) > 0.0)
            for (int i = k + 1; i < 6; ++i) A[6 * i + k] = A[6 * i + k] / akk;
    }
    for (int k = 0; k < 6; ++k) {
        const int p = tr[k];
        const double t = b[k];
        b[k] = b[p];
        b[p] = t;
    }
    for (int i = 0; i < 6; ++i)
        for (int j = i + 1; j < 6; ++j) b[j] = b[j] - A[6 * j + i] * b[i];
    for (int i = 0; i < 6; ++i) {
        const double d = A[7 * i];
        b[i] = fabs(d) > 1.0 / DBL_MAX ? b[i] / d : 0.0;
    }
    for (int i = 5; i >= 0; --i)
        for (int j = 0; j < i; ++j) b[j] = b[j] - A[6 * i + j] * b[i];
    for (int k = 5; k >= 0; --k) {
        const int p = tr[k];
        const double t = b[k];
        b[k] = b[p];
        b[p] = t;
    }
}

static void qmul(const double* a, const double* b, double* o) {
    o[0] = ((a[0] * b[0] - a[1] * b[1]) - a[2] * b[2]) - a[3] * b[3];
    o[1] = ((a[0] * b[1] + a[1] * b[0]) + a[2] * b[3]) - a[3] * b[2];
    o[2] = ((a[0] * b[2] + a[2] * b[0]) + a[3] * b[1]) - a[1] * b[3];
    o[3] = ((a[0] * b[3] + a[3] * b[0]) + a[1] * b[2]) - a[2] * b[1];
}

// The quaternion (w, x, y, z) of AngleAxis(angle, axis): w = cos(angle/2), v = sin(angle/2) axis.
void orc_fgr_angle_axis(double angle, const double* axis, double* q) {
    const double h = 0.5 * angle;
    const double s = orc_fgr_sincos(h, 0);
    q[0] = orc_fgr_sincos(h, 1);
    q[1] = s * axis[0];
    q[2] = s * axis[1];
    q[3] = s * axis[2];
}

// Quaternion::toRotationMatrix, R row-major 3x3.
void orc_fgr_quat_to_matrix(const double* q, double* R) {
    const double tx = 2.0 * q[1], ty = 2.0 * q[2], tz = 2.0 * q[3];
    const double twx = tx * q[0], twy = ty * q[0], twz = tz * q[0];
    const double txx = tx * q[1], txy = ty * q[1], txz = tz * q[1];
    const double tyy = ty * q[2], tyz = tz * q[2], tzz = tz * q[3];
    R[0] = 1.0 - (tyy + tzz), R[1] = txy - twz, R[2] = txz + twy;
    R[3] = txy + twz, R[4] = 1.0 - (txx + tzz), R[5] = tyz - twx;
    R[6] = txz - twy, R[7] = tyz + twx, R[8] = 1.0 - (txx + tyy);
}

void orc_fgr_quat_mul(const double* a, const double* b, double* o) { qmul(a, b, o); }

// TransformVector6dToMatrix4d: D row-major 4x4.
void orc_fgr_vec6_to_mat4(const double* x, double* D) {
    static const double Z[3] = {0.0, 0.0, 1.0}, Y[3] = {0.0, 1.0, 0.0}, X[3] = {1.0, 0.0, 0.0};
    double qz[4], qy[4], qx[4], q1[4], q[4], R[9];
    orc_fgr_angle_axis(x[2], Z, qz);
    orc_fgr_angle_axis(x[1], Y, qy);
    orc_fgr_angle_axis(x[0], X, qx);
    qmul(qz, qy, q1);
    qmul(q1, qx, q);
    orc_fgr_quat_to_matrix(q, R);
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) D[4 * r + c] = R[3 * r + c];
        D[4 * r + 3] = x[3 + r];
    }
    D[12] = D[13] = D[14] = 0.0;
    D[15] = 1.0;
}

static double det3(const double* M, int r0, int r1, int r2, int c0, int c1, int c2) {
    const double a = M[4 * r0 + c0], b = M[4 * r0 + c1], c = M[4 * r0 + c2];
    const double d = M[4 * r1 + c0], e = M[4 * r1 + c1], f = M[4 * r1 + c2];
    const double g = M[4 * r2 + c0], h = M[4 * r2 + c1], i = M[4 * r2 + c2];
    return (a * (e * i - f * h) - b * (d * i - f * g)) + c * (d * h - e * g);
}

// Matrix4d::inverse as stated (inverse4 in fgr.cu): M and out row-major, distinct.
void orc_fgr_inverse4(const double* M, double* out) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            const int r0 = i == 0 ? 1 : 0, r1 = i <= 1 ? 2 : 1, r2 = i <= 2 ? 3 : 2;
            const int c0 = j == 0 ? 1 : 0, c1 = j <= 1 ? 2 : 1, c2 = j <= 2 ? 3 : 2;
            const double m = det3(M, r0, r1, r2, c0, c1, c2);
            out[4 * j + i] = (i + j) & 1 ? -m : m;
        }
    const double det = ((M[0] * out[0] + M[4] * out[1]) + M[8] * out[2]) + M[12] * out[3];
    for (int k = 0; k < 16; ++k) out[k] = out[k] / det;
}

// Eigen's isIdentity() at 1e-12.
int orc_fgr_is_identity(const double* T) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            const double v = T[4 * i + j];
            if (i == j ? !(fabs(v - 1.0) <= fmin(fabs(v), 1.0) * 1e-12) : !(fabs(v) <= 1e-12)) return 0;
        }
    return 1;
}

static double row4(const double* M, int j, double x, double y, double z) {
    return ((M[4 * j] * x + M[4 * j + 1] * y) + M[4 * j + 2] * z) + M[4 * j + 3] * 1.0;
}

// The Jacobian rows of OptimizePairwiseRegistration: J[k][0..5] for row k = x, y, z of the point q.
static void jac(const double* q, double J[3][6]) {
    memset(J, 0, sizeof(double) * 18);
    J[0][1] = -q[2], J[0][2] = q[1], J[0][3] = -1;
    J[1][2] = -q[0], J[1][0] = q[2], J[1][4] = -1;
    J[2][0] = -q[1], J[2][1] = q[0], J[2][5] = -1;
}

// Returns 0, -1 for too few draws, -2 for no memory, -3 for scale_global <= 0 (stats[0] then holds nothing).
// pairs [K][2] index (source, target), or (target, source) when swapped: the tuple test then runs on (target,
// source) and its pairs are swapped back, as the feature call's n < m branch does.
// stats: tuples, trials consumed, pairs optimised, warnings (the ncorr <= 2 one); fr: fitness, rmse, scale_global.
// pairs_out receives the optimiser's pairs [stats[2]][2] (capacity: max(K, 3 max(1, maximum_tuple_count))).
int orc_fgr(const float* src, int64_t n, const float* tgt, int64_t m, const int64_t* pairs, int64_t K, int swapped,
            const int* draws, int64_t num_draws, const fgr_option_t* opt, int64_t tile, double* T_out,
            int64_t* corres_out, int64_t* stats, double* fr, int64_t* pairs_out) {
    stats[0] = stats[1] = stats[2] = stats[3] = 0;
    fr[0] = fr[1] = fr[2] = 0.0;
    // NormalizePointCloud
    double mean[2][3], scale = 0.0;
    for (int c = 0; c < 2; ++c) {
        const float* p = c ? tgt : src;
        const int64_t k = c ? m : n;
        for (int a = 0; a < 3; ++a) {
            double s = 0.0;
            for (int64_t i = 0; i < k; ++i) s = s + (double)p[3 * i + a];
            mean[c][a] = s / (double)(int)k;
        }
        for (int64_t i = 0; i < k; ++i) {
            const double v = sqrt(sq3(p[3 * i] - mean[c][0], p[3 * i + 1] - mean[c][1], p[3 * i + 2] - mean[c][2]));
            if (v > scale) scale = v;
        }
    }
    const double sg = opt->use_absolute_scale ? 1.0 : scale;
    fr[2] = sg;
    if (!(sg > 0)) return -3;
    // AdvancedMatching
    int64_t np = K;
    if (opt->tuple_test) {
        np = 0;
        if (K <= 2) {
            stats[3] = 1;
        } else {
            const float* A = swapped ? tgt : src;
            const float* B = swapped ? src : tgt;
            const int64_t ntrial = K * 100;
            int64_t cnt = 0, i;
            for (i = 0; i < ntrial; ++i) {
                if (3 * (i + 1) > num_draws) return -1;
                int64_t id[3][2];
                for (int k = 0; k < 3; ++k) {
                    const int64_t r = draws[3 * i + k];
                    id[k][0] = pairs[2 * r];
                    id[k][1] = pairs[2 * r + 1];
                }
                double l[2][3];
                for (int c = 0; c < 2; ++c) {
                    const float* P = c ? B : A;
                    for (int e = 0; e < 3; ++e) {
                        const float* u = P + 3 * id[e][c];
                        const float* v = P + 3 * id[(e + 1) % 3][c];
                        l[c][e] = sqrt(sq3((double)u[0] - v[0], (double)u[1] - v[1], (double)u[2] - v[2]));
                    }
                }
                const double s = opt->tuple_scale;
                if ((l[0][0] * s < l[1][0]) && (l[1][0] < l[0][0] / s) && (l[0][1] * s < l[1][1]) &&
                    (l[1][1] < l[0][1] / s) && (l[0][2] * s < l[1][2]) && (l[1][2] < l[0][2] / s)) {
                    for (int k = 0; k < 3; ++k) {
                        pairs_out[2 * np] = id[k][swapped ? 1 : 0];
                        pairs_out[2 * np + 1] = id[k][swapped ? 0 : 1];
                        ++np;
                    }
                    ++cnt;
                }
                if (cnt >= opt->maximum_tuple_count) {
                    ++i;
                    break;
                }
            }
            stats[0] = cnt;
            stats[1] = i;
        }
    } else {
        memcpy(pairs_out, pairs, sizeof(int64_t) * 2 * (size_t)K);
    }
    stats[2] = np;
    // OptimizePairwiseRegistration on the normalised clouds
    double trans[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    if (np >= 10 && opt->iteration_number > 0) {
        double* P = malloc(sizeof(double) * 6 * (size_t)np);
        if (!P) return -2;
        double* Q = P + 3 * np;
        for (int64_t c = 0; c < np; ++c)
            for (int a = 0; a < 3; ++a) {
                P[3 * c + a] = ((double)src[3 * pairs_out[2 * c] + a] - mean[0][a]) / sg;
                Q[3 * c + a] = ((double)tgt[3 * pairs_out[2 * c + 1] + a] - mean[1][a]) / sg;
            }
        double par = sg, delta[16];
        for (int itr = 0; itr < opt->iteration_number; ++itr) {
            double JTJ[36] = {0}, JTr[6] = {0};
            for (int64_t c = 0; c < np; ++c) {
                double* q = Q + 3 * c;
                if (itr > 0) {
                    const double w = row4(delta, 3, q[0], q[1], q[2]);
                    const double o0 = row4(delta, 0, q[0], q[1], q[2]), o1 = row4(delta, 1, q[0], q[1], q[2]),
                                 o2 = row4(delta, 2, q[0], q[1], q[2]);
                    q[0] = o0 / w, q[1] = o1 / w, q[2] = o2 / w;
                }
                const double* p = P + 3 * c;
                const double r[3] = {p[0] - q[0], p[1] - q[1], p[2] - q[2]};
                const double t = par / (sq3(r[0], r[1], r[2]) + par);
                const double s = t * t;
                double J[3][6];
                jac(q, J);
                for (int k = 0; k < 3; ++k)   // the dense update, as upstream: the zero terms leave every sum as it is
                    for (int e = 0; e < 6; ++e) {
                        for (int f = 0; f < 6; ++f) JTJ[6 * e + f] = JTJ[6 * e + f] + (J[k][e] * J[k][f]) * s;
                        JTr[e] = JTr[e] + (J[k][e] * r[k]) * s;
                    }
            }
            for (int k = 0; k < 36; ++k) JTJ[k] = -JTJ[k];
            orc_fgr_ldlt_solve6(JTJ, JTr);
            orc_fgr_vec6_to_mat4(JTr, delta);
            double nt[16];
            for (int r = 0; r < 4; ++r)
                for (int c = 0; c < 4; ++c)
                    nt[4 * r + c] = ((delta[4 * r] * trans[c] + delta[4 * r + 1] * trans[4 + c]) +
                                     delta[4 * r + 2] * trans[8 + c]) + delta[4 * r + 3] * trans[12 + c];
            memcpy(trans, nt, sizeof(nt));
            if (opt->decrease_mu && itr % 4 == 0 && par > opt->maximum_correspondence_distance)
                par = par / opt->division_factor;
        }
        free(P);
    }
    // GetTransformationOriginalScale and the inverse
    double M[16] = {0};
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) M[4 * r + c] = trans[4 * r + c];
        const double rm = (-trans[4 * r] * mean[1][0] + -trans[4 * r + 1] * mean[1][1]) + -trans[4 * r + 2] * mean[1][2];
        M[4 * r + 3] = (rm + trans[4 * r + 3] * sg) + mean[0][r];
    }
    M[15] = 1.0;
    orc_fgr_inverse4(M, T_out);
    // EvaluateRegistration
    const double md = opt->maximum_correspondence_distance, r2 = md * md;
    for (int64_t i = 0; i < n; ++i) corres_out[i] = -1;
    if (md <= 0.0 || n == 0) return 0;
    double* d2 = malloc(sizeof(double) * (size_t)n);
    if (!d2) return -2;
    const int ident = orc_fgr_is_identity(T_out);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        double x = src[3 * i], y = src[3 * i + 1], z = src[3 * i + 2];
        if (!ident) {
            const double w = row4(T_out, 3, x, y, z);
            const double o0 = row4(T_out, 0, x, y, z), o1 = row4(T_out, 1, x, y, z), o2 = row4(T_out, 2, x, y, z);
            x = o0 / w, y = o1 / w, z = o2 / w;
        }
        double best = INFINITY;
        int64_t bi = -1;
        for (int64_t j = 0; j < m; ++j) {
            const double d = sq3(x - tgt[3 * j], y - tgt[3 * j + 1], z - tgt[3 * j + 2]);
            if (d < r2 && d < best) {
                best = d;
                bi = j;
            }
        }
        corres_out[i] = bi;
        d2[i] = best;
    }
    int64_t cnt = 0;
    double err = 0.0;
    for (int64_t lo = 0; lo < n; lo += tile) {
        double e = 0.0;
        for (int64_t j = lo; j < n && j < lo + tile; ++j)
            if (corres_out[j] >= 0) {
                ++cnt;
                e += d2[j];
            }
        err += e;
    }
    free(d2);
    fr[0] = cnt ? (double)cnt / (double)n : 0.0;
    fr[1] = cnt ? sqrt(err / (double)cnt) : 0.0;
    return 0;
}
