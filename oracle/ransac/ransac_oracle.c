// ransac_oracle.c — CPU oracle of global registration by RANSAC, pipelines::registration::
// RegistrationRANSACBasedOnCorrespondence (pipelines/registration/Registration.cpp:195-379) run on one thread with
// TransformationEstimationPointToPoint(false) and the three checkers, restated in C in the orders DESIGN.md §4.25
// states.  TEST INFRASTRUCTURE.  With one tile for the whole cloud it equals the reference's own function, compiled
// unmodified into oracle/_ref/libo3dref_ransac.so (oracle/ref_shim_ransac), bit for bit (tests/test_oracle_ransac.py).
//
// It takes the draws as input (the library's generator is checked on its own).  f64 throughout, each op rounded
// (-ffp-contract=off), in the stated orders.  The nearest target point is found by brute force over all m target
// points (OpenMP over the source points).  The sum of d^2 runs over each tile of `tile` source points in index order,
// then over the tiles in order; tile >= n gives upstream's single sequential sum.
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    int use_edge_length, use_distance, use_normal;
    double edge_length_similarity;
    double distance_threshold;
    double cos_normal_angle_threshold;
} checkers_t;

static double sq3(double x, double y, double z) { return (x * x + y * y) + z * z; }

static void xform(const double* T, const float* p, double* o) {
    const double x = p[0], y = p[1], z = p[2];
    o[0] = ((T[0] * x + T[1] * y) + T[2] * z) + T[3];
    o[1] = ((T[4] * x + T[5] * y) + T[6] * z) + T[7];
    o[2] = ((T[8] * x + T[9] * y) + T[10] * z) + T[11];
}

// kabsch_rotation of open3d_b200/csrc/reduce.cuh, op for op.
static int jacobi(double G[3][3], double V[3][3], int P, int Q) {
    double alpha = 0, beta = 0, gamma = 0;
    for (int r = 0; r < 3; ++r) {
        alpha += G[r][P] * G[r][P];
        beta += G[r][Q] * G[r][Q];
        gamma += G[r][P] * G[r][Q];
    }
    if (!(gamma * gamma > 1e-32 * alpha * beta)) return 0;
    const double zeta = (beta - alpha) / (2.0 * gamma);
    const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
    const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
    for (int r = 0; r < 3; ++r) {
        const double gp = G[r][P], gq = G[r][Q], vp = V[r][P], vq = V[r][Q];
        G[r][P] = c * gp - s * gq;
        G[r][Q] = s * gp + c * gq;
        V[r][P] = c * vp - s * vq;
        V[r][Q] = s * vp + c * vq;
    }
    return 1;
}

void orc_ransac_kabsch(const double* H, double* R) {
    double G[3][3], V[3][3];
    double scale = 0;
    for (int k = 0; k < 9; ++k) scale = fmax(scale, fabs(H[k]));
    const double inv = scale > 0 ? 1.0 / scale : 0.0;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            G[r][c] = H[3 * r + c] * inv;
            V[r][c] = r == c ? 1.0 : 0.0;
        }
    for (int sweep = 0; sweep < 40; ++sweep) {
        int any = jacobi(G, V, 0, 1);
        any |= jacobi(G, V, 0, 2);
        any |= jacobi(G, V, 1, 2);
        if (!any) break;
    }
    double n2[3];
    for (int c = 0; c < 3; ++c) n2[c] = G[0][c] * G[0][c] + G[1][c] * G[1][c] + G[2][c] * G[2][c];
    const int k = (n2[0] <= n2[1] && n2[0] <= n2[2]) ? 0 : (n2[1] <= n2[2] ? 1 : 2);
    const int ci = (k + 1) % 3, cj = (k + 2) % 3;
    double gi[3], gj[3], vi[3], vj[3], ni = n2[ci], nj = n2[cj];
    for (int r = 0; r < 3; ++r) {
        gi[r] = G[r][ci];
        gj[r] = G[r][cj];
        vi[r] = V[r][ci];
        vj[r] = V[r][cj];
    }
    if (nj > ni) {
        for (int r = 0; r < 3; ++r) {
            double t = gi[r];
            gi[r] = gj[r];
            gj[r] = t;
            t = vi[r];
            vi[r] = vj[r];
            vj[r] = t;
        }
        const double t = ni;
        ni = nj;
        nj = t;
    }
    double ui[3], uj[3];
    if (ni > 0) {
        const double s = 1.0 / sqrt(ni);
        for (int r = 0; r < 3; ++r) ui[r] = gi[r] * s;
    } else {
        ui[0] = 1.0;
        ui[1] = ui[2] = 0.0;
    }
    if (!(nj > 1e-28 * ni)) {
        const double ax = fabs(ui[0]), ay = fabs(ui[1]), az = fabs(ui[2]);
        gj[0] = (ax <= ay && ax <= az) ? 1.0 : 0.0;
        gj[1] = (gj[0] == 0.0 && ay <= az) ? 1.0 : 0.0;
        gj[2] = (gj[0] == 0.0 && gj[1] == 0.0) ? 1.0 : 0.0;
    }
    {
        const double d = gj[0] * ui[0] + gj[1] * ui[1] + gj[2] * ui[2];
        for (int r = 0; r < 3; ++r) uj[r] = gj[r] - d * ui[r];
        const double s = 1.0 / sqrt(uj[0] * uj[0] + uj[1] * uj[1] + uj[2] * uj[2]);
        for (int r = 0; r < 3; ++r) uj[r] *= s;
    }
    const double uk[3] = {ui[1] * uj[2] - ui[2] * uj[1], ui[2] * uj[0] - ui[0] * uj[2], ui[0] * uj[1] - ui[1] * uj[0]};
    const double vk[3] = {vi[1] * vj[2] - vi[2] * vj[1], vi[2] * vj[0] - vi[0] * vj[2], vi[0] * vj[1] - vi[1] * vj[0]};
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R[3 * r + c] = ui[r] * vi[c] + uj[r] * vj[c] + uk[r] * vk[c];
}

// Eigen::umeyama(src, dst, false) over the sample's pairs in sample order -> rows 0..2 of T.
void orc_ransac_estimate(const float* src, const float* tgt, const int64_t* pairs /* [rn][2] */, int rn,
                         double* T) {
    double ms[3] = {0, 0, 0}, mt[3] = {0, 0, 0}, H[9] = {0}, R[9];
    for (int k = 0; k < rn; ++k)
        for (int c = 0; c < 3; ++c) {
            ms[c] += src[3 * pairs[2 * k] + c];
            mt[c] += tgt[3 * pairs[2 * k + 1] + c];
        }
    const double inv = 1.0 / (double)rn;
    for (int c = 0; c < 3; ++c) {
        ms[c] *= inv;
        mt[c] *= inv;
    }
    for (int k = 0; k < rn; ++k) {
        double s[3], t[3];
        for (int c = 0; c < 3; ++c) {
            s[c] = (double)src[3 * pairs[2 * k] + c] - ms[c];
            t[c] = (double)tgt[3 * pairs[2 * k + 1] + c] - mt[c];
        }
        for (int j = 0; j < 3; ++j)
            for (int c = 0; c < 3; ++c) H[3 * j + c] += t[j] * s[c];
    }
    for (int q = 0; q < 9; ++q) H[q] *= inv;
    orc_ransac_kabsch(H, R);
    for (int j = 0; j < 3; ++j) {
        T[4 * j] = R[3 * j];
        T[4 * j + 1] = R[3 * j + 1];
        T[4 * j + 2] = R[3 * j + 2];
        T[4 * j + 3] = mt[j] - ((R[3 * j] * ms[0] + R[3 * j + 1] * ms[1]) + R[3 * j + 2] * ms[2]);
    }
}

static int checks_pass(const float* src, const float* snrm, const float* tgt, const float* tnrm,
                       const int64_t* pairs, int rn, const double* T, const checkers_t* ck) {
    if (ck->use_edge_length)
        for (int i = 0; i < rn; ++i)
            for (int j = i + 1; j < rn; ++j) {
                const float *si = src + 3 * pairs[2 * i], *sj = src + 3 * pairs[2 * j];
                const float *ti = tgt + 3 * pairs[2 * i + 1], *tj = tgt + 3 * pairs[2 * j + 1];
                const double ds = sqrt(sq3((double)si[0] - sj[0], (double)si[1] - sj[1], (double)si[2] - sj[2]));
                const double dt = sqrt(sq3((double)ti[0] - tj[0], (double)ti[1] - tj[1], (double)ti[2] - tj[2]));
                if (ds < dt * ck->edge_length_similarity || dt < ds * ck->edge_length_similarity) return 0;
            }
    if (ck->use_distance)
        for (int k = 0; k < rn; ++k) {
            double p[3];
            xform(T, src + 3 * pairs[2 * k], p);
            const float* t = tgt + 3 * pairs[2 * k + 1];
            if (sqrt(sq3(t[0] - p[0], t[1] - p[1], t[2] - p[2])) > ck->distance_threshold) return 0;
        }
    if (ck->use_normal && snrm && tnrm)
        for (int k = 0; k < rn; ++k) {
            const float* s = snrm + 3 * pairs[2 * k];
            const float* t = tnrm + 3 * pairs[2 * k + 1];
            double q[3];
            for (int j = 0; j < 3; ++j) q[j] = (T[4 * j] * s[0] + T[4 * j + 1] * s[1]) + T[4 * j + 2] * s[2];
            if ((t[0] * q[0] + t[1] * q[1]) + t[2] * q[2] < ck->cos_normal_angle_threshold) return 0;
        }
    return 1;
}

// Nearest target point of every transformed source point within r^2 (strict), ties to the lowest index.
static void nearest_all(const float* src, int64_t n, const float* tgt, int64_t m, const double* T, double r2,
                        int64_t* idx, double* d2) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        double p[3];
        xform(T, src + 3 * i, p);
        double best = INFINITY;
        int64_t bi = -1;
        for (int64_t j = 0; j < m; ++j) {
            const double d = sq3(p[0] - tgt[3 * j], p[1] - tgt[3 * j + 1], p[2] - tgt[3 * j + 2]);
            if (d < r2 && d < best) {   // ascending j: the first of equal distances stays
                best = d;
                bi = j;
            }
        }
        idx[i] = bi;
        d2[i] = best;
    }
}

// Returns 0, -1 for too few draws, -2 for no memory.  stats: drawn, validated, best index; fr: fitness, rmse.
int orc_ransac(const float* src, const float* snrm, int64_t n, const float* tgt, const float* tnrm, int64_t m,
               const int64_t* corres, int64_t K, const int* draws, int64_t num_draws, double max_dist, int rn,
               int max_iteration, double confidence, const checkers_t* ck, int64_t tile, double* T_out,
               int64_t* corres_out, int64_t* stats, double* fr) {
    for (int k = 0; k < 16; ++k) T_out[k] = k % 5 == 0 ? 1.0 : 0.0;
    for (int64_t i = 0; i < n; ++i) corres_out[i] = -1;
    stats[0] = stats[1] = 0;
    stats[2] = -1;
    fr[0] = fr[1] = 0.0;
    if (rn < 3 || K < rn || max_dist <= 0.0 || max_iteration <= 0) return 0;
    const double r2 = max_dist * max_dist, log_conf = log(1.0 - confidence);
    int64_t* pairs = malloc(sizeof(int64_t) * 2 * (size_t)rn);
    int64_t* idx = malloc(sizeof(int64_t) * (size_t)(n ? n : 1));
    double* d2 = malloc(sizeof(double) * (size_t)(n ? n : 1));
    if (!pairs || !idx || !d2) {
        free(pairs);
        free(idx);
        free(d2);
        return -2;
    }
    int rc = 0;
    int est_k = max_iteration;
    double best_fit = 0.0, best_rmse = 0.0, bestT[12];
    int64_t best = -1, validated = 0, i = 0;
    for (; i < max_iteration && i < est_k; ++i) {
        if ((i + 1) * rn > num_draws) {
            rc = -1;
            break;
        }
        for (int k = 0; k < rn; ++k) {
            const int64_t c = draws[i * rn + k];
            pairs[2 * k] = corres[2 * c];
            pairs[2 * k + 1] = corres[2 * c + 1];
        }
        double T[12];
        orc_ransac_estimate(src, tgt, pairs, rn, T);
        if (!checks_pass(src, snrm, tgt, tnrm, pairs, rn, T, ck)) continue;
        nearest_all(src, n, tgt, m, T, r2, idx, d2);
        int64_t cnt = 0;
        double err = 0.0;
        for (int64_t lo = 0; lo < n; lo += tile) {
            double e = 0.0;
            for (int64_t j = lo; j < n && j < lo + tile; ++j)
                if (idx[j] >= 0) {
                    ++cnt;
                    e += d2[j];
                }
            err += e;
        }
        const double fit = cnt ? (double)cnt / (double)n : 0.0;
        const double rmse = cnt ? sqrt(err / (double)cnt) : 0.0;
        if (fit > best_fit || (fit == best_fit && rmse < best_rmse)) {
            best_fit = fit;
            best_rmse = rmse;
            best = i;
            memcpy(bestT, T, sizeof(bestT));
            int64_t inl = 0;   // EvaluateInlierCorrespondenceRatio over all K pairs
            for (int64_t k = 0; k < K; ++k) {
                double p[3];
                xform(T, src + 3 * corres[2 * k], p);
                const float* t = tgt + 3 * corres[2 * k + 1];
                inl += sq3(p[0] - t[0], p[1] - t[1], p[2] - t[2]) < r2;
            }
            const double ratio = (double)inl / (double)K;
            double est = log_conf / log(1.0 - pow(ratio, (double)rn));
            if (est < 0) est = est_k;
            if (est < est_k) est_k = (int)ceil(est);
        }
        ++validated;
    }
    stats[0] = i;
    stats[1] = validated;
    stats[2] = best;
    fr[0] = best_fit;
    fr[1] = best_rmse;
    if (best >= 0 && rc == 0) {
        for (int k = 0; k < 12; ++k) T_out[k] = bestT[k];
        nearest_all(src, n, tgt, m, bestT, r2, corres_out, d2);
    }
    free(pairs);
    free(idx);
    free(d2);
    return rc;
}
