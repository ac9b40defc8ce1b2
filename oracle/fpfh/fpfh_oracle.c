/* fpfh_oracle.c — CPU restatement of t::pipelines::registration::ComputeFPFHFeature and CorrespondencesFromFeatures
 * (t/pipelines/registration/Feature.cpp:23-333, t/pipelines/kernel/FeatureImpl.h:23-293), Float32.
 *
 * TEST INFRASTRUCTURE ONLY, like the rest of oracle/: the product never links or calls it.
 *
 * Precision follows the reference's CPU build (g++ -ffp-contract=off), whose object code calls libm's f64 acos and
 * atan2 (the float arguments promote): the swap test compares two f64 acos values, feature[0] is the f64 atan2 rounded
 * to f32, every other pair-feature operation is f32 in upstream's order; the bins are f64 (M_PI, 11 * (...), floor),
 * hist_incr is 100.0 / (float)(count - 1) in f64 rounded to f32, and the FPFH scale 100.0 / sum likewise.  The device
 * evaluates the same f64 functions (DESIGN.md §4.24).  Checked bit for bit against the reference's own code compiled
 * into oracle/_ref/libo3dref_fpfh.so (tests/test_oracle_fpfh.py).
 *
 * Neighbour lists: brute force, dist^2 = fmaf(dz, dz, fmaf(dy, dy, dx * dx)) with d = p - q (the library's canonical
 * distance), the k nearest by (dist^2, index) with dist^2 <= thr.
 * Feature 1-NN: brute force, dist = sum over d of fmaf(s - t, s - t, acc) from 0 in index order, strict < from
 * (+inf, 0), so ties go to the lowest index.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static inline float dist2(const float* t, const float* q) {
    const float dx = t[0] - q[0], dy = t[1] - q[1], dz = t[2] - q[2];
    return fmaf(dz, dz, fmaf(dy, dy, dx * dx));
}

/* lists of the m query points q_ids (NULL: every point) among the n points: idx / d2 [m, kp] (-1 / 0 past the count),
 * cnt [m]; kp = min(k, n) */
void orc_fpfh_lists_f32(const float* pts, int64_t n, const int32_t* q_ids, int64_t m, int k, float thr, int32_t* idx,
                        float* d2, int32_t* cnt) {
    const int kp = k < n ? k : (int)n;
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t r = 0; r < m; ++r) {
        const int64_t qi = q_ids ? q_ids[r] : r;
        int32_t* bi = idx + r * kp;
        float* bd = d2 + r * kp;
        int c = 0;
        for (int64_t j = 0; j < n; ++j) {
            const float d = dist2(pts + 3 * j, pts + 3 * qi);
            if (!(d <= thr)) continue;
            if (c == kp && (d > bd[c - 1] || (d == bd[c - 1] && j > bi[c - 1]))) continue;
            int pos = c < kp ? c : kp - 1;
            while (pos > 0 && (bd[pos - 1] > d || (bd[pos - 1] == d && bi[pos - 1] > j))) {
                bd[pos] = bd[pos - 1];
                bi[pos] = bi[pos - 1];
                --pos;
            }
            bd[pos] = d;
            bi[pos] = (int32_t)j;
            if (c < kp) ++c;
        }
        for (int e = c; e < kp; ++e) {
            bi[e] = -1;
            bd[e] = 0.0f;
        }
        cnt[r] = c;
    }
}

static inline float dot3(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static inline void cross3(const float* a, const float* b, float* c) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

/* ComputePairFeature<float> */
void orc_pair_feature_f32(const float* p1, const float* n1, const float* p2, const float* n2, float* f) {
    float d[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]}, m1[3], m2[3], v[3], w[3];
    f[3] = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    if (f[3] == 0) {
        f[0] = f[1] = f[2] = f[3] = 0;
        return;
    }
    const float a1 = dot3(n1, d) / f[3], a2 = dot3(n2, d) / f[3];
    if (acos(fabs(a1)) > acos(fabs(a2))) {
        for (int k = 0; k < 3; ++k) {
            m1[k] = n2[k];
            m2[k] = n1[k];
            d[k] *= -1;
        }
        f[2] = -a2;
    } else {
        for (int k = 0; k < 3; ++k) {
            m1[k] = n1[k];
            m2[k] = n2[k];
        }
        f[2] = a1;
    }
    cross3(d, m1, v);
    const float vn = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    if (vn == 0.0) {
        f[0] = f[1] = f[2] = f[3] = 0;
        return;
    }
    v[0] /= vn;
    v[1] /= vn;
    v[2] /= vn;
    cross3(m1, v, w);
    f[1] = dot3(v, m2);
    f[0] = (float)atan2((double)dot3(w, m2), (double)dot3(m1, m2));
}

static inline int bin(double x) {
    const int h = (int)floor(x);
    return h >= 11 ? 10 : (h > 0 ? h : 0);
}

/* The whole function over lists idx / d2 [n, kp] and cnt [n] of every point: fpfh [ns, 33] for the rows sel[0..ns)
 * (sel NULL: every point, ns = n).  A selected row equals that point's row of the whole function. */
void orc_fpfh_f32(const float* pts, const float* nrm, int64_t n, const int32_t* idx, const float* d2,
                  const int32_t* cnt, int kp, const int64_t* sel, int64_t ns, float* out) {
    float* spfh = calloc((size_t)n * 33, sizeof(float));
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        const int c = cnt[i];
        if (c <= 1) continue;
        const float incr = 100.0 / (float)(c - 1);
        for (int e = 1; e < c; ++e) {
            const int64_t q = idx[i * kp + e];
            float f[4] = {0};
            orc_pair_feature_f32(pts + 3 * i, nrm + 3 * i, pts + 3 * q, nrm + 3 * q, f);
            spfh[i * 33 + bin(11 * (f[0] + M_PI) / (2.0 * M_PI))] += incr;
            spfh[i * 33 + 11 + bin(11 * (f[1] + 1.0) * 0.5)] += incr;
            spfh[i * 33 + 22 + bin(11 * (f[2] + 1.0) * 0.5)] += incr;
        }
    }
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < ns; ++r) {
        const int64_t i = sel ? sel[r] : r;
        float* o = out + r * 33;
        memset(o, 0, 33 * sizeof(float));
        const int c = cnt[i];
        if (c <= 1) continue;
        float sum[3] = {0, 0, 0};
        for (int e = 1; e < c; ++e) {
            const float dist = d2[i * kp + e];
            if (dist == 0.0) continue;
            const int64_t q = idx[i * kp + e];
            for (int j = 0; j < 33; ++j) {
                const float val = spfh[q * 33 + j] / dist;
                sum[j / 11] += val;
                o[j] += val;
            }
        }
        for (int j = 0; j < 3; ++j) sum[j] = sum[j] != 0.0 ? 100.0 / sum[j] : 0.0;
        for (int j = 0; j < 33; ++j) {
            o[j] *= sum[j / 11];
            o[j] += spfh[i * 33 + j];
        }
    }
    free(spfh);
}

/* nn[i] = the nearest row of t [nt, dim] to q[i] */
void orc_feature_nn_f32(const float* q, int64_t nq, const float* t, int64_t nt, int dim, int64_t* nn) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < nq; ++i) {
        float best = INFINITY;
        int64_t bi = 0;
        for (int64_t j = 0; j < nt; ++j) {
            float acc = 0.0f;
            for (int d = 0; d < dim; ++d) {
                const float diff = q[i * dim + d] - t[j * dim + d];
                acc = fmaf(diff, diff, acc);
            }
            if (acc < best) {
                best = acc;
                bi = j;
            }
        }
        nn[i] = bi;
    }
}
