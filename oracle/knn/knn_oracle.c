/* knn_oracle.c — CPU oracle of the exact k-nearest-neighbour search (o3db_knn_search) and of its two consumers,
 * PointCloud::RemoveStatisticalOutliers and PointCloud::ComputeMetrics (t/geometry/PointCloud.cpp:678-714,
 * 1805-1835; t/geometry/kernel/Metrics.cpp), written out from DESIGN.md §4.17.
 *
 * TEST INFRASTRUCTURE ONLY.  The search is a brute force over every dataset point; the cloud-wide sums follow the
 * device's fixed reduction order (orc_fixed_order_sum) so that every result is comparable bit for bit.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* canonical dist^2, d = point - query (oracle/icp_oracle.c dist2_f32) */
static inline float dist2_f32(const float* p, const float* q) {
    const float dx = p[0] - q[0];
    const float dy = p[1] - q[1];
    const float dz = p[2] - q[2];
    return fmaf(dz, dz, fmaf(dy, dy, dx * dx));
}

/* Keep the k best, ascending by dist^2, ties to the lower index, in a sorted array. */
static inline void knn_insert(int32_t* bi, float* bd, int* cnt, int k, int32_t idx, float d) {
    int n = *cnt;
    if (n == k) {
        if (d > bd[n - 1] || (d == bd[n - 1] && idx > bi[n - 1])) return;
        n = k - 1;
    }
    int pos = n;
    while (pos > 0 && (bd[pos - 1] > d || (bd[pos - 1] == d && bi[pos - 1] > idx))) {
        bd[pos] = bd[pos - 1];
        bi[pos] = bi[pos - 1];
        --pos;
    }
    bd[pos] = d;
    bi[pos] = idx;
    *cnt = n + 1;
}

#define ORC_KNN_MAX 32

/* idx / d2: [N, k'] with k' = min(k, M); a query with a non-finite coordinate gets -1 / 0 */
void orc_knn_f32(const float* points, int64_t M, const float* queries, int64_t N, int k, int32_t* idx, float* d2) {
    const int kp = (int)(k < M ? k : M);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < N; ++i) {
        int32_t bi[ORC_KNN_MAX];
        float bd[ORC_KNN_MAX];
        int cnt = 0;
        const float* q = queries + 3 * i;
        if (isfinite(q[0]) && isfinite(q[1]) && isfinite(q[2]))
            for (int64_t j = 0; j < M; ++j) knn_insert(bi, bd, &cnt, kp, (int32_t)j, dist2_f32(points + 3 * j, q));
        for (int j = 0; j < kp; ++j) {
            idx[i * kp + j] = j < cnt ? bi[j] : -1;
            d2[i * kp + j] = j < cnt ? bd[j] : 0.0f;
        }
    }
}

/* The device's sum order (knn.cu): G = clamp(ceil(n / 256), 1, 1024) blocks of 256 threads; thread t of block b adds
 * v[b*256 + t + j*G*256], j = 0, 1, ..., in turn from 0; each warp combines its 32 lanes by the xor butterfly (offsets
 * 16, 8, 4, 2, 1; lane 0's value is kept); the block adds its 8 warp sums in order from 0; the host adds the G block
 * sums in order from 0. */
double orc_fixed_order_sum(const double* v, int64_t n) {
    int64_t G = (n + 255) / 256;
    if (G < 1) G = 1;
    if (G > 1024) G = 1024;
    double total = 0;
    for (int64_t b = 0; b < G; ++b) {
        double block = 0;
        for (int w = 0; w < 8; ++w) {
            double lane[32];
            for (int l = 0; l < 32; ++l) {
                double acc = 0;
                for (int64_t i = b * 256 + w * 32 + l; i < n; i += G * 256) acc += v[i];
                lane[l] = acc;
            }
            for (int o = 16; o > 0; o >>= 1) {
                double next[32];
                for (int l = 0; l < 32; ++l) next[l] = lane[l] + lane[l ^ o];
                memcpy(lane, next, sizeof(lane));
            }
            block += lane[0];
        }
        total += block;
    }
    return total;
}

/* RemoveStatisticalOutliers from the k' nearest dist^2 of every point (d2 [n, kp]); stats = {cloud_mean, std, thr}.
 *   avg_i      = fl32(sum_j sqrtf(d2_ij), j in neighbour order) * (float)(1.0 / k')
 *   cloud_mean = (double)((float)S * (float)(1.0 / n)),  S = fixed-order f64 sum of avg_i
 *   c_i        = avg_i - (float)cloud_mean  (f32),  sq_sum = fixed-order f64 sum of (double)(c_i * c_i)
 *   std        = sqrt(sq_sum / (n - 1)),  thr = cloud_mean + std_ratio * std,  keep_i = avg_i <= (float)thr */
void orc_statistical_outliers_f32(const float* d2, int64_t n, int kp, double std_ratio, float* avg, uint8_t* mask,
                                  double* stats) {
    double* v = (double*)calloc((size_t)(n > 0 ? n : 1), sizeof(double));
    const float inv_k = (float)(1.0 / kp);
    for (int64_t i = 0; i < n; ++i) {
        float s = 0.0f;
        for (int j = 0; j < kp; ++j) s += sqrtf(d2[i * kp + j]);
        avg[i] = s * inv_k;
        v[i] = (double)avg[i];
    }
    const double cloud_mean = (double)((float)orc_fixed_order_sum(v, n) * (float)(1.0 / (double)n));
    const float mean_f = (float)cloud_mean;
    for (int64_t i = 0; i < n; ++i) {
        const float c = avg[i] - mean_f;
        v[i] = (double)(c * c);
    }
    const double sq_sum = orc_fixed_order_sum(v, n);
    const double std_dev = sqrt(sq_sum / (double)(n - 1));
    const double thr = cloud_mean + std_ratio * std_dev;
    for (int64_t i = 0; i < n; ++i) mask[i] = avg[i] <= (float)thr;
    stats[0] = cloud_mean;
    stats[1] = std_dev;
    stats[2] = thr;
    free(v);
}

/* ComputeMetrics from the 1-NN dist^2 of cloud 1 in cloud 2 (d12 [n1]) and back (d21 [n2]).  metrics: 0 Chamfer,
 * 1 Hausdorff, 2 FScore (one value per radius), as Metrics.cpp:
 *   mean = (float)S * (float)(1.0 / n), S = fixed-order f64 sum of (double)sqrtf(d2);  Chamfer = mean21 + mean12
 *   Hausdorff = max(max12, max21) of sqrtf(d2)
 *   precision = (float)(count12 * (100.0 / n1)), count = #{sqrtf(d2) < (float)radius}, recall likewise;
 *   fscore = 2 * p * r / (p + r) in f32, 0 when p + r == 0 */
void orc_metrics_f32(const float* d12, int64_t n1, const float* d21, int64_t n2, const int* metrics, int nm,
                     const float* radius, int nr, float* out) {
    const float* d[2] = {d12, d21};
    const int64_t n[2] = {n1, n2};
    float mean[2], mx[2];
    for (int k = 0; k < 2; ++k) {
        double* v = (double*)malloc((size_t)n[k] * sizeof(double));
        mx[k] = 0.0f;
        for (int64_t i = 0; i < n[k]; ++i) {
            const float s = sqrtf(d[k][i]);
            v[i] = (double)s;
            mx[k] = fmaxf(mx[k], s);
        }
        mean[k] = (float)orc_fixed_order_sum(v, n[k]) * (float)(1.0 / (double)n[k]);
        free(v);
    }
    int o = 0;
    for (int m = 0; m < nm; ++m) {
        if (metrics[m] == 0) {
            out[o++] = mean[1] + mean[0];
        } else if (metrics[m] == 1) {
            out[o++] = mx[0] > mx[1] ? mx[0] : mx[1];
        } else {
            for (int r = 0; r < nr; ++r) {
                int64_t c[2] = {0, 0};
                for (int k = 0; k < 2; ++k)
                    for (int64_t i = 0; i < n[k]; ++i) c[k] += sqrtf(d[k][i]) < radius[r];
                const float p = (float)((double)c[0] * (100.0 / (double)n1));
                const float q = (float)((double)c[1] * (100.0 / (double)n2));
                float f = 0.0f;
                if (p + q > 0) f = 2 * p * q / (p + q);
                out[o++] = f;
            }
        }
    }
}
