// ransac.cu — global registration by RANSAC on the device: pipelines::registration::
// RegistrationRANSACBasedOnCorrespondence (pipelines/registration/Registration.cpp:195-379) with the point-to-point
// estimate and the three checkers of CorrespondenceChecker.cpp, run as upstream runs it on one thread.
// DESIGN.md §4.25.
//
// The draws come from the library's random engine on the host, in batches of hypotheses; the engine is copied before
// each batch, and once the serial rule has stopped the copy is restored and only the consumed prefix redrawn.  On the
// device, in f64 (this file is compiled with -fmad=false: every op is rounded on its own):
//   hypothesis  one thread per drawn hypothesis: the sample's pairs, the Umeyama estimate without scaling (means,
//               cross-covariance, kabsch_rotation, t = mean_t - R mean_s), then the checkers; a scan of the passing
//               flags and a compaction list the passing hypotheses in draw order;
//   waves       kRanWave passing hypotheses at a time:
//     validate  one CTA per (tile of kRanTile source points, hypothesis): each thread transforms its point and finds
//               its nearest target point within the distance in the cell-sorted target (radius_visit, f64 predicate);
//               thread 0 sums the tile's matches and squared distances in index order.  CTAs past the point tiles
//               count the correspondence pairs within the distance of the transformed source;
//     select    one CTA: each thread sums its hypothesis's partials in tile order, then one thread applies upstream's
//               serial rule (stop at est_k, strict better-than, est_k from the inlier ratio of the correspondences);
//               once it has stopped, the later waves' kernels return at once;
//   emit        the [n] correspondence set of the best transformation.
// The call synchronises the stream 1 + 2 per batch + 1 times: the target index build (which also reads the input
// checks), the batch's passing count and the batch's end state, and the final read-back.
#include <cfloat>
#include <climits>
#include <cmath>
#include <random>
#include <vector>

#include "common.cuh"
#include "grid.cuh"
#include "reduce.cuh"   // kabsch_rotation, kThreads
#include "scan.cuh"

namespace o3db {

constexpr int kRanWave = 64;     // passing hypotheses per wave: the threads of the select CTA
constexpr int kRanTile = 128;    // source points per tile of the validation sums: the threads of a validate CTA
constexpr int kRanBatch = 8192;  // hypotheses drawn per batch (fewer when ransac_n is large, see batch_size)
constexpr int kRanT = 256;       // threads per CTA of the elementwise kernels

// Device state of the serial walk: upstream's best_result, est_k_global and total_validation.
struct RanState {
    double fitness;
    double rmse;
    double T[12];            // rows 0..2 of the best transformation (identity while there is none)
    long long best;          // draw index of the best hypothesis, -1 while there is none
    long long validated;     // hypotheses that passed the checkers and were validated, in draw order
    long long last;          // draw index of the last validated hypothesis, -1 for none
    int est_k;
    int done;                // a passing hypothesis at or past est_k was met, or est_k <= last + 1
};

struct RanArgs {
    const float* src;        // [n,3]
    const float* src_nrm;    // [n,3] or null
    const float* tgt;        // [m,3]
    const float* tgt_nrm;    // [m,3] or null
    const int64_t* corres;   // [K,2]
    int64_t n, m, K;
    double r2;               // max_correspondence_distance^2
    double log_conf;         // std::log(1 - confidence), on the host
    int ransac_n;
    int use_edge, use_dist, use_normal;
    double edge, dist, cos_normal;
    RadiusView view;         // the target, cell-sorted
    int tiles;               // ceil(n / kRanTile)
    int base;                // draw index of the batch's first hypothesis
    const int* draws;        // [batch][ransac_n]
    double* Ts;              // [batch][12]
    unsigned* pass;          // [batch + 1]: passing flags, then their exclusive scan
    int* list;               // [batch]: batch-local indices of the passing hypotheses, in order
    int* part_cnt;           // [tiles][kRanWave]
    double* part_err;        // [tiles][kRanWave]
    int* corr_cnt;           // [kRanWave]: correspondence pairs within the distance, zeroed by select
    RanState* state;
    int64_t* out;            // [n]
};

__device__ __forceinline__ void load3(const float* p, int64_t i, double& x, double& y, double& z) {
    x = (double)__ldg(p + 3 * i);
    y = (double)__ldg(p + 3 * i + 1);
    z = (double)__ldg(p + 3 * i + 2);
}

// The stated order of every Matrix4d * Vector4d(x, y, z, 1) product, row j: ((T_j0 x + T_j1 y) + T_j2 z) + T_j3.
// Row 3 of every hypothesis is (0, 0, 0, 1), so Transform's division by the fourth component is by exactly 1.
__device__ __forceinline__ void xform(const double* T, double x, double y, double z, double& ox, double& oy,
                                      double& oz) {
    ox = ((T[0] * x + T[1] * y) + T[2] * z) + T[3];
    oy = ((T[4] * x + T[5] * y) + T[6] * z) + T[7];
    oz = ((T[8] * x + T[9] * y) + T[10] * z) + T[11];
}

// Eigen's squaredNorm / dot of three, in the stated order ((a0 b0 + a1 b1) + a2 b2).
__device__ __forceinline__ double sq3(double x, double y, double z) { return (x * x + y * y) + z * z; }

// One thread per hypothesis of the batch: the estimate and the checkers (Registration.cpp:284-301).
__global__ void __launch_bounds__(kRanT) ransac_hypothesis_kernel(RanArgs a, int hb) {
    const int h = blockIdx.x * kRanT + threadIdx.x;
    if (h >= hb) return;
    const int* d = a.draws + (int64_t)h * a.ransac_n;
    const int64_t* c = a.corres;
    // TransformationEstimationPointToPoint: Eigen::umeyama(src, dst, false) over the sample in sample order
    double ms0 = 0, ms1 = 0, ms2 = 0, mt0 = 0, mt1 = 0, mt2 = 0;
    for (int k = 0; k < a.ransac_n; ++k) {
        double x, y, z;
        load3(a.src, c[2 * (int64_t)d[k]], x, y, z);
        ms0 += x;
        ms1 += y;
        ms2 += z;
        load3(a.tgt, c[2 * (int64_t)d[k] + 1], x, y, z);
        mt0 += x;
        mt1 += y;
        mt2 += z;
    }
    const double inv = 1.0 / (double)a.ransac_n;
    ms0 *= inv;
    ms1 *= inv;
    ms2 *= inv;
    mt0 *= inv;
    mt1 *= inv;
    mt2 *= inv;
    double H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};   // H[3 j + k] = sum (t_j - mt_j)(s_k - ms_k), then * inv
    for (int k = 0; k < a.ransac_n; ++k) {
        double sx, sy, sz, tx, ty, tz;
        load3(a.src, c[2 * (int64_t)d[k]], sx, sy, sz);
        load3(a.tgt, c[2 * (int64_t)d[k] + 1], tx, ty, tz);
        sx -= ms0;
        sy -= ms1;
        sz -= ms2;
        tx -= mt0;
        ty -= mt1;
        tz -= mt2;
        H[0] += tx * sx;
        H[1] += tx * sy;
        H[2] += tx * sz;
        H[3] += ty * sx;
        H[4] += ty * sy;
        H[5] += ty * sz;
        H[6] += tz * sx;
        H[7] += tz * sy;
        H[8] += tz * sz;
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) H[k] *= inv;
    double R[9];
    kabsch_rotation(H, R);
    double T[12];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        T[4 * j] = R[3 * j];
        T[4 * j + 1] = R[3 * j + 1];
        T[4 * j + 2] = R[3 * j + 2];
    }
    T[3] = mt0 - ((R[0] * ms0 + R[1] * ms1) + R[2] * ms2);
    T[7] = mt1 - ((R[3] * ms0 + R[4] * ms1) + R[5] * ms2);
    T[11] = mt2 - ((R[6] * ms0 + R[7] * ms1) + R[8] * ms2);
    double* out = a.Ts + 12 * (int64_t)h;
#pragma unroll
    for (int k = 0; k < 12; ++k) out[k] = T[k];

    bool ok = true;
    if (a.use_edge)   // CorrespondenceCheckerBasedOnEdgeLength (CorrespondenceChecker.cpp:19-40)
        for (int i = 0; i < a.ransac_n && ok; ++i) {
            double si0, si1, si2, ti0, ti1, ti2;
            load3(a.src, c[2 * (int64_t)d[i]], si0, si1, si2);
            load3(a.tgt, c[2 * (int64_t)d[i] + 1], ti0, ti1, ti2);
            for (int j = i + 1; j < a.ransac_n && ok; ++j) {
                double sx, sy, sz, tx, ty, tz;
                load3(a.src, c[2 * (int64_t)d[j]], sx, sy, sz);
                load3(a.tgt, c[2 * (int64_t)d[j] + 1], tx, ty, tz);
                const double ds = sqrt(sq3(si0 - sx, si1 - sy, si2 - sz));
                const double dt = sqrt(sq3(ti0 - tx, ti1 - ty, ti2 - tz));
                ok = !(ds < dt * a.edge || dt < ds * a.edge);
            }
        }
    if (a.use_dist)   // CorrespondenceCheckerBasedOnDistance (:42-57)
        for (int k = 0; k < a.ransac_n && ok; ++k) {
            double x, y, z, px, py, pz, tx, ty, tz;
            load3(a.src, c[2 * (int64_t)d[k]], x, y, z);
            xform(T, x, y, z, px, py, pz);
            load3(a.tgt, c[2 * (int64_t)d[k] + 1], tx, ty, tz);
            ok = !(sqrt(sq3(tx - px, ty - py, tz - pz)) > a.dist);
        }
    if (a.use_normal && a.src_nrm && a.tgt_nrm)   // CorrespondenceCheckerBasedOnNormal (:59-80)
        for (int k = 0; k < a.ransac_n && ok; ++k) {
            double x, y, z, tx, ty, tz;
            load3(a.src_nrm, c[2 * (int64_t)d[k]], x, y, z);
            // the rotated normal: ((T_j0 x + T_j1 y) + T_j2 z) + T_j3 * 0, and adding a zero changes no comparison
            const double nx = (T[0] * x + T[1] * y) + T[2] * z;
            const double ny = (T[4] * x + T[5] * y) + T[6] * z;
            const double nz = (T[8] * x + T[9] * y) + T[10] * z;
            load3(a.tgt_nrm, c[2 * (int64_t)d[k] + 1], tx, ty, tz);
            ok = !((tx * nx + ty * ny) + tz * nz < a.cos_normal);
        }
    a.pass[h] = ok;
}

// After the scan: the batch-local indices of the passing hypotheses, in order.
__global__ void __launch_bounds__(kRanT) ransac_compact_kernel(RanArgs a, int hb) {
    const int h = blockIdx.x * kRanT + threadIdx.x;
    if (h < hb && a.pass[h + 1] != a.pass[h]) a.list[a.pass[h]] = h;
}

// The nearest target point of source point i under T: d^2 = ((dx^2 + dy^2) + dz^2) in f64 from the transformed point,
// a match when d^2 < r^2 (SearchHybrid's strict bound), ties to the lowest index.  Returns the index or -1.
// The cells are binned from the query rounded to f32: view.rr = r (1 + 1e-5) and lo_bound / hi_bound's 2 ulp of |q|
// cover that rounding (half an ulp) as well as the rounding of the box ends (DESIGN.md §4.25).
__device__ __forceinline__ int nearest(const RanArgs& a, const double* T, int64_t i, double& best_d2) {
    double x, y, z, px, py, pz;
    load3(a.src, i, x, y, z);
    xform(T, x, y, z, px, py, pz);
    const float4 q = make_float4((float)px, (float)py, (float)pz, 0.f);
    double d2 = 0.0;
    int idx = -1, best = -1;
    best_d2 = INFINITY;
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

// Wave w: grid = (tiles + ceil(K / kRanTile), hypotheses of the wave), block = kRanTile.
// blockIdx.x < tiles: GetRegistrationResultAndCorrespondences (Registration.cpp:74-104) over one tile of the
// transformed source, its match count and sum of d^2 in index order; beyond: EvaluateInlierCorrespondenceRatio
// (:106-125) over one tile of the pairs.
__global__ void __launch_bounds__(kRanTile) ransac_validate_kernel(RanArgs a, int w) {
    __shared__ double s_d2[kRanTile];
    __shared__ bool s_in[kRanTile];
    if (*(volatile int*)&a.state->done) return;
    const int slot = blockIdx.y;
    double T[12];
    const double* Th = a.Ts + 12 * (int64_t)a.list[w * kRanWave + slot];
#pragma unroll
    for (int k = 0; k < 12; ++k) T[k] = Th[k];
    if ((int)blockIdx.x >= a.tiles) {
        const int64_t k = (int64_t)(blockIdx.x - a.tiles) * kRanTile + threadIdx.x;
        bool in = false;
        if (k < a.K) {
            double x, y, z, px, py, pz, tx, ty, tz;
            load3(a.src, a.corres[2 * k], x, y, z);
            xform(T, x, y, z, px, py, pz);
            load3(a.tgt, a.corres[2 * k + 1], tx, ty, tz);
            in = sq3(px - tx, py - ty, pz - tz) < a.r2;
        }
        const int cnt = __syncthreads_count(in);
        if (threadIdx.x == 0 && cnt) atomicAdd(&a.corr_cnt[slot], cnt);
        return;
    }
    const int64_t i = (int64_t)blockIdx.x * kRanTile + threadIdx.x;
    double d2 = 0.0;
    const bool in = i < a.n && nearest(a, T, i, d2) >= 0;
    s_d2[threadIdx.x] = d2;
    s_in[threadIdx.x] = in;
    __syncthreads();
    if (threadIdx.x != 0) return;
    const int m = (int)min((int64_t)kRanTile, a.n - (int64_t)blockIdx.x * kRanTile);
    int cnt = 0;
    double err = 0.0;
    for (int j = 0; j < m; ++j)
        if (s_in[j]) {
            ++cnt;
            err += s_d2[j];
        }
    const size_t o = (size_t)blockIdx.x * kRanWave + slot;
    a.part_cnt[o] = cnt;
    a.part_err[o] = err;
}

// Wave w of cw hypotheses: one CTA of kRanWave threads.  Sums each hypothesis's partials in tile order, then walks the
// wave in draw order with the serial rule of Registration.cpp:279-341.
__global__ void __launch_bounds__(kRanWave) ransac_select_kernel(RanArgs a, int w, int cw) {
    __shared__ double s_fit[kRanWave], s_rmse[kRanWave], s_ratio[kRanWave];
    RanState* st = a.state;
    if (*(volatile int*)&st->done) return;
    const int k = threadIdx.x;
    if (k < cw) {
        long long cnt = 0;
        double err = 0.0;
#pragma unroll 16   // loads run ahead of the ordered sum, which is latency-bound otherwise
        for (int t = 0; t < a.tiles; ++t) {
            const size_t o = (size_t)t * kRanWave + k;
            cnt += a.part_cnt[o];
            err += a.part_err[o];
        }
        s_fit[k] = cnt ? (double)cnt / (double)a.n : 0.0;
        s_rmse[k] = cnt ? sqrt(err / (double)cnt) : 0.0;
        s_ratio[k] = (double)a.corr_cnt[k] / (double)a.K;
        a.corr_cnt[k] = 0;
    }
    __syncthreads();
    if (k != 0) return;
    RanState s = *st;
    for (int j = 0; j < cw; ++j) {
        const int h = a.list[w * kRanWave + j];
        const long long i = (long long)a.base + h;
        if (i >= s.est_k) {
            s.done = 1;
            break;
        }
        const double fit = s_fit[j], rmse = s_rmse[j];
        if (fit > s.fitness || (fit == s.fitness && rmse < s.rmse)) {   // IsBetterRANSACThan
            s.fitness = fit;
            s.rmse = rmse;
            s.best = i;
            const double* Th = a.Ts + 12 * (int64_t)h;
            for (int q = 0; q < 12; ++q) s.T[q] = Th[q];
            double est = a.log_conf / log(1.0 - pow(s_ratio[j], (double)a.ransac_n));
            if (est < 0) est = (double)s.est_k;   // est_k_local == est_k_global on one thread
            if (est < (double)s.est_k) s.est_k = (int)ceil(est);
        }
        ++s.validated;
        s.last = i;
    }
    if (s.est_k <= s.last + 1) s.done = 1;
    *st = s;
}

// The correspondence set of the best transformation: out[i] = its nearest target point within the distance, or -1.
__global__ void __launch_bounds__(kRanT) ransac_emit_kernel(RanArgs a) {
    const int64_t i = (int64_t)blockIdx.x * kRanT + threadIdx.x;
    if (i >= a.n) return;
    const RanState* st = a.state;
    double d2;
    a.out[i] = st->best >= 0 ? nearest(a, st->T, i, d2) : -1;
}

// Input checks: bad[0] = 1 for a non-finite source coordinate, bad[1] = 1 for a pair outside [0, n) x [0, m).
__global__ void __launch_bounds__(kRanT) ransac_check_kernel(RanArgs a, unsigned* bad) {
    const int64_t i = (int64_t)blockIdx.x * kRanT + threadIdx.x;
    if (i < a.n) flag_nonfinite(a.src, i, bad);
    if (i < a.K) {
        const int64_t s = a.corres[2 * i], t = a.corres[2 * i + 1];
        if (s < 0 || s >= a.n || t < 0 || t >= a.m) atomicOr(bad + 1, 1u);
    }
}

// nonfinite = 1 when any target coordinate is NaN or infinite (grid_index_finite)
__global__ void __launch_bounds__(kThreads) ransac_finite_kernel(const float* __restrict__ pts, int64_t n,
                                                                 unsigned* __restrict__ nonfinite) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) flag_nonfinite(pts, i, nonfinite);
}

// Hypotheses per batch: kRanBatch, fewer for large samples so that a batch's draws stay within 2^22 ints.
int batch_size(int ransac_n) { return std::max(1, std::min(kRanBatch, (1 << 22) / ransac_n)); }

}  // namespace o3db

using namespace o3db;

extern "C" {

int o3db_random_uniform_ints(int low, int high, int64_t count, int* out_host) {
    // UniformIntGenerator<int> (utility/Random.h:63-90)
    O3DB_REQUIRE(low >= 0, "low must be > 0, but got %d.", low);
    O3DB_REQUIRE(low <= high, "low must be <= high, but got low=%d and high=%d.", low, high);
    O3DB_REQUIRE(count >= 0 && (count == 0 || out_host), "o3db_random_uniform_ints: bad count or null output");
    std::uniform_int_distribution<int> dist(low, high);
    std::lock_guard<std::mutex> lock(random_mutex());
    std::mt19937& engine = random_engine();
    for (int64_t k = 0; k < count; ++k) out_host[k] = dist(engine);
    return O3DB_OK;
}

int o3db_registration_ransac(const float* source_dev, const float* source_normals_dev, int64_t n,
                             const float* target_dev, const float* target_normals_dev, int64_t m,
                             const int64_t* correspondences_dev, int64_t K, double max_correspondence_distance,
                             int ransac_n, int max_iteration, double confidence,
                             const o3db_ransac_checkers* checkers, double* transformation_host,
                             int64_t* correspondence_set_dev, o3db_ransac_stats* stats, void* stream) {
    O3DB_REQUIRE(transformation_host, "o3db_registration_ransac: null transformation");
    O3DB_REQUIRE(n >= 0 && n < INT_MAX && m >= 0 && m < INT_MAX && K >= 0 && K < INT_MAX,
                 "o3db_registration_ransac: point and correspondence counts must be below 2^31 - 1 (got n=%lld, "
                 "m=%lld, K=%lld)", (long long)n, (long long)m, (long long)K);
    O3DB_REQUIRE(n == 0 || (source_dev && correspondence_set_dev),
                 "o3db_registration_ransac: null source or correspondence set");
    O3DB_REQUIRE(!std::isnan(max_correspondence_distance) && !std::isinf(max_correspondence_distance),
                 "RegistrationRANSAC: max_correspondence_distance must be finite (got %g)",
                 max_correspondence_distance);
    cudaStream_t st = (cudaStream_t)stream;
    for (int k = 0; k < 16; ++k) transformation_host[k] = k % 5 == 0 ? 1.0 : 0.0;
    if (stats) *stats = o3db_ransac_stats{0, 0, -1, 0.0, 0.0};
    // Registration.cpp:354-357 and an empty loop: the identity, no correspondences, no draws
    if (ransac_n < 3 || K < ransac_n || max_correspondence_distance <= 0.0 || max_iteration <= 0) {
        if (n > 0) O3DB_CUDA_CHECK(cudaMemsetAsync(correspondence_set_dev, 0xff, (size_t)n * sizeof(int64_t), st));
        return O3DB_OK;
    }
    O3DB_REQUIRE(target_dev && correspondences_dev, "o3db_registration_ransac: null target or correspondences");
    configure_memory_pool();
    const int B = batch_size(ransac_n);
    const int tiles = (int)ceil_div(n, kRanTile);
    const int ctiles = (int)ceil_div(K, kRanTile);
    DevPtr<RanState> state;
    DevPtr<int> draws, list, part_cnt, corr_cnt;
    DevPtr<double> Ts, part_err;
    DevPtr<unsigned> pass, bad;
    if (int rc = dev_alloc(state, 1, st)) return rc;
    if (int rc = dev_alloc(draws, (size_t)B * ransac_n, st)) return rc;
    if (int rc = dev_alloc(list, (size_t)B, st)) return rc;
    if (int rc = dev_alloc(Ts, (size_t)B * 12, st)) return rc;
    if (int rc = dev_alloc(pass, (size_t)B + 1 + ceil_div(B, kScanTile), st)) return rc;
    if (int rc = dev_alloc(part_cnt, (size_t)std::max(tiles, 1) * kRanWave, st)) return rc;
    if (int rc = dev_alloc(part_err, (size_t)std::max(tiles, 1) * kRanWave, st)) return rc;
    if (int rc = dev_alloc(corr_cnt, kRanWave, st)) return rc;
    if (int rc = dev_alloc(bad, 2, st)) return rc;
    struct Readback {
        RanState state;
        unsigned bad[2];
        unsigned passed;
    };
    PinnedPtr<Readback> h = pinned_block<Readback>();
    std::vector<int> hdraws((size_t)B * ransac_n);
    if (!h) {
        set_last_error("o3db_registration_ransac: out of pinned host memory");
        return O3DB_ERR_CUDA;
    }

    RanArgs a{};
    a.src = source_dev;
    a.src_nrm = source_normals_dev;
    a.tgt = target_dev;
    a.tgt_nrm = target_normals_dev;
    a.corres = correspondences_dev;
    a.n = n;
    a.m = m;
    a.K = K;
    a.r2 = max_correspondence_distance * max_correspondence_distance;
    a.log_conf = std::log(1.0 - confidence);
    a.ransac_n = ransac_n;
    if (checkers) {
        a.use_edge = checkers->use_edge_length != 0;
        a.use_dist = checkers->use_distance != 0;
        a.use_normal = checkers->use_normal != 0;
        a.edge = checkers->edge_length_similarity;
        a.dist = checkers->distance_threshold;
        a.cos_normal = checkers->cos_normal_angle_threshold;
    }
    a.tiles = tiles;
    a.draws = draws.get();
    a.Ts = Ts.get();
    a.pass = pass.get();
    a.list = list.get();
    a.part_cnt = part_cnt.get();
    a.part_err = part_err.get();
    a.corr_cnt = corr_cnt.get();
    a.state = state.get();
    a.out = correspondence_set_dev;

    O3DB_CUDA_CHECK(cudaMemsetAsync(bad.get(), 0, 2 * sizeof(unsigned), st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(corr_cnt.get(), 0, kRanWave * sizeof(int), st));
    ransac_check_kernel<<<(unsigned)ceil_div(std::max(n, K), kRanT), kRanT, 0, st>>>(a, bad.get());
    O3DB_LAUNCH_CHECK();
    O3DB_CUDA_CHECK(cudaMemcpyAsync(h->bad, bad.get(), 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    // the target's cell-sorted index; its synchronise also completes the input checks above
    o3db_nns index;
    if (int rc = grid_index_finite(&index, target_dev, m, max_correspondence_distance, ransac_finite_kernel,
                                   "RegistrationRANSAC: the target point cloud has non-finite coordinates; remove them "
                                   "first with remove_non_finite_points",
                                   st))
        return rc;
    O3DB_REQUIRE(!h->bad[0], "RegistrationRANSAC: the source point cloud has non-finite coordinates; remove them first "
                             "with remove_non_finite_points");
    O3DB_REQUIRE(!h->bad[1], "RegistrationRANSAC: a correspondence lies outside [0, %lld) x [0, %lld)", (long long)n,
                 (long long)m);
    // as remove.cu: rr >= the radius after its rounding to f32; a radius beyond the f32 range bins every point
    const double rr = max_correspondence_distance * (1.0 + 1e-5);
    a.view = RadiusView{index.g, index.pts4.get(), index.cell_start.get(),
                        rr < (double)FLT_MAX ? (float)rr : INFINITY};

    h->state = RanState{};
    h->state.T[0] = h->state.T[5] = h->state.T[10] = 1.0;
    h->state.best = -1;
    h->state.last = -1;
    h->state.est_k = max_iteration;
    O3DB_CUDA_CHECK(cudaMemcpyAsync(state.get(), &h->state, sizeof(RanState), cudaMemcpyHostToDevice, st));

    // RANSACCorrespondenceReduction::operator() (Registration.cpp:279-341) on one thread, B hypotheses at a time
    std::uniform_int_distribution<int> dist(0, (int)K - 1);
    std::lock_guard<std::mutex> lock(random_mutex());
    std::mt19937& engine = random_engine();
    for (int base = 0; base < max_iteration; base += B) {
        const int hb = std::min(B, max_iteration - base);
        const std::mt19937 saved = engine;
        for (int64_t k = 0; k < (int64_t)hb * ransac_n; ++k) hdraws[k] = dist(engine);
        O3DB_CUDA_CHECK(cudaMemcpyAsync(draws.get(), hdraws.data(), (size_t)hb * ransac_n * sizeof(int),
                                        cudaMemcpyHostToDevice, st));
        a.base = base;
        const unsigned grid = (unsigned)ceil_div(hb, kRanT);
        ransac_hypothesis_kernel<<<grid, kRanT, 0, st>>>(a, hb);
        O3DB_LAUNCH_CHECK();
        if (int rc = exclusive_scan_u32(pass.get(), hb, pass.get() + B + 1, st)) return rc;
        ransac_compact_kernel<<<grid, kRanT, 0, st>>>(a, hb);
        O3DB_LAUNCH_CHECK();
        O3DB_CUDA_CHECK(cudaMemcpyAsync(&h->passed, pass.get() + hb, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
        O3DB_CUDA_CHECK(cudaStreamSynchronize(st));   // the batch's passing count sizes its waves
        const int passed = (int)h->passed;
        for (int w = 0; w * kRanWave < passed; ++w) {
            const int cw = std::min(kRanWave, passed - w * kRanWave);
            ransac_validate_kernel<<<dim3((unsigned)(tiles + ctiles), (unsigned)cw), kRanTile, 0, st>>>(a, w);
            O3DB_LAUNCH_CHECK();
            ransac_select_kernel<<<1, kRanWave, 0, st>>>(a, w, cw);
            O3DB_LAUNCH_CHECK();
        }
        O3DB_CUDA_CHECK(cudaMemcpyAsync(&h->state, state.get(), sizeof(RanState), cudaMemcpyDeviceToHost, st));
        O3DB_CUDA_CHECK(cudaStreamSynchronize(st));   // the batch's end state: stopped or not
        const RanState& s = h->state;
        const int end = base + hb;
        if (s.done || s.est_k <= end) {
            // the first hypothesis not drawn: every one between the last validated one and est_k was drawn
            const int stop = (int)std::min<long long>(end, std::max<long long>(s.last + 1, s.est_k));
            engine = saved;
            for (int64_t k = 0; k < (int64_t)(stop - base) * ransac_n; ++k) (void)dist(engine);
            if (stats) stats->drawn = stop;
            break;
        }
        if (stats) stats->drawn = end;
    }
    if (n > 0) {
        ransac_emit_kernel<<<(unsigned)ceil_div(n, kRanT), kRanT, 0, st>>>(a);
        O3DB_LAUNCH_CHECK();
    }
    O3DB_CUDA_CHECK(cudaMemcpyAsync(&h->state, state.get(), sizeof(RanState), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));   // the result
    const RanState& s = h->state;
    for (int k = 0; k < 12; ++k) transformation_host[k] = s.T[k];
    if (stats) {
        stats->validated = s.validated;
        stats->best_index = s.best;
        stats->fitness = s.fitness;
        stats->inlier_rmse = s.rmse;
    }
    return O3DB_OK;
}

}  // extern "C"
