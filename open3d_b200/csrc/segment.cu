// segment.cu — RANSAC plane segmentation on the device: geometry::PointCloud::SegmentPlane
// (geometry/PointCloudSegmentation.cpp:157-279), which upstream's tensor PointCloud::SegmentPlane runs on the host.
// DESIGN.md §4.21.
//
// The samples are drawn on the host from the library's random engine, all num_iterations of them, as upstream does.
// On the device, in f64 with every op rounded and no FMA:
//   hypothesis  one thread per sample: ComputeTrianglePlane for ransac_n == 3, else GetPlaneFromPoints;
//   waves       kSegWave hypotheses at a time:
//     score     one CTA per tile of kSegTile points, staged in shared memory as f64; each thread owns one hypothesis
//               and walks the tile in index order, keeping its inlier count and squared-distance sum in registers;
//               the per-tile partials go to a [tiles][kSegWave] buffer;
//     select    one CTA: each thread sums its hypothesis's partials in tile order, then one thread applies upstream's
//               serial rule (skip once evaluated > break, strict better-than, break from the probability) to the
//               wave in index order.  Once the rule has fired, the later waves' kernels return at once;
//   inliers     ballot / scan / emit of the points within the threshold of the best hypothesis, in index order;
//   refit       GetPlaneFromPoints over those inliers: per-tile centroid sums, the centroid, per-tile second moments,
//               the plane, every sum in the tile order of the score pass.
// The number of launches depends on n and num_iterations only; the call synchronises once, to read the inlier count.
#include <climits>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "scan.cuh"

namespace o3db {

constexpr int kSegWave = 128;    // hypotheses per wave: the threads of a score CTA
constexpr int kSegTile = 1024;   // points per tile of the score and refit sums
constexpr int kSegT = 256;       // threads per CTA of the inlier and hypothesis kernels

// Device state of the serial walk, upstream's RANSACResult result, break_iteration and iteration_count.
struct SegState {
    double fitness;
    double rmse;
    unsigned long long brk;
    unsigned long long count;
    long long best;      // index of the best hypothesis, -1 while there is none
    int done;            // count > brk: every later hypothesis is skipped
    double centroid[3];  // of the final inliers, between the two refit passes
};

struct SegArgs {
    const float* pts;        // [n,3]
    int64_t n;
    double thr;
    double probability;
    int ransac_n;
    int num_iterations;
    int tiles;               // ceil(n / kSegTile)
    const int64_t* samples;  // [num_iterations][ransac_n]
    double* planes;          // [num_iterations][4]
    int* part_cnt;           // [tiles][kSegWave]
    double* part_err;        // [tiles][kSegWave]
    double* part_sum;        // [tiles][6]: refit sums
    SegState* state;
    unsigned* counts;        // [ceil(n / kSegT) + 1]: inlier counts per CTA, then their exclusive scan
    int64_t* inliers;        // [n]
    double* plane_out;       // [4]
};

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }

// Eigen's Vector4d::dot(a, b) for plane · (x, y, z, 1): two packets of two, added, then the halves, so
// (a·x + c·z) + (b·y + d).
__device__ __forceinline__ double plane_dist(const double* pl, double x, double y, double z) {
    return fabs(dadd(dadd(dmul(pl[0], x), dmul(pl[2], z)), dadd(dmul(pl[1], y), pl[3])));
}

// Eigen's Vector3d::dot, a packet of two and the third term: (a0·b0 + a1·b1) + a2·b2.
__device__ __forceinline__ double dot3(double a0, double a1, double a2, double b0, double b1, double b2) {
    return dadd(dadd(dmul(a0, b0), dmul(a1, b1)), dmul(a2, b2));
}

// abc / |abc| and d = -abc · p (TriangleMesh.cpp:1254-1261, PointCloudSegmentation.cpp:147-154); (0,0,0,0) when
// |abc| == 0.
__device__ __forceinline__ void finish_plane(double a, double b, double c, double p0, double p1, double p2,
                                             double* out) {
    const double norm = __dsqrt_rn(dot3(a, b, c, a, b, c));
    if (norm == 0.0) {
        out[0] = out[1] = out[2] = out[3] = 0.0;
        return;
    }
    a = __ddiv_rn(a, norm);
    b = __ddiv_rn(b, norm);
    c = __ddiv_rn(c, norm);
    out[0] = a;
    out[1] = b;
    out[2] = c;
    out[3] = -dot3(a, b, c, p0, p1, p2);
}

// GetPlaneFromPoints (PointCloudSegmentation.cpp:131-154) from the centroid and the six second-moment sums.
__device__ void plane_from_moments(const double* cen, double xx, double xy, double xz, double yy, double yz,
                                   double zz, double* out) {
    const double det_x = dsub(dmul(yy, zz), dmul(yz, yz));
    const double det_y = dsub(dmul(xx, zz), dmul(xz, xz));
    const double det_z = dsub(dmul(xx, yy), dmul(xy, xy));
    double a, b, c;
    if (det_x > det_y && det_x > det_z) {
        a = det_x;
        b = dsub(dmul(xz, yz), dmul(xy, zz));
        c = dsub(dmul(xy, yz), dmul(xz, yy));
    } else if (det_y > det_z) {
        a = dsub(dmul(xz, yz), dmul(xy, zz));
        b = det_y;
        c = dsub(dmul(xy, xz), dmul(yz, xx));
    } else {
        a = dsub(dmul(xy, yz), dmul(xz, yy));
        b = dsub(dmul(xy, xz), dmul(yz, xx));
        c = det_z;
    }
    finish_plane(a, b, c, cen[0], cen[1], cen[2], out);
}

__device__ __forceinline__ void load_point(const float* pts, int64_t i, double& x, double& y, double& z) {
    x = (double)__ldg(pts + 3 * i);
    y = (double)__ldg(pts + 3 * i + 1);
    z = (double)__ldg(pts + 3 * i + 2);
}

// One thread per hypothesis: the plane through its sampled points (PointCloudSegmentation.cpp:219-226).
__global__ void __launch_bounds__(kSegT) segment_hypothesis_kernel(SegArgs a) {
    const int h = blockIdx.x * kSegT + threadIdx.x;
    if (h >= a.num_iterations) return;
    const int64_t* s = a.samples + (int64_t)h * a.ransac_n;
    double* out = a.planes + 4 * (int64_t)h;
    if (a.ransac_n == 3) {   // ComputeTrianglePlane (TriangleMesh.cpp:1248-1262)
        double x0, y0, z0, x1, y1, z1, x2, y2, z2;
        load_point(a.pts, s[0], x0, y0, z0);
        load_point(a.pts, s[1], x1, y1, z1);
        load_point(a.pts, s[2], x2, y2, z2);
        const double e0x = dsub(x1, x0), e0y = dsub(y1, y0), e0z = dsub(z1, z0);
        const double e1x = dsub(x2, x0), e1y = dsub(y2, y0), e1z = dsub(z2, z0);
        finish_plane(dsub(dmul(e0y, e1z), dmul(e0z, e1y)), dsub(dmul(e0z, e1x), dmul(e0x, e1z)),
                     dsub(dmul(e0x, e1y), dmul(e0y, e1x)), x0, y0, z0, out);
        return;
    }
    double cen[3] = {0.0, 0.0, 0.0};   // GetPlaneFromPoints over the sample, in sample order
    for (int k = 0; k < a.ransac_n; ++k) {
        double x, y, z;
        load_point(a.pts, s[k], x, y, z);
        cen[0] = dadd(cen[0], x);
        cen[1] = dadd(cen[1], y);
        cen[2] = dadd(cen[2], z);
    }
    const double m = (double)a.ransac_n;
    cen[0] = __ddiv_rn(cen[0], m);
    cen[1] = __ddiv_rn(cen[1], m);
    cen[2] = __ddiv_rn(cen[2], m);
    double xx = 0, xy = 0, xz = 0, yy = 0, yz = 0, zz = 0;
    for (int k = 0; k < a.ransac_n; ++k) {
        double x, y, z;
        load_point(a.pts, s[k], x, y, z);
        const double rx = dsub(x, cen[0]), ry = dsub(y, cen[1]), rz = dsub(z, cen[2]);
        xx = dadd(xx, dmul(rx, rx));
        xy = dadd(xy, dmul(rx, ry));
        xz = dadd(xz, dmul(rx, rz));
        yy = dadd(yy, dmul(ry, ry));
        yz = dadd(yz, dmul(ry, rz));
        zz = dadd(zz, dmul(rz, rz));
    }
    plane_from_moments(cen, xx, xy, xz, yy, yz, zz, out);
}

// Stages tile t's points in shared memory as f64; returns the number of points in the tile.
__device__ __forceinline__ int stage_tile(const SegArgs& a, int t, double* sx, double* sy, double* sz) {
    const int64_t lo = (int64_t)t * kSegTile;
    const int m = (int)min((int64_t)kSegTile, a.n - lo);
    for (int j = threadIdx.x; j < m; j += blockDim.x) load_point(a.pts, lo + j, sx[j], sy[j], sz[j]);
    __syncthreads();
    return m;
}

// Wave w: grid = tiles, block = kSegWave.  EvaluateRANSACBasedOnDistance (PointCloudSegmentation.cpp:78-107) over one
// tile: count and error in index order.
__global__ void __launch_bounds__(kSegWave) segment_score_kernel(SegArgs a, int w) {
    __shared__ double sx[kSegTile], sy[kSegTile], sz[kSegTile];
    if (*(volatile int*)&a.state->done) return;
    const int h = w * kSegWave + threadIdx.x;
    const int m = stage_tile(a, blockIdx.x, sx, sy, sz);
    if (h >= a.num_iterations) return;
    double pl[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) pl[k] = a.planes[4 * (int64_t)h + k];
    int cnt = 0;
    double err = 0.0;
#pragma unroll 4
    for (int j = 0; j < m; ++j) {
        const double d = plane_dist(pl, sx[j], sy[j], sz[j]);
        const bool in = d < a.thr;
        cnt += in;
        err = in ? dadd(err, dmul(d, d)) : err;
    }
    const size_t o = (size_t)blockIdx.x * kSegWave + threadIdx.x;
    a.part_cnt[o] = cnt;
    a.part_err[o] = err;
}

// size_t(v) as x86-64 code compiled by gcc converts it: v is min(q, num_iterations) >= -0, or -inf or NaN when
// fitness^ransac_n rounds 1 - it to 1, and those give 2^63 there (cvttsd2si's integer indefinite).
__device__ __forceinline__ unsigned long long host_size_t(double v) {
    return v >= 0.0 ? (unsigned long long)v : 1ull << 63;
}

// Wave w: one CTA of kSegWave threads.  Sums each hypothesis's partials in tile order, then walks the wave with the
// serial rule of PointCloudSegmentation.cpp:200-253.
__global__ void __launch_bounds__(kSegWave) segment_select_kernel(SegArgs a, int w) {
    __shared__ double s_fit[kSegWave], s_rmse[kSegWave];
    __shared__ bool s_valid[kSegWave];
    SegState* st = a.state;
    if (*(volatile int*)&st->done) return;
    const int h = w * kSegWave + threadIdx.x;
    if (h < a.num_iterations) {
        long long cnt = 0;
        double err = 0.0;
#pragma unroll 16   // loads run ahead of the ordered sum, which is latency-bound otherwise
        for (int t = 0; t < a.tiles; ++t) {
            const size_t o = (size_t)t * kSegWave + threadIdx.x;
            cnt += a.part_cnt[o];
            err = dadd(err, a.part_err[o]);
        }
        const double* pl = a.planes + 4 * (int64_t)h;
        s_valid[threadIdx.x] = !(pl[0] == 0.0 && pl[1] == 0.0 && pl[2] == 0.0 && pl[3] == 0.0);   // isZero(0)
        s_fit[threadIdx.x] = cnt ? __ddiv_rn((double)cnt, (double)a.n) : 0.0;
        s_rmse[threadIdx.x] = cnt ? __dsqrt_rn(__ddiv_rn(err, (double)cnt)) : 0.0;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    const int hw = min(kSegWave, a.num_iterations - w * kSegWave);
    SegState s = *st;
    for (int k = 0; k < hw; ++k) {
        if (s.count > s.brk) break;
        if (!s_valid[k]) continue;
        const double fit = s_fit[k], rmse = s_rmse[k];
        if (fit > s.fitness || (fit == s.fitness && rmse < s.rmse)) {
            s.fitness = fit;
            s.rmse = rmse;
            s.best = w * kSegWave + k;
            if (fit < 1.0) {
                const double q = log(1.0 - a.probability) / log(1.0 - pow(fit, (double)a.ransac_n));
                const double n_it = (double)a.num_iterations;
                s.brk = host_size_t(n_it < q ? n_it : q);   // std::min(q, n_it)
            } else {
                s.brk = 0;
            }
        }
        ++s.count;
    }
    s.done = s.count > s.brk;
    *st = s;
}

__device__ __forceinline__ const double* best_plane(const SegArgs& a) {
    const long long b = a.state->best;
    return b >= 0 ? a.planes + 4 * b : nullptr;
}

__device__ __forceinline__ bool final_inlier(const SegArgs& a, const double* pl, int64_t i) {
    if (!pl || i >= a.n) return false;
    double x, y, z;
    load_point(a.pts, i, x, y, z);
    return plane_dist(pl, x, y, z) < a.thr;
}

// Final inliers (PointCloudSegmentation.cpp:256-268): a count per CTA, then, after the scan, the indices.
__global__ void __launch_bounds__(kSegT) segment_count_kernel(SegArgs a) {
    __shared__ unsigned s_warp[kSegT / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned m = __ballot_sync(0xffffffffu, final_inlier(a, best_plane(a), (int64_t)blockIdx.x * kSegT +
                                                                                   threadIdx.x));
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned t = 0;
#pragma unroll
        for (int k = 0; k < kSegT / 32; ++k) t += s_warp[k];
        a.counts[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(kSegT) segment_emit_kernel(SegArgs a) {
    __shared__ unsigned s_warp[kSegT / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t i = (int64_t)blockIdx.x * kSegT + threadIdx.x;
    const bool ok = final_inlier(a, best_plane(a), i);
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    if (!ok) return;
    unsigned base = 0;
#pragma unroll
    for (int k = 0; k < kSegT / 32; ++k) base += k < warp ? s_warp[k] : 0u;
    a.inliers[(size_t)a.counts[blockIdx.x] + base + __popc(m & ((1u << lane) - 1u))] = i;
}

// Refit pass over tile blockIdx.x (grid = tiles, block = kSegWave): the final inliers staged with their flags, then
// one thread sums them in index order.  pass 0: x, y, z; pass 1: the six second moments about the centroid.
__global__ void __launch_bounds__(kSegWave) segment_refit_tile_kernel(SegArgs a, int pass) {
    __shared__ double sx[kSegTile], sy[kSegTile], sz[kSegTile];
    __shared__ bool sin[kSegTile];
    const double* pl = best_plane(a);
    const int m = stage_tile(a, blockIdx.x, sx, sy, sz);
    for (int j = threadIdx.x; j < m; j += kSegWave) sin[j] = pl && plane_dist(pl, sx[j], sy[j], sz[j]) < a.thr;
    __syncthreads();
    if (threadIdx.x != 0) return;
    double* out = a.part_sum + 6 * (size_t)blockIdx.x;
    if (pass == 0) {
        double cx = 0.0, cy = 0.0, cz = 0.0;
        for (int j = 0; j < m; ++j)
            if (sin[j]) {
                cx = dadd(cx, sx[j]);
                cy = dadd(cy, sy[j]);
                cz = dadd(cz, sz[j]);
            }
        out[0] = cx;
        out[1] = cy;
        out[2] = cz;
        return;
    }
    const double c0 = a.state->centroid[0], c1 = a.state->centroid[1], c2 = a.state->centroid[2];
    double xx = 0, xy = 0, xz = 0, yy = 0, yz = 0, zz = 0;
    for (int j = 0; j < m; ++j)
        if (sin[j]) {
            const double rx = dsub(sx[j], c0), ry = dsub(sy[j], c1), rz = dsub(sz[j], c2);
            xx = dadd(xx, dmul(rx, rx));
            xy = dadd(xy, dmul(rx, ry));
            xz = dadd(xz, dmul(rx, rz));
            yy = dadd(yy, dmul(ry, ry));
            yz = dadd(yz, dmul(ry, rz));
            zz = dadd(zz, dmul(rz, rz));
        }
    out[0] = xx;
    out[1] = xy;
    out[2] = xz;
    out[3] = yy;
    out[4] = yz;
    out[5] = zz;
}

// One thread: the tile partials of a refit pass summed in tile order.  pass 0: the centroid, the sums over the number
// of final inliers (the scan's total); pass 1: the refit plane.
__global__ void segment_refit_finish_kernel(SegArgs a, int pass, int ctas) {
    double s[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll 8   // loads run ahead of the ordered sums
    for (int t = 0; t < a.tiles; ++t)
#pragma unroll
        for (int k = 0; k < 6; ++k)
            if (pass == 1 || k < 3) s[k] = dadd(s[k], a.part_sum[6 * (size_t)t + k]);
    if (pass == 0) {
        const double k = (double)a.counts[ctas];
#pragma unroll
        for (int c = 0; c < 3; ++c) a.state->centroid[c] = __ddiv_rn(s[c], k);
        return;
    }
    plane_from_moments(a.state->centroid, s[0], s[1], s[2], s[3], s[4], s[5], a.plane_out);
}

}  // namespace o3db

using namespace o3db;

extern "C" {

int o3db_random_seed(int seed) {
    std::lock_guard<std::mutex> lock(random_mutex());
    random_engine() = std::mt19937(seed);
    return O3DB_OK;
}

int o3db_random_sample_indices(int64_t n, int sample_size, int num_samples, int64_t* out_host) {
    O3DB_REQUIRE(n >= 1 && sample_size >= 1 && sample_size <= n && num_samples >= 0,
                 "o3db_random_sample_indices: bad arguments (n=%lld, sample_size=%d, num_samples=%d)", (long long)n,
                 sample_size, num_samples);
    O3DB_REQUIRE(num_samples == 0 || out_host, "o3db_random_sample_indices: null output");
    // RandomSampler<size_t> (PointCloudSegmentation.cpp:30-55): one distribution over [0, n-1], repeats redrawn
    std::uniform_int_distribution<size_t> dist(0, (size_t)n - 1);
    std::lock_guard<std::mutex> lock(random_mutex());
    std::mt19937& engine = random_engine();
    for (int64_t s = 0; s < num_samples; ++s) {
        int64_t* row = out_host + s * sample_size;
        for (int k = 0; k < sample_size;) {
            const int64_t idx = (int64_t)dist(engine);
            bool seen = false;
            for (int j = 0; j < k; ++j) seen |= row[j] == idx;
            if (!seen) row[k++] = idx;
        }
    }
    return O3DB_OK;
}

int o3db_segment_plane(const float* positions_dev, int64_t n, double distance_threshold, int ransac_n,
                       int num_iterations, double probability, double* plane_dev, int64_t* inliers_dev,
                       int64_t* num_inliers, o3db_segment_stats* stats, void* stream) {
    O3DB_REQUIRE(plane_dev && num_inliers, "o3db_segment_plane: null plane or inlier count");
    O3DB_REQUIRE(probability > 0 && probability <= 1, "Probability must be > 0 and <= 1.0");
    O3DB_REQUIRE(ransac_n >= 3, "ransac_n should be set to higher than or equal to 3.");
    O3DB_REQUIRE(n >= ransac_n, "There must be at least 'ransac_n' points.");
    O3DB_REQUIRE(n < INT_MAX, "o3db_segment_plane: bad point count (%lld)", (long long)n);
    O3DB_REQUIRE(positions_dev && inliers_dev, "o3db_segment_plane: null positions or inliers");
    O3DB_REQUIRE(num_iterations <= 0 || (int64_t)num_iterations * ransac_n < INT_MAX,
                 "o3db_segment_plane: num_iterations * ransac_n must be below 2^31 (got %d * %d)", num_iterations,
                 ransac_n);
    cudaStream_t st = (cudaStream_t)stream;
    configure_memory_pool();
    const int H = std::max(num_iterations, 0);
    std::vector<int64_t> samples((size_t)H * ransac_n);
    if (int rc = o3db_random_sample_indices(n, ransac_n, H, samples.data())) return rc;

    const int tiles = (int)ceil_div(n, kSegTile);
    const int64_t ctas = ceil_div(n, kSegT);
    const int waves = (int)ceil_div(H, kSegWave);
    DevPtr<SegState> state;
    DevPtr<int64_t> d_samples;
    DevPtr<double> planes, part_err, part_sum;
    DevPtr<int> part_cnt;
    DevPtr<unsigned> counts;
    if (int rc = dev_alloc(state, 1, st)) return rc;
    if (int rc = dev_alloc(d_samples, std::max<size_t>(samples.size(), 1), st)) return rc;
    if (int rc = dev_alloc(planes, 4 * (size_t)std::max(H, 1), st)) return rc;
    if (int rc = dev_alloc(part_cnt, (size_t)tiles * kSegWave, st)) return rc;
    if (int rc = dev_alloc(part_err, (size_t)tiles * kSegWave, st)) return rc;
    if (int rc = dev_alloc(part_sum, (size_t)tiles * 6, st)) return rc;
    if (int rc = dev_alloc(counts, (size_t)(ctas + 1 + ceil_div(ctas, kScanTile)), st)) return rc;
    struct Readback {
        SegState state;
        unsigned total;
    };
    PinnedPtr<Readback> h = pinned_block<Readback>();
    if (!h) {
        set_last_error("o3db_segment_plane: out of pinned host memory");
        return O3DB_ERR_CUDA;
    }
    h->state = SegState{0.0, 0.0, ~0ull, 0ull, -1ll, 0, {0.0, 0.0, 0.0}};
    O3DB_CUDA_CHECK(cudaMemcpyAsync(state.get(), &h->state, sizeof(SegState), cudaMemcpyHostToDevice, st));
    if (H > 0)
        O3DB_CUDA_CHECK(cudaMemcpyAsync(d_samples.get(), samples.data(), samples.size() * sizeof(int64_t),
                                        cudaMemcpyHostToDevice, st));

    SegArgs a{};
    a.pts = positions_dev;
    a.n = n;
    a.thr = distance_threshold;
    a.probability = probability;
    a.ransac_n = ransac_n;
    a.num_iterations = H;
    a.tiles = tiles;
    a.samples = d_samples.get();
    a.planes = planes.get();
    a.part_cnt = part_cnt.get();
    a.part_err = part_err.get();
    a.part_sum = part_sum.get();
    a.state = state.get();
    a.counts = counts.get();
    a.inliers = inliers_dev;
    a.plane_out = plane_dev;
    if (H > 0) {
        segment_hypothesis_kernel<<<(unsigned)ceil_div(H, kSegT), kSegT, 0, st>>>(a);
        O3DB_LAUNCH_CHECK();
    }
    for (int w = 0; w < waves; ++w) {
        segment_score_kernel<<<(unsigned)tiles, kSegWave, 0, st>>>(a, w);
        O3DB_LAUNCH_CHECK();
        segment_select_kernel<<<1, kSegWave, 0, st>>>(a, w);
        O3DB_LAUNCH_CHECK();
    }
    segment_count_kernel<<<(unsigned)ctas, kSegT, 0, st>>>(a);
    O3DB_LAUNCH_CHECK();
    if (int rc = exclusive_scan_u32(counts.get(), ctas, counts.get() + ctas + 1, st)) return rc;
    segment_emit_kernel<<<(unsigned)ctas, kSegT, 0, st>>>(a);
    O3DB_LAUNCH_CHECK();
    for (int pass = 0; pass < 2; ++pass) {
        segment_refit_tile_kernel<<<(unsigned)tiles, kSegWave, 0, st>>>(a, pass);
        O3DB_LAUNCH_CHECK();
        segment_refit_finish_kernel<<<1, 1, 0, st>>>(a, pass, (int)ctas);
        O3DB_LAUNCH_CHECK();
    }
    O3DB_CUDA_CHECK(cudaMemcpyAsync(&h->state, state.get(), sizeof(SegState), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaMemcpyAsync(&h->total, counts.get() + ctas, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));   // the one host synchronisation: the inlier count
    *num_inliers = h->total;
    if (stats) {
        stats->best_index = h->state.best;
        stats->evaluated = (int64_t)h->state.count;
        stats->fitness = h->state.fitness;
        stats->inlier_rmse = h->state.rmse;
    }
    return O3DB_OK;
}

}  // extern "C"
