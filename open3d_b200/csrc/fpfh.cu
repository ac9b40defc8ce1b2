// fpfh.cu — t::pipelines::registration::ComputeFPFHFeature and CorrespondencesFromFeatures
// (t/pipelines/registration/Feature.cpp:23-333, kernel/FeatureImpl.h:23-293) on the device.  DESIGN.md §4.24.
//
// FPFH:
//   lists     knn.cu's wide search (knn_lists): the min(max_nn, n) nearest points, capped at dist^2 <= (float)r^2 in
//             hybrid mode; upstream's hybrid list is the prefix of the k-nearest list within the cap;
//   SPFH      one warp per point, one lane per list entry after the first (dropped as the point itself).  The pair
//             feature is f32 in upstream's order with _rn intrinsics (no FMA); acos and atan2 are evaluated in f64, as
//             upstream's object code calls them: the swap test compares the f64 acos values, atan2 is rounded to f32;
//             the bins are upstream's f64 expressions.
//             Every increment of a bin adds the same hist_incr, so a bin is `count` sequential f32 adds of it: the
//             lanes count into shared memory, then one lane per bin adds;
//   FPFH      one thread per output row: fpfh[j] += spfh[nbr][j] / d2 in list order, the three sum[j / 11] serially
//             over (neighbour, bin), entries with d2 == 0 skipped; then 100.0 / sum in f64 rounded to f32, the scale
//             and the point's own SPFH, as upstream.
// With indices, the SPFH pass runs on the selected points and their neighbours only, and each output row equals the
// row of the call without indices.
//
// Correspondences: an exact brute-force 1-NN over feature rows, one thread per query, the target rows tiled through
// shared memory; the distance is the f32 sum over d = 0..D-1 of fmaf(diff, diff, acc), ties to the lowest target index.
// The mutual check is a gather and compare, one scan, one count read.
//
// Every call makes the same launches whatever the data.  No kernel uses stack or local memory.
#include <climits>
#include <cmath>
#include <memory>

#include "common.cuh"
#include "grid.cuh"
#include "scan.cuh"

namespace o3db {

static constexpr int kFpfhThreads = 256;
static constexpr int kFpfhWarps = kFpfhThreads / 32;
static constexpr int kBins = 33;
static constexpr int kFeatTile = 32;    // target rows per shared-memory tile of the feature 1-NN
static constexpr int kFeatChunk = 11;   // feature dimensions per register chunk (33 = 3 x 11)
static constexpr unsigned kBadPosition = 1u, kBadNormal = 2u, kBadIndex = 4u;

#define MUL(a, b) __fmul_rn(a, b)
#define ADD(a, b) __fadd_rn(a, b)
#define SUB(a, b) __fsub_rn(a, b)

// bit kBadPosition: a position coordinate is NaN or infinite; kBadNormal: a normal component is
__global__ void __launch_bounds__(kFpfhThreads) fpfh_check_kernel(const float* __restrict__ pts,
                                                                  const float* __restrict__ nrm, int64_t n,
                                                                  unsigned* __restrict__ bad) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* p = pts + 3 * i;
    const float* q = nrm + 3 * i;
    unsigned b = 0;
    if (!isfinite(p[0]) || !isfinite(p[1]) || !isfinite(p[2])) b |= kBadPosition;
    if (!isfinite(q[0]) || !isfinite(q[1]) || !isfinite(q[2])) b |= kBadNormal;
    if (b) atomicOr(bad, b);
}

// flag[indices[i]] = 1; an index outside [0, n) sets kBadIndex
__global__ void __launch_bounds__(kFpfhThreads) fpfh_select_kernel(const int64_t* __restrict__ indices, int64_t k,
                                                                   int64_t n, unsigned* __restrict__ flag,
                                                                   unsigned* __restrict__ bad) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= k) return;
    const int64_t p = indices[i];
    if (p < 0 || p >= n)
        atomicOr(bad, kBadIndex);
    else
        flag[p] = 1u;
}

// After the exclusive scan of a 0/1 flag per point: rows[scan[p]] = p for every flagged p, in ascending point order.
__global__ void __launch_bounds__(kFpfhThreads) fpfh_compact_kernel(const unsigned* __restrict__ scan, int64_t n,
                                                                    int32_t* __restrict__ rows) {
    const int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (p < n && scan[p + 1] != scan[p]) rows[scan[p]] = (int32_t)p;
}

// out[r] = pts[rows[r]]: the query positions of the listed points
__global__ void __launch_bounds__(kFpfhThreads) fpfh_gather_kernel(const float* __restrict__ pts,
                                                                   const int32_t* __restrict__ rows, int64_t m,
                                                                   float* __restrict__ out) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= m) return;
    const int64_t p = rows[r];
    out[3 * r] = pts[3 * p];
    out[3 * r + 1] = pts[3 * p + 1];
    out[3 * r + 2] = pts[3 * p + 2];
}

// flag[every entry of the m lists] = 1 (the selected points themselves are already flagged)
__global__ void __launch_bounds__(kFpfhThreads) fpfh_mark_kernel(const int32_t* __restrict__ idx,
                                                                 const int32_t* __restrict__ cnt, int64_t m, int kp,
                                                                 unsigned* __restrict__ flag) {
    const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (e >= m * kp) return;
    if ((int)(e % kp) < cnt[e / kp]) flag[idx[e]] = 1u;
}

__device__ __forceinline__ float dot3(const float* a, const float* b) {
    return ADD(ADD(MUL(a[0], b[0]), MUL(a[1], b[1])), MUL(a[2], b[2]));
}
__device__ __forceinline__ void cross3(const float* a, const float* b, float* c) {
    c[0] = SUB(MUL(a[1], b[2]), MUL(a[2], b[1]));
    c[1] = SUB(MUL(a[2], b[0]), MUL(a[0], b[2]));
    c[2] = SUB(MUL(a[0], b[1]), MUL(a[1], b[0]));
}

// ComputePairFeature<float> (FeatureImpl.h:23-85), f[0..3]
__device__ __forceinline__ void pair_feature(const float* p1, const float* n1, const float* p2, const float* n2,
                                             float* f) {
    float d[3] = {SUB(p2[0], p1[0]), SUB(p2[1], p1[1]), SUB(p2[2], p1[2])};
    f[3] = __fsqrt_rn(ADD(ADD(MUL(d[0], d[0]), MUL(d[1], d[1])), MUL(d[2], d[2])));
    f[0] = f[1] = f[2] = 0.0f;
    if (f[3] == 0.0f) {
        f[3] = 0.0f;
        return;
    }
    const float a1 = __fdiv_rn(dot3(n1, d), f[3]);
    const float a2 = __fdiv_rn(dot3(n2, d), f[3]);
    float m1[3], m2[3];
    if (acos((double)fabsf(a1)) > acos((double)fabsf(a2))) {   // f64 acos compared in f64, as upstream's object code
        for (int k = 0; k < 3; ++k) {
            m1[k] = n2[k];
            m2[k] = n1[k];
            d[k] = -d[k];
        }
        f[2] = -a2;
    } else {
        for (int k = 0; k < 3; ++k) {
            m1[k] = n1[k];
            m2[k] = n2[k];
        }
        f[2] = a1;
    }
    float v[3];
    cross3(d, m1, v);
    const float vn = __fsqrt_rn(ADD(ADD(MUL(v[0], v[0]), MUL(v[1], v[1])), MUL(v[2], v[2])));
    if (vn == 0.0f) {
        f[0] = f[1] = f[2] = f[3] = 0.0f;
        return;
    }
    v[0] = __fdiv_rn(v[0], vn);
    v[1] = __fdiv_rn(v[1], vn);
    v[2] = __fdiv_rn(v[2], vn);
    float w[3];
    cross3(m1, v, w);
    f[1] = dot3(v, m2);
    f[0] = (float)atan2((double)dot3(w, m2), (double)dot3(m1, m2));
}

// UpdateSPFHFeature's bin of one feature: floor in f64, clamped to 0..10
__device__ __forceinline__ int spfh_bin(double x) {
    const int h = (int)floor(x);
    return h >= 11 ? 10 : max(0, h);
}

// One warp per SPFH row r (point rows ? rows[r] : r): bins counted in shared memory, then `count` f32 adds of
// hist_incr = (float)(100.0 / (float)(cnt - 1)) per bin.  A row with cnt <= 1 is zero.
__global__ void __launch_bounds__(kFpfhThreads) fpfh_spfh_kernel(const float* __restrict__ pts,
                                                                 const float* __restrict__ nrm,
                                                                 const int32_t* __restrict__ rows, int64_t m,
                                                                 const int32_t* __restrict__ idx,
                                                                 const int32_t* __restrict__ cnt, int kp,
                                                                 float* __restrict__ spfh) {
    __shared__ unsigned s_count[kFpfhWarps][kBins];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t r = blockIdx.x * (int64_t)kFpfhWarps + w;
    if (r >= m) return;   // whole warps leave together
    for (int j = lane; j < kBins; j += 32) s_count[w][j] = 0u;
    __syncwarp();
    const int c = cnt[r];
    const int64_t p = rows ? rows[r] : r;
    for (int e = 1 + lane; e < c; e += 32) {
        const int64_t q = idx[r * kp + e];
        float f[4];
        pair_feature(pts + 3 * p, nrm + 3 * p, pts + 3 * q, nrm + 3 * q, f);
        const int h1 = spfh_bin(__ddiv_rn(__dmul_rn(11.0, __dadd_rn((double)f[0], M_PI)), 2.0 * M_PI));
        const int h2 = spfh_bin(__dmul_rn(__dmul_rn(11.0, __dadd_rn((double)f[1], 1.0)), 0.5));
        const int h3 = spfh_bin(__dmul_rn(__dmul_rn(11.0, __dadd_rn((double)f[2], 1.0)), 0.5));
        atomicAdd(&s_count[w][h1], 1u);
        atomicAdd(&s_count[w][h2 + 11], 1u);
        atomicAdd(&s_count[w][h3 + 22], 1u);
    }
    __syncwarp();
    const float incr = c > 1 ? (float)__ddiv_rn(100.0, (double)(float)(c - 1)) : 0.0f;
    for (int j = lane; j < kBins; j += 32) {
        float v = 0.0f;
        for (unsigned t = s_count[w][j]; t > 0; --t) v = ADD(v, incr);
        spfh[r * kBins + j] = v;
    }
}

// One thread per output row i: the point sel ? sel[i] : i, its list and SPFH at row map ? map[point] : point.
__global__ void __launch_bounds__(kFpfhThreads) fpfh_kernel(const int32_t* __restrict__ sel, int64_t ns,
                                                            const unsigned* __restrict__ map,
                                                            const int32_t* __restrict__ idx,
                                                            const float* __restrict__ d2,
                                                            const int32_t* __restrict__ cnt, int kp,
                                                            const float* __restrict__ spfh, float* __restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= ns) return;
    const int64_t p = sel ? sel[i] : i;
    const int64_t r = map ? (int64_t)map[p] : p;
    float f[kBins];
#pragma unroll
    for (int j = 0; j < kBins; ++j) f[j] = 0.0f;
    const int c = cnt[r];
    if (c > 1) {
        float sum[3] = {0.0f, 0.0f, 0.0f};
        for (int e = 1; e < c; ++e) {
            const float dist = d2[r * kp + e];
            if (dist == 0.0f) continue;
            const int64_t q = idx[r * kp + e];
            const float* s = spfh + (map ? (int64_t)map[q] : q) * kBins;
#pragma unroll
            for (int j = 0; j < kBins; ++j) {
                const float val = __fdiv_rn(__ldg(&s[j]), dist);
                sum[j / 11] = ADD(sum[j / 11], val);
                f[j] = ADD(f[j], val);
            }
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) sum[k] = sum[k] != 0.0f ? (float)__ddiv_rn(100.0, (double)sum[k]) : 0.0f;
        const float* own = spfh + r * kBins;
#pragma unroll
        for (int j = 0; j < kBins; ++j) f[j] = ADD(MUL(f[j], sum[j / 11]), own[j]);
    }
#pragma unroll
    for (int j = 0; j < kBins; ++j) out[i * kBins + j] = f[j];
}

// The nearest target row of each query row: dist = f32 sum over d of fmaf(q - t, q - t, acc) in index order, strict
// < against the best so far from (+inf, 0), targets ascending, so ties go to the lowest index.  Dimensions past D are
// read as 0 on both sides, which leaves every sum unchanged.
__global__ void __launch_bounds__(kFpfhThreads) feature_nn_kernel(const float* __restrict__ query, int64_t nq,
                                                                  const float* __restrict__ target, int64_t nt, int dim,
                                                                  int64_t* __restrict__ nn) {
    __shared__ float s_t[kFeatTile][kFeatChunk];
    const int64_t qi = blockIdx.x * (int64_t)kFpfhThreads + threadIdx.x;
    float best = INFINITY;
    int64_t bi = 0;
    for (int64_t t0 = 0; t0 < nt; t0 += kFeatTile) {
        float acc[kFeatTile];
#pragma unroll
        for (int t = 0; t < kFeatTile; ++t) acc[t] = 0.0f;
        for (int d0 = 0; d0 < dim; d0 += kFeatChunk) {
            float qv[kFeatChunk];
#pragma unroll
            for (int d = 0; d < kFeatChunk; ++d) qv[d] = qi < nq && d0 + d < dim ? query[qi * dim + d0 + d] : 0.0f;
            __syncthreads();
            for (int e = threadIdx.x; e < kFeatTile * kFeatChunk; e += kFpfhThreads) {
                const int t = e / kFeatChunk, d = e % kFeatChunk;
                s_t[t][d] = t0 + t < nt && d0 + d < dim ? target[(t0 + t) * dim + d0 + d] : 0.0f;
            }
            __syncthreads();
#pragma unroll
            for (int t = 0; t < kFeatTile; ++t)
#pragma unroll
                for (int d = 0; d < kFeatChunk; ++d) {
                    const float diff = SUB(qv[d], s_t[t][d]);
                    acc[t] = __fmaf_rn(diff, diff, acc[t]);
                }
        }
#pragma unroll
        for (int t = 0; t < kFeatTile; ++t)
            if (t0 + t < nt && acc[t] < best) {
                best = acc[t];
                bi = t0 + t;
            }
    }
    if (qi < nq) nn[qi] = bi;
}

// keep[i] = 1 when the source row i and its nearest target row are each other's nearest
__global__ void __launch_bounds__(kFpfhThreads) mutual_flag_kernel(const int64_t* __restrict__ ij,
                                                                   const int64_t* __restrict__ ji, int64_t n,
                                                                   unsigned* __restrict__ keep) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) keep[i] = ji[ij[i]] == i ? 1u : 0u;
}

// corres[k] = (i, ij[i]) for every i when scan is null, else for every kept i, at k = scan[i]
__global__ void __launch_bounds__(kFpfhThreads) corres_write_kernel(const int64_t* __restrict__ ij, int64_t n,
                                                                    const unsigned* __restrict__ scan,
                                                                    int64_t* __restrict__ corres) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (scan && scan[i + 1] == scan[i]) return;
    const int64_t k = scan ? (int64_t)scan[i] : i;
    corres[2 * k] = i;
    corres[2 * k + 1] = ij[i];
}

#undef MUL
#undef ADD
#undef SUB

static unsigned grid_for(int64_t n) { return (unsigned)ceil_div(n, kFpfhThreads); }

// Reads a device u32 to the host (one synchronise).
static int read_u32(const unsigned* dev, unsigned* host, cudaStream_t st) {
    O3DB_CUDA_CHECK(cudaMemcpyAsync(host, dev, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    return O3DB_OK;
}

// Flag per point -> (in place) its exclusive scan, rows [total] of the flagged points ascending, total on the host.
static int compact_flags(DevPtr<unsigned>& flag, int64_t n, DevPtr<int32_t>& rows, unsigned* total, cudaStream_t st) {
    DevPtr<unsigned> scratch;
    if (int rc = dev_alloc(scratch, (size_t)ceil_div(n, kScanTile), st)) return rc;
    if (int rc = exclusive_scan_u32(flag.get(), n, scratch.get(), st)) return rc;
    if (int rc = read_u32(flag.get() + n, total, st)) return rc;
    if (int rc = dev_alloc(rows, std::max<size_t>(*total, 1), st)) return rc;
    fpfh_compact_kernel<<<grid_for(n), kFpfhThreads, 0, st>>>(flag.get(), n, rows.get());
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

// The lists of the m points rows[0..m) (rows null: every point, queries = positions).
static int search_lists(const o3db_knn* index, const float* pts, const int32_t* rows, int64_t m, int max_nn, float thr,
                        int kp, DevPtr<int32_t>& idx, DevPtr<float>& d2, DevPtr<int32_t>& cnt, cudaStream_t st) {
    if (int rc = dev_alloc(idx, (size_t)m * kp, st)) return rc;
    if (int rc = dev_alloc(d2, (size_t)m * kp, st)) return rc;
    if (int rc = dev_alloc(cnt, (size_t)m, st)) return rc;
    DevPtr<float> q;
    if (rows) {
        if (int rc = dev_alloc(q, (size_t)m * 3, st)) return rc;
        fpfh_gather_kernel<<<grid_for(m), kFpfhThreads, 0, st>>>(pts, rows, m, q.get());
        O3DB_LAUNCH_CHECK();
    }
    return knn_lists(index, rows ? q.get() : pts, m, max_nn, thr, idx.get(), d2.get(), cnt.get(), st);
}

}  // namespace o3db

extern "C" {

int o3db_compute_fpfh_feature(const float* positions_dev, const float* normals_dev, int64_t n, int max_nn,
                              double radius, const int64_t* indices_dev, int64_t num_indices, float* fpfh_dev,
                              int64_t* num_rows, void* stream) {
    using namespace o3db;
    O3DB_REQUIRE(n >= 0 && n < INT_MAX / 3, "o3db_compute_fpfh_feature: bad point count");
    O3DB_REQUIRE(max_nn > 3, "max_nn must be greater than 3.");
    O3DB_REQUIRE(max_nn <= kKnnWideMax, "ComputeFPFHFeature: max_nn = %d exceeds the largest list this search supports (%d)",
                 max_nn, kKnnWideMax);
    O3DB_REQUIRE(radius >= 0, "radius must be greater than 0.");
    O3DB_REQUIRE(std::isfinite(radius), "ComputeFPFHFeature: radius must be finite (got %g)", radius);
    O3DB_REQUIRE(num_rows != nullptr, "o3db_compute_fpfh_feature: num_rows is null");
    O3DB_REQUIRE(num_indices >= -1 && (indices_dev || num_indices <= 0),
                 "o3db_compute_fpfh_feature: bad indices");
    *num_rows = 0;
    const bool select = num_indices >= 0;
    if (n == 0 || num_indices == 0) return O3DB_OK;
    O3DB_REQUIRE(positions_dev && normals_dev && fpfh_dev, "o3db_compute_fpfh_feature: null positions / normals / out");
    cudaStream_t st = (cudaStream_t)stream;
    const float thr = radius > 0 ? (float)radius * (float)radius : INFINITY;
    const int kp = (int)std::min<int64_t>(max_nn, n);

    DevPtr<unsigned> bad, sel_flag;
    int rc = dev_alloc(bad, 1, st);
    if (rc) return rc;
    O3DB_CUDA_CHECK(cudaMemsetAsync(bad.get(), 0, sizeof(unsigned), st));
    fpfh_check_kernel<<<grid_for(n), kFpfhThreads, 0, st>>>(positions_dev, normals_dev, n, bad.get());
    O3DB_LAUNCH_CHECK();
    if (select) {
        if ((rc = dev_alloc(sel_flag, (size_t)n + 1, st))) return rc;
        O3DB_CUDA_CHECK(cudaMemsetAsync(sel_flag.get(), 0, ((size_t)n + 1) * sizeof(unsigned), st));
        fpfh_select_kernel<<<grid_for(num_indices), kFpfhThreads, 0, st>>>(indices_dev, num_indices, n, sel_flag.get(),
                                                                           bad.get());
        O3DB_LAUNCH_CHECK();
    }
    unsigned h_bad = 0;
    if ((rc = read_u32(bad.get(), &h_bad, st))) return rc;
    O3DB_REQUIRE(!(h_bad & kBadPosition),
                 "ComputeFPFHFeature: the point cloud has NaN or infinite positions; remove them with "
                 "remove_non_finite_points() first");
    O3DB_REQUIRE(!(h_bad & kBadNormal), "ComputeFPFHFeature: the point cloud has NaN or infinite normal components");
    O3DB_REQUIRE(!(h_bad & kBadIndex), "ComputeFPFHFeature: an index is outside [0, %lld)", (long long)n);

    o3db_knn* raw = nullptr;
    rc = o3db_knn_create(positions_dev, n, stream, &raw);
    const std::unique_ptr<o3db_knn, HandleDestroy<o3db_knn_destroy>> index(raw);
    if (rc) return rc;

    DevPtr<int32_t> idx, cnt;
    DevPtr<float> d2, spfh;
    if (!select) {
        if ((rc = search_lists(index.get(), positions_dev, nullptr, n, max_nn, thr, kp, idx, d2, cnt, st))) return rc;
        if ((rc = dev_alloc(spfh, (size_t)n * kBins, st))) return rc;
        fpfh_spfh_kernel<<<(unsigned)ceil_div(n, kFpfhWarps), kFpfhThreads, 0, st>>>(
                positions_dev, normals_dev, nullptr, n, idx.get(), cnt.get(), kp, spfh.get());
        O3DB_LAUNCH_CHECK();
        fpfh_kernel<<<grid_for(n), kFpfhThreads, 0, st>>>(nullptr, n, nullptr, idx.get(), d2.get(), cnt.get(), kp,
                                                          spfh.get(), fpfh_dev);
        O3DB_LAUNCH_CHECK();
        *num_rows = n;
    } else {
        // the selected points, ascending and distinct; their lists flag the points whose SPFH their rows read
        DevPtr<unsigned> req_flag;
        if ((rc = dev_alloc(req_flag, (size_t)n + 1, st))) return rc;
        O3DB_CUDA_CHECK(cudaMemcpyAsync(req_flag.get(), sel_flag.get(), ((size_t)n + 1) * sizeof(unsigned),
                                        cudaMemcpyDeviceToDevice, st));
        DevPtr<int32_t> sel, req;
        unsigned ns = 0, nr = 0;
        if ((rc = compact_flags(sel_flag, n, sel, &ns, st))) return rc;
        {
            DevPtr<int32_t> sidx, scnt;
            DevPtr<float> sd2;
            if ((rc = search_lists(index.get(), positions_dev, sel.get(), ns, max_nn, thr, kp, sidx, sd2, scnt, st)))
                return rc;
            fpfh_mark_kernel<<<grid_for((int64_t)ns * kp), kFpfhThreads, 0, st>>>(sidx.get(), scnt.get(), ns, kp,
                                                                                   req_flag.get());
            O3DB_LAUNCH_CHECK();
        }
        // req_flag becomes the point -> SPFH row map of the required points
        if ((rc = compact_flags(req_flag, n, req, &nr, st))) return rc;
        if ((rc = search_lists(index.get(), positions_dev, req.get(), nr, max_nn, thr, kp, idx, d2, cnt, st)))
            return rc;
        if ((rc = dev_alloc(spfh, (size_t)nr * kBins, st))) return rc;
        fpfh_spfh_kernel<<<(unsigned)ceil_div(nr, kFpfhWarps), kFpfhThreads, 0, st>>>(
                positions_dev, normals_dev, req.get(), nr, idx.get(), cnt.get(), kp, spfh.get());
        O3DB_LAUNCH_CHECK();
        fpfh_kernel<<<grid_for(ns), kFpfhThreads, 0, st>>>(sel.get(), ns, req_flag.get(), idx.get(), d2.get(),
                                                           cnt.get(), kp, spfh.get(), fpfh_dev);
        O3DB_LAUNCH_CHECK();
        *num_rows = ns;
    }
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));   // the index and the lists are freed on return
    return O3DB_OK;
}

int o3db_correspondences_from_features(const float* source_dev, int64_t n, const float* target_dev, int64_t m,
                                       int dim, int mutual_filter, float mutual_consistent_ratio, int64_t* corres_dev,
                                       int64_t* num_corres, int64_t* num_mutual, void* stream) {
    using namespace o3db;
    O3DB_REQUIRE(num_corres != nullptr, "o3db_correspondences_from_features: num_corres is null");
    O3DB_REQUIRE(n >= 0 && m >= 0 && n < INT_MAX && m < INT_MAX, "o3db_correspondences_from_features: bad row counts");
    O3DB_REQUIRE(dim >= 1, "o3db_correspondences_from_features: feature dimension must be at least 1 (got %d)", dim);
    *num_corres = 0;
    if (num_mutual) *num_mutual = 0;
    if (n == 0) return O3DB_OK;
    O3DB_REQUIRE(m > 0, "CorrespondencesFromFeatures: the target features are empty");
    O3DB_REQUIRE(source_dev && target_dev && corres_dev, "o3db_correspondences_from_features: null argument");
    cudaStream_t st = (cudaStream_t)stream;
    DevPtr<int64_t> ij, ji;
    int rc = dev_alloc(ij, (size_t)n, st);
    if (rc) return rc;
    feature_nn_kernel<<<grid_for(n), kFpfhThreads, 0, st>>>(source_dev, n, target_dev, m, dim, ij.get());
    O3DB_LAUNCH_CHECK();
    if (!mutual_filter) {
        corres_write_kernel<<<grid_for(n), kFpfhThreads, 0, st>>>(ij.get(), n, nullptr, corres_dev);
        O3DB_LAUNCH_CHECK();
        O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
        *num_corres = n;
        return O3DB_OK;
    }
    if ((rc = dev_alloc(ji, (size_t)m, st))) return rc;
    feature_nn_kernel<<<grid_for(m), kFpfhThreads, 0, st>>>(target_dev, m, source_dev, n, dim, ji.get());
    O3DB_LAUNCH_CHECK();
    DevPtr<unsigned> keep, scratch;
    if ((rc = dev_alloc(keep, (size_t)n + 1, st))) return rc;
    if ((rc = dev_alloc(scratch, (size_t)ceil_div(n, kScanTile), st))) return rc;
    mutual_flag_kernel<<<grid_for(n), kFpfhThreads, 0, st>>>(ij.get(), ji.get(), n, keep.get());
    O3DB_LAUNCH_CHECK();
    if ((rc = exclusive_scan_u32(keep.get(), n, scratch.get(), st))) return rc;
    unsigned k = 0;
    if ((rc = read_u32(keep.get() + n, &k, st))) return rc;
    if (num_mutual) *num_mutual = k;
    // upstream: result_mutual.GetLength() > mutual_consistent_ratio * arange_source.GetLength(), in f32
    const bool enough = (float)k > mutual_consistent_ratio * (float)n;
    corres_write_kernel<<<grid_for(n), kFpfhThreads, 0, st>>>(ij.get(), n, enough ? keep.get() : nullptr, corres_dev);
    O3DB_LAUNCH_CHECK();
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    *num_corres = enough ? (int64_t)k : n;
    return O3DB_OK;
}

}  // extern "C"
