// smooth.cu — point-cloud smoothing on the device: t::geometry::PointCloud::SmoothLaplacian, SmoothTaubin, SmoothMLS
// and SmoothBilateral (kernel/PointCloudImpl.h:1341-1753).  Each is a neighbour search followed by per-point arithmetic;
// the arithmetic is upstream's, in f32 with no FMA contraction, in neighbour-list order.  DESIGN.md §4.18.
#include <climits>
#include <cmath>

#include "common.cuh"
#include "eigen3x3.cuh"
#include "reduce.cuh"

namespace o3db {

static constexpr int kSmoothMaxNn = 32;   // the largest neighbour list either search returns

#define MUL(a, b) __fmul_rn(a, b)
#define ADD(a, b) __fadd_rn(a, b)
#define SUB(a, b) __fsub_rn(a, b)
#define DIV(a, b) __fdiv_rn(a, b)

// upstream's exp of an f32 argument, evaluated in f64 and rounded once: CUDA's expf is up to 2 ulp off
__device__ __forceinline__ float exp_rn(float x) { return __double2float_rn(exp((double)x)); }

// ApplyLaplacianPass (PointCloudImpl.h:1357-1406), one point, from the f32 sum of its `count` neighbours other than
// itself: p + alpha * (mean * inv_count - p), inv_count = (float)(1.0 / count); with no neighbour the point is copied.
__device__ __forceinline__ void laplacian_store(const float* p, const float m[3], int count, float alpha, float* out) {
    if (count == 0) {
        out[0] = p[0];
        out[1] = p[1];
        out[2] = p[2];
        return;
    }
    const float inv_count = __double2float_rn(__ddiv_rn(1.0, (double)count));
#pragma unroll
    for (int k = 0; k < 3; ++k) out[k] = ADD(p[k], MUL(alpha, SUB(MUL(m[k], inv_count), p[k])));
}

// One Laplacian pass over given neighbour lists idx [n, kp] (-1 = none): one thread per point.
__global__ void __launch_bounds__(kThreads) smooth_gather_pass_kernel(const float* __restrict__ cur,
                                                                      const int32_t* __restrict__ idx, int64_t n,
                                                                      int kp, float alpha, float* __restrict__ next) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float p[3] = {cur[3 * i], cur[3 * i + 1], cur[3 * i + 2]};
    float m[3] = {0.f, 0.f, 0.f};
    int count = 0;
    for (int s = 0; s < kp; ++s) {
        const int j = idx[i * kp + s];
        if (j < 0 || j == i) continue;
        m[0] = ADD(m[0], cur[3 * (int64_t)j]);
        m[1] = ADD(m[1], cur[3 * (int64_t)j + 1]);
        m[2] = ADD(m[2], cur[3 * (int64_t)j + 2]);
        ++count;
    }
    laplacian_store(p, m, count, alpha, next + 3 * i);
}

// SmoothMLSCPU's per-point body (PointCloudImpl.h:1559-1655): weights exp(-d2 * inv_radius2), weighted centroid and
// covariance in f32, the fast eigen solve, and the projection onto the fitted plane.  Point i's list is
// idx[i * stride, + count), count = cnt[i] (hybrid) or stride (KNN, where d2 is NULL and every distance is 0).  out
// holds a copy of the positions on entry; nrm (NULL when the cloud has none) is updated in place.
__global__ void __launch_bounds__(kThreads) smooth_mls_kernel(const float* __restrict__ pts,
                                                              const int32_t* __restrict__ idx,
                                                              const float* __restrict__ d2,
                                                              const int32_t* __restrict__ cnt, int64_t n, int stride,
                                                              float inv_radius2, float* __restrict__ out,
                                                              float* __restrict__ nrm) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t o = i * stride;
    const int count = cnt ? cnt[i] : stride;
    const float p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
    if (count < 3) {
        if (nrm) {
            float* v = nrm + 3 * i;
            const float norm = __fsqrt_rn(ADD(ADD(MUL(v[0], v[0]), MUL(v[1], v[1])), MUL(v[2], v[2])));
            if (norm > 0) {
                v[0] = DIV(v[0], norm);
                v[1] = DIV(v[1], norm);
                v[2] = DIV(v[2], norm);
            }
        }
        return;
    }
    float c[3] = {0.f, 0.f, 0.f}, wsum = 0.f;
    for (int s = 0; s < count; ++s) {
        const int j = idx[o + s];
        if (j < 0) continue;
        const float w = exp_rn(MUL(-(d2 ? d2[o + s] : 0.f), inv_radius2));
        c[0] = ADD(c[0], MUL(w, pts[3 * (int64_t)j]));
        c[1] = ADD(c[1], MUL(w, pts[3 * (int64_t)j + 1]));
        c[2] = ADD(c[2], MUL(w, pts[3 * (int64_t)j + 2]));
        wsum = ADD(wsum, w);
    }
    if (wsum <= 0) return;
    c[0] = DIV(c[0], wsum);
    c[1] = DIV(c[1], wsum);
    c[2] = DIV(c[2], wsum);
    float C[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int s = 0; s < count; ++s) {
        const int j = idx[o + s];
        if (j < 0) continue;
        const float w = exp_rn(MUL(-(d2 ? d2[o + s] : 0.f), inv_radius2));
        const float x = SUB(pts[3 * (int64_t)j], c[0]), y = SUB(pts[3 * (int64_t)j + 1], c[1]),
                    z = SUB(pts[3 * (int64_t)j + 2], c[2]);
        C[0] = ADD(C[0], MUL(MUL(w, x), x));
        C[1] = ADD(C[1], MUL(MUL(w, x), y));
        C[2] = ADD(C[2], MUL(MUL(w, x), z));
        C[4] = ADD(C[4], MUL(MUL(w, y), y));
        C[5] = ADD(C[5], MUL(MUL(w, y), z));
        C[8] = ADD(C[8], MUL(MUL(w, z), z));
    }
    C[3] = C[1];
    C[6] = C[2];
    C[7] = C[5];
    float v[3];
    normal_from_covariance(C, v);
    const float proj = ADD(ADD(MUL(SUB(p[0], c[0]), v[0]), MUL(SUB(p[1], c[1]), v[1])), MUL(SUB(p[2], c[2]), v[2]));
#pragma unroll
    for (int k = 0; k < 3; ++k) out[3 * i + k] = SUB(p[k], MUL(proj, v[k]));
    if (nrm) {
#pragma unroll
        for (int k = 0; k < 3; ++k) nrm[3 * i + k] = v[k];
    }
}

// SmoothBilateralCPU's per-point body (PointCloudImpl.h:1697-1749): weights
// exp(-d2 * inv_s2 - r * r * inv_r2), r the offset along the point's unit normal; the weighted mean of the neighbours.
// out holds a copy of the positions on entry.
__global__ void __launch_bounds__(kThreads) smooth_bilateral_kernel(const float* __restrict__ pts,
                                                                    const float* __restrict__ nrm,
                                                                    const int32_t* __restrict__ idx,
                                                                    const float* __restrict__ d2,
                                                                    const int32_t* __restrict__ cnt, int64_t n,
                                                                    int max_nn, float inv_s2, float inv_r2,
                                                                    float* __restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int count = cnt[i];
    if (count <= 1) return;
    float nx = nrm[3 * i], ny = nrm[3 * i + 1], nz = nrm[3 * i + 2];
    const float norm = __fsqrt_rn(ADD(ADD(MUL(nx, nx), MUL(ny, ny)), MUL(nz, nz)));
    if (norm <= 0) return;
    nx = DIV(nx, norm);
    ny = DIV(ny, norm);
    nz = DIV(nz, norm);
    const float p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
    const int64_t o = i * max_nn;
    float ws[3] = {0.f, 0.f, 0.f}, wsum = 0.f;
    for (int s = 0; s < count; ++s) {
        const int j = idx[o + s];
        if (j < 0) continue;
        const float q[3] = {pts[3 * (int64_t)j], pts[3 * (int64_t)j + 1], pts[3 * (int64_t)j + 2]};
        const float r = ADD(ADD(MUL(SUB(p[0], q[0]), nx), MUL(SUB(p[1], q[1]), ny)), MUL(SUB(p[2], q[2]), nz));
        const float w = exp_rn(SUB(MUL(-d2[o + s], inv_s2), MUL(MUL(r, r), inv_r2)));
        ws[0] = ADD(ws[0], MUL(w, q[0]));
        ws[1] = ADD(ws[1], MUL(w, q[1]));
        ws[2] = ADD(ws[2], MUL(w, q[2]));
        wsum = ADD(wsum, w);
    }
    if (wsum > 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) out[3 * i + k] = DIV(ws[k], wsum);
    }
}

#undef MUL
#undef ADD
#undef SUB
#undef DIV

using NnsPtr = std::unique_ptr<o3db_nns, HandleDestroy<o3db_nns_destroy>>;
using KnnPtr = std::unique_ptr<o3db_knn, HandleDestroy<o3db_knn_destroy>>;

static int copy_points(float* dst, const float* src, int64_t n, cudaStream_t st) {
    O3DB_CUDA_CHECK(cudaMemcpyAsync(dst, src, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return O3DB_OK;
}

// The hybrid search of the cloud on itself (idx, d2 [n, max_nn], cnt [n]); the index is returned so that the caller's
// kernels run before it is destroyed.
static int hybrid_self(const float* pts, int64_t n, double radius, int max_nn, NnsPtr& index, DevPtr<int32_t>& idx,
                       DevPtr<float>& d2, DevPtr<int32_t>& cnt, cudaStream_t st) {
    o3db_nns* raw = nullptr;
    int rc = o3db_nns_create(pts, n, radius, st, &raw);
    if (rc) return rc;
    index.reset(raw);
    if ((rc = dev_alloc(idx, (size_t)n * max_nn, st))) return rc;
    if ((rc = dev_alloc(d2, (size_t)n * max_nn, st))) return rc;
    if ((rc = dev_alloc(cnt, (size_t)n, st))) return rc;
    return o3db_nns_hybrid_search(index.get(), pts, n, radius, max_nn, idx.get(), d2.get(), cnt.get(), st);
}

}  // namespace o3db

using namespace o3db;

extern "C" {

int o3db_smooth_laplacian(const float* positions_dev, int64_t n, int64_t iterations, const double* factors_host,
                          int num_factors, int max_nn, int fixed_neighborhoods, float* out_dev, void* stream) {
    O3DB_REQUIRE(n >= 0 && n < INT_MAX / 3, "o3db_smooth_laplacian: bad point count");
    O3DB_REQUIRE(iterations >= 0, "iterations must be non-negative (got %lld)", (long long)iterations);
    O3DB_REQUIRE((num_factors == 1 || num_factors == 2) && factors_host != nullptr,
                 "o3db_smooth_laplacian: one or two factors per iteration");
    if (n == 0) return O3DB_OK;
    O3DB_REQUIRE(positions_dev != nullptr && out_dev != nullptr && positions_dev != out_dev,
                 "o3db_smooth_laplacian: null or aliased positions / output");
    cudaStream_t st = (cudaStream_t)stream;
    if (iterations == 0 || max_nn <= 0) return copy_points(out_dev, positions_dev, n, st);
    const int64_t kp = std::min<int64_t>(n, (int64_t)max_nn + 1);
    O3DB_REQUIRE(kp <= kSmoothMaxNn,
                 "max_nn = %d asks for %lld neighbours including the point itself; the search supports at most %d",
                 max_nn, (long long)kp, kSmoothMaxNn);
    const int64_t passes = iterations * num_factors;
    DevPtr<float> tmp;
    if (passes > 1) {
        if (int rc = dev_alloc(tmp, (size_t)n * 3, st)) return rc;
    }
    // pass p writes out_dev when passes - 1 - p is even, so that the last pass lands there
    auto dst = [&](int64_t p) { return ((passes - 1 - p) & 1) ? tmp.get() : out_dev; };
    DevPtr<int32_t> idx;
    if (int rc = dev_alloc(idx, (size_t)n * kp, st)) return rc;
    for (int64_t p = 0; p < passes; ++p) {
        const float* cur = p == 0 ? positions_dev : dst(p - 1);
        if (p == 0 || !fixed_neighborhoods) {   // the k' nearest points of every point of cur, itself included
            o3db_knn* raw = nullptr;
            if (int rc = o3db_knn_create(cur, n, st, &raw)) return rc;
            const KnnPtr index(raw);   // destroyed after a synchronise, once the search has run
            if (int rc = o3db_knn_search(raw, cur, n, (int)kp, O3DB_INDEX_INT32, idx.get(), nullptr, st)) return rc;
        }
        smooth_gather_pass_kernel<<<(unsigned)ceil_div(n, kThreads), kThreads, 0, st>>>(
            cur, idx.get(), n, (int)kp, (float)factors_host[p % num_factors], dst(p));
        O3DB_LAUNCH_CHECK();
    }
    return O3DB_OK;
}

int o3db_smooth_mls(const float* positions_dev, int64_t n, double radius, int max_nn, float* out_dev,
                    float* normals_dev, void* stream) {
    O3DB_REQUIRE(n >= 0 && n < INT_MAX / 3, "o3db_smooth_mls: bad point count");
    if (n == 0) return O3DB_OK;
    O3DB_REQUIRE(positions_dev != nullptr && out_dev != nullptr && positions_dev != out_dev,
                 "o3db_smooth_mls: null or aliased positions / output");
    cudaStream_t st = (cudaStream_t)stream;
    if (radius <= 0 && max_nn <= 0) return copy_points(out_dev, positions_dev, n, st);
    O3DB_REQUIRE(max_nn > 0, "SmoothMLS with max_nn <= 0 uses a fixed-radius search, which open3d_b200 does not build; "
                             "pass max_nn in 1..%d",
                 kSmoothMaxNn);
    const int64_t kp = radius > 0 ? max_nn : std::min<int64_t>(n, max_nn);
    O3DB_REQUIRE(kp <= kSmoothMaxNn, "SmoothMLS: max_nn = %d exceeds the largest neighbour count the search supports (%d)",
                 max_nn, kSmoothMaxNn);
    if (int rc = copy_points(out_dev, positions_dev, n, st)) return rc;
    const unsigned nb = (unsigned)ceil_div(n, kThreads);
    if (radius > 0) {
        NnsPtr index;
        DevPtr<int32_t> idx, cnt;
        DevPtr<float> d2;
        if (int rc = hybrid_self(positions_dev, n, radius, max_nn, index, idx, d2, cnt, st)) return rc;
        smooth_mls_kernel<<<nb, kThreads, 0, st>>>(positions_dev, idx.get(), d2.get(), cnt.get(), n, max_nn,
                                                   (float)(1.0 / (radius * radius)), out_dev, normals_dev);
        O3DB_LAUNCH_CHECK();
        return O3DB_OK;
    }
    o3db_knn* raw = nullptr;
    if (int rc = o3db_knn_create(positions_dev, n, st, &raw)) return rc;
    const KnnPtr index(raw);
    DevPtr<int32_t> idx;
    if (int rc = dev_alloc(idx, (size_t)n * kp, st)) return rc;
    if (int rc = o3db_knn_search(raw, positions_dev, n, (int)kp, O3DB_INDEX_INT32, idx.get(), nullptr, st)) return rc;
    smooth_mls_kernel<<<nb, kThreads, 0, st>>>(positions_dev, idx.get(), nullptr, nullptr, n, (int)kp, 0.0f, out_dev,
                                               normals_dev);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

int o3db_smooth_bilateral(const float* positions_dev, const float* normals_dev, int64_t n, double radius, int max_nn,
                          double sigma_s, double sigma_r, float* out_dev, void* stream) {
    O3DB_REQUIRE(n >= 0 && n < INT_MAX / 3, "o3db_smooth_bilateral: bad point count");
    if (n == 0) return O3DB_OK;
    O3DB_REQUIRE(sigma_s > 0 && sigma_r > 0, "Sigma values must be positive.");
    O3DB_REQUIRE(normals_dev != nullptr,
                 "SmoothBilateral needs normals: upstream estimates them with the KNN-only EstimateNormals(), which "
                 "open3d_b200 does not build; call estimate_normals(max_nn, radius) first");
    O3DB_REQUIRE(positions_dev != nullptr && out_dev != nullptr && positions_dev != out_dev,
                 "o3db_smooth_bilateral: null or aliased positions / output");
    O3DB_REQUIRE(radius > 0, "SmoothBilateral: the hybrid search needs a positive radius");
    O3DB_REQUIRE(max_nn >= 1 && max_nn <= kSmoothMaxNn, "SmoothBilateral: max_nn must be in 1..%d", kSmoothMaxNn);
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = copy_points(out_dev, positions_dev, n, st)) return rc;
    NnsPtr index;
    DevPtr<int32_t> idx, cnt;
    DevPtr<float> d2;
    if (int rc = hybrid_self(positions_dev, n, radius, max_nn, index, idx, d2, cnt, st)) return rc;
    smooth_bilateral_kernel<<<(unsigned)ceil_div(n, kThreads), kThreads, 0, st>>>(
        positions_dev, normals_dev, idx.get(), d2.get(), cnt.get(), n, max_nn,
        (float)(1.0 / (2.0 * sigma_s * sigma_s)), (float)(1.0 / (2.0 * sigma_r * sigma_r)), out_dev);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

}  // extern "C"
