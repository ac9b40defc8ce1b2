// boundary.cu — t::geometry::PointCloud::ComputeBoundaryPoints (t/geometry/PointCloud.cpp:803-853,
// kernel/PointCloudImpl.h:354-506) on the device.  DESIGN.md §4.22.
//
// The hybrid search of the cloud on itself (radius, max_nn <= 32), then one warp per point, one lane per neighbour
// slot after the first (upstream drops a list's first entry as the point itself, which leaves m = count - 1 <= 31):
//   frame     GetCoordinateSystemOnPlane (:354-379), f32 in upstream's order with no FMA;
//   angles    atan2(dot(v, d), dot(u, d)) with d = p_j - p_i: the dot products f32 in dot_3x1's order, atan2 evaluated
//             in f64 and rounded to f32 (a correctly rounded atan2f; the reference calls libm's, which is not);
//             empty slots are +inf;
//   sort      a 32-wide bitonic sort over __shfl_xor.  The mask depends only on the sorted values, and the order of
//             +0 and -0 changes no gap, so any correct sort gives the heap sort's answer when no angle is NaN;
//   test      IsBoundaryPoints (:424-440): the largest consecutive gap by std::max from 0 (a NaN gap never wins, so a
//             NaN frame gives 0), the wrap gap 2*M_PI - a[m-1] + a[0] in f64 rounded to f32, then max_gap > the
//             threshold in radians, compared in f64.  m == 0 leaves the mask false.
// A check kernel flags non-finite positions and infinite normal components first; the flag is read at the index
// build's synchronise, before the search runs.  The launches of a call do not depend on the data; neither kernel uses
// stack or local memory.
#include <climits>
#include <cmath>
#include <memory>

#include "common.cuh"

namespace o3db {

static constexpr int kBndThreads = 256;
static constexpr int kBndWarps = kBndThreads / 32;

#define MUL(a, b) __fmul_rn(a, b)
#define ADD(a, b) __fadd_rn(a, b)
#define SUB(a, b) __fsub_rn(a, b)

// 1 when any position coordinate is not finite or any normal component is infinite (a NaN normal is allowed: it gives
// a NaN frame, as upstream)
__global__ void __launch_bounds__(kBndThreads) boundary_check_kernel(const float* __restrict__ pts,
                                                                     const float* __restrict__ nrm, int64_t n,
                                                                     unsigned* __restrict__ bad) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* p = pts + 3 * i;
    const float* q = nrm + 3 * i;
    if (!isfinite(p[0]) || !isfinite(p[1]) || !isfinite(p[2]) || isinf(q[0]) || isinf(q[1]) || isinf(q[2]))
        atomicOr(bad, 1u);
}

__global__ void __launch_bounds__(kBndThreads) boundary_kernel(const float* __restrict__ pts,
                                                               const float* __restrict__ nrm,
                                                               const int32_t* __restrict__ idx,
                                                               const int32_t* __restrict__ cnt, int64_t n, int max_nn,
                                                               double threshold, uint8_t* __restrict__ mask,
                                                               float* __restrict__ max_gap) {
    const int64_t i = blockIdx.x * (int64_t)kBndWarps + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= n) return;   // whole warps leave together
    const int m = cnt[i] - 1;
    float a = INFINITY;
    if (lane < m) {
        const int k = idx[i * max_nn + lane + 1];
        // GetCoordinateSystemOnPlane: abs of the f32 difference, compared with 1e-6 in f64
        const float nx = nrm[3 * i], ny = nrm[3 * i + 1], nz = nrm[3 * i + 2];
        float v0, v1, v2;
        if (!((double)fabsf(SUB(nx, nz)) < 1e-6) || !((double)fabsf(SUB(ny, nz)) < 1e-6)) {
            const float inv = __fdiv_rn(1.0f, __fsqrt_rn(ADD(MUL(nx, nx), MUL(ny, ny))));
            v0 = MUL(-ny, inv);
            v1 = MUL(nx, inv);
            v2 = 0.0f;
        } else {
            const float inv = __fdiv_rn(1.0f, __fsqrt_rn(ADD(MUL(ny, ny), MUL(nz, nz))));
            v0 = 0.0f;
            v1 = MUL(-nz, inv);
            v2 = MUL(ny, inv);
        }
        // u = cross_3x1(n, v)
        const float u0 = SUB(MUL(ny, v2), MUL(nz, v1));
        const float u1 = SUB(MUL(nz, v0), MUL(nx, v2));
        const float u2 = SUB(MUL(nx, v1), MUL(ny, v0));
        const float* q = pts + 3 * i;
        const float* r = pts + 3 * (int64_t)k;
        const float d0 = SUB(r[0], q[0]), d1 = SUB(r[1], q[1]), d2 = SUB(r[2], q[2]);
        const float y = ADD(ADD(MUL(v0, d0), MUL(v1, d1)), MUL(v2, d2));
        const float x = ADD(ADD(MUL(u0, d0), MUL(u1, d1)), MUL(u2, d2));
        a = (float)atan2((double)y, (double)x);
    }
    // bitonic sort, ascending along the lanes
#pragma unroll
    for (int size = 2; size <= 32; size <<= 1) {
#pragma unroll
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            const float b = __shfl_xor_sync(0xffffffffu, a, stride);
            const bool up = (lane & size) == 0;
            const bool lower = (lane & stride) == 0;
            a = (lower == up) ? fminf(a, b) : fmaxf(a, b);
        }
    }
    // consecutive gaps a[l+1] - a[l], l < m - 1; std::max's rule (replace only when greater) from 0
    const float next = __shfl_down_sync(0xffffffffu, a, 1);
    const float g = lane < m - 1 ? SUB(next, a) : 0.0f;
    float best = g > 0.0f ? g : 0.0f;   // no NaN and no -0 below this line
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, off));
    const float first = __shfl_sync(0xffffffffu, a, 0);
    const float last = __shfl_sync(0xffffffffu, a, m > 0 ? m - 1 : 0);
    if (lane == 0) {
        bool is_boundary = false;
        if (m > 0) {
            const float wrap = (float)__dadd_rn(__dsub_rn(2.0 * M_PI, (double)last), (double)first);
            if (wrap > best) best = wrap;
            is_boundary = (double)best > threshold;
        } else {
            best = 0.0f;
        }
        mask[i] = is_boundary ? 1 : 0;
        if (max_gap) max_gap[i] = best;
    }
}

#undef MUL
#undef ADD
#undef SUB

}  // namespace o3db

extern "C" int o3db_compute_boundary_points(const float* positions_dev, const float* normals_dev, int64_t n,
                                            double radius, int max_nn, double angle_threshold, uint8_t* mask_dev,
                                            float* max_gap_dev, void* stream) {
    using namespace o3db;
    O3DB_REQUIRE(n >= 0 && n < INT_MAX / 3, "o3db_compute_boundary_points: bad point count");
    O3DB_REQUIRE(radius > 0 && std::isfinite(radius),
                 "ComputeBoundaryPoints: radius must be positive and finite (got %g)", radius);
    O3DB_REQUIRE(max_nn >= 1 && max_nn <= 32,
                 "ComputeBoundaryPoints: max_nn must be in 1..32, the hybrid search's limit (got %d)", max_nn);
    if (n == 0) return O3DB_OK;
    O3DB_REQUIRE(positions_dev && normals_dev && mask_dev, "o3db_compute_boundary_points: null positions / normals / mask");
    cudaStream_t st = (cudaStream_t)stream;
    DevPtr<unsigned> bad;
    int rc = dev_alloc(bad, 1, st);
    if (rc) return rc;
    O3DB_CUDA_CHECK(cudaMemsetAsync(bad.get(), 0, sizeof(unsigned), st));
    boundary_check_kernel<<<(unsigned)ceil_div(n, kBndThreads), kBndThreads, 0, st>>>(positions_dev, normals_dev, n,
                                                                                       bad.get());
    O3DB_LAUNCH_CHECK();
    unsigned* h_bad = static_cast<unsigned*>(pinned_acquire(sizeof(unsigned)));
    O3DB_REQUIRE(h_bad != nullptr, "out of pinned host memory");
    const std::unique_ptr<void, void (*)(void*)> h_bad_owner(h_bad, pinned_release);
    O3DB_CUDA_CHECK(cudaMemcpyAsync(h_bad, bad.get(), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    // the index build synchronises the stream (for its bounding box), which also delivers the flag
    o3db_nns* raw = nullptr;
    rc = o3db_nns_create(positions_dev, n, radius, stream, &raw);
    const std::unique_ptr<o3db_nns, HandleDestroy<o3db_nns_destroy>> index(raw);
    if (rc) O3DB_CUDA_CHECK(cudaStreamSynchronize(st));   // an early failure may not have synchronised
    O3DB_REQUIRE(*h_bad == 0,
                 "ComputeBoundaryPoints: the point cloud has non-finite positions or infinite normal components");
    if (rc) return rc;
    DevPtr<int32_t> idx, cnt;
    rc = dev_alloc(idx, (size_t)n * max_nn, st);
    if (rc) return rc;
    rc = dev_alloc(cnt, (size_t)n, st);
    if (rc) return rc;
    rc = o3db_nns_hybrid_search(index.get(), positions_dev, n, radius, max_nn, idx.get(), nullptr, cnt.get(), stream);
    if (rc) return rc;
    const double threshold = angle_threshold * M_PI / 180.0;   // IsBoundaryPoints's f64 expression
    boundary_kernel<<<(unsigned)ceil_div(n, kBndWarps), kBndThreads, 0, st>>>(
            positions_dev, normals_dev, idx.get(), cnt.get(), n, max_nn, threshold, mask_dev, max_gap_dev);
    O3DB_LAUNCH_CHECK();
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));   // the index is destroyed on return; its buffers must outlive the kernel
    return O3DB_OK;
}
