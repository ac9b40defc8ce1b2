// remove.cu — the clean-up filters of t::geometry::PointCloud on the device, each writing a keep-mask at the original
// index: RemoveRadiusOutliers, RemoveDuplicatedPoints and RemoveNonFinitePoints (t/geometry/PointCloud.cpp:650-676,
// 716-760).  DESIGN.md §4.23.
//
//   radius      the cloud sorted into the cell grid of DBSCAN (grid_index_finite), cells of at least the radius; one
//               thread per sorted slot counts the points within the radius, itself included, with the predicate of
//               upstream's CUDA radius search, and stops once the count reaches nb_points;
//   duplicates  the voxel down-sampling's claim on hash.cuh, keyed on the bits of the three coordinates: each point
//               finds its group (the index of the point whose claim won), then an atomicMin per group keeps the
//               group's lowest index;
//   non-finite  one elementwise pass.
// The launches of a call do not depend on the data; no kernel uses stack or local memory.
#include <cfloat>
#include <climits>
#include <cmath>

#include "common.cuh"
#include "grid.cuh"
#include "hash.cuh"
#include "reduce.cuh"   // kThreads

namespace o3db {

// upstream's NeighborTest<L2, float> (core/nns/FixedRadiusSearchImpl.cuh:41-59) as nvcc compiles it for sm_90a with
// its default flags: d = p - q, dist = d.dot(d) = ((0 + d0 d0) + d1 d1) + d2 d2 contracted to three FFMAs, the first
// with a zero addend, and a neighbour iff dist <= thr, thr = r * r in f32.
__device__ __forceinline__ bool radius_neighbour(const float4 p, const float4 q, float thr) {
    const float d0 = __fsub_rn(p.x, q.x);
    const float d1 = __fsub_rn(p.y, q.y);
    const float d2 = __fsub_rn(p.z, q.z);
    const float dist = __fmaf_rn(d2, d2, __fmaf_rn(d1, d1, __fmaf_rn(d0, d0, 0.f)));
    return dist <= thr;
}

// mask[original index of slot s] = at least `need` points lie within the radius of it, itself included
__global__ void __launch_bounds__(kThreads) remove_radius_kernel(RadiusView v, float thr, int64_t n, int need,
                                                                 uint8_t* __restrict__ mask) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n) return;
    const float4 q = __ldg(&v.pts[s]);
    int count = 0;
    radius_visit(
            v, q, 0u, [&](const float4 p) { return radius_neighbour(p, q, thr); },
            [&](unsigned) { return ++count < need; });
    mask[__float_as_int(q.w)] = count >= need;
}

// nonfinite = 1 when any coordinate is NaN or infinite (grid_index_finite)
__global__ void __launch_bounds__(kThreads) remove_finite_kernel(const float* __restrict__ pts, int64_t n,
                                                                 unsigned* __restrict__ nonfinite) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) flag_nonfinite(pts, i, nonfinite);
}

// pass 1: every point claims the bucket of its key, the bits of its coordinates.  The table's committed keys are the
// positions themselves, so the winner commits its own index at once and every bit pattern is a valid key.
// group[i] = the winner's index, or -1 when the bucket was still provisional when point i looked (pass 2 resolves it).
__global__ void __launch_bounds__(kThreads) remove_dup_claim_kernel(const int* __restrict__ keys, int n, Table tab,
                                                                    int* __restrict__ group) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned bucket = 0;
    const int r = probe<true>(tab, keys, i, keys[3 * i], keys[3 * i + 1], keys[3 * i + 2], &bucket);
    int g = -1;
    if (r == kResInserted) {
        atomicExch(&tab.table[bucket], i);   // provisional marker -> committed index
        g = i;
    } else if (r >= 0) {
        g = r;
    }
    group[i] = g;
}

// pass 2: first[group] = the group's lowest index (first is 0xffffffff on entry)
__global__ void __launch_bounds__(kThreads) remove_dup_first_kernel(const int* __restrict__ keys, int n, Table tab,
                                                                    int* __restrict__ group,
                                                                    unsigned* __restrict__ first) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int g = group[i];
    if (g < 0) {
        unsigned bucket;
        g = probe<false>(tab, nullptr, 0, keys[3 * i], keys[3 * i + 1], keys[3 * i + 2], &bucket);
        group[i] = g;
    }
    if (g >= 0) atomicMin(&first[g], (unsigned)i);   // g < 0 cannot happen: every key was committed in pass 1
}

// pass 3: a point is kept when it is its group's lowest index
__global__ void __launch_bounds__(kThreads) remove_dup_mask_kernel(int n, const int* __restrict__ group,
                                                                   const unsigned* __restrict__ first,
                                                                   uint8_t* __restrict__ mask) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int g = group[i];
    mask[i] = g >= 0 && first[g] == (unsigned)i;
}

// RemoveNonFinitePoints (PointCloud.cpp:716-738): both flags keep the finite points, remove_nan alone the points
// without a NaN coordinate, remove_inf alone those without an infinite one, neither every point.
__global__ void __launch_bounds__(kThreads) remove_non_finite_kernel(const float* __restrict__ pts, int64_t n,
                                                                     int remove_nan, int remove_inf,
                                                                     uint8_t* __restrict__ mask) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
    const bool nan = isnan(x) || isnan(y) || isnan(z);
    const bool inf = isinf(x) || isinf(y) || isinf(z);
    mask[i] = !(remove_nan && nan) && !(remove_inf && inf);
}

}  // namespace o3db

using namespace o3db;

extern "C" {

int o3db_remove_radius_outliers(const float* positions_dev, int64_t n, int64_t nb_points, double search_radius,
                                uint8_t* mask_dev, void* stream) {
    O3DB_REQUIRE(positions_dev != nullptr && mask_dev != nullptr, "o3db_remove_radius_outliers: null positions or mask");
    O3DB_REQUIRE(n >= 0 && n < INT_MAX, "o3db_remove_radius_outliers: bad point count (%lld)", (long long)n);
    // PointCloud.cpp:652-656
    O3DB_REQUIRE(nb_points >= 1 && !(search_radius <= 0),
                 "Illegal input parameters, number of points and radius must be positive");
    O3DB_REQUIRE(std::isfinite(search_radius), "RemoveRadiusOutliers: search_radius must be finite (got %g)",
                 search_radius);
    if (n == 0) return O3DB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    o3db_nns index;
    if (int rc = grid_index_finite(&index, positions_dev, n, search_radius, remove_finite_kernel,
                                   "RemoveRadiusOutliers: the point cloud has non-finite coordinates; remove them "
                                   "first with remove_non_finite_points",
                                   st))
        return rc;
    // FixedRadiusSearchOps.cu passes T(radius); FixedRadiusSearchImpl.cuh:299 squares it in T.  rr >= the radius after
    // its rounding to f32; a radius beyond the f32 range bins every point into the box.
    const float r = (float)search_radius;
    const float thr = r * r;
    const double rr = search_radius * (1.0 + 1e-5);
    const RadiusView v{index.g, index.pts4.get(), index.cell_start.get(), rr < (double)FLT_MAX ? (float)rr : INFINITY};
    // a count never exceeds n, so an nb_points above n is n + 1: no point is kept
    const int need = (int)std::min<int64_t>(nb_points, n + 1);
    remove_radius_kernel<<<(unsigned)ceil_div(n, kThreads), kThreads, 0, st>>>(v, thr, n, need, mask_dev);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

int o3db_remove_duplicated_points(const float* positions_dev, int64_t n, uint8_t* mask_dev, void* stream) {
    O3DB_REQUIRE(positions_dev != nullptr && mask_dev != nullptr,
                 "o3db_remove_duplicated_points: null positions or mask");
    O3DB_REQUIRE(n >= 0 && n < INT_MAX, "o3db_remove_duplicated_points: bad point count (%lld)", (long long)n);
    if (n == 0) return O3DB_OK;
    configure_memory_pool();
    cudaStream_t st = (cudaStream_t)stream;
    // the voxel down-sampling's sizing, at least 2n buckets, capped at 2^31 (> n, so the table never fills)
    unsigned nb = 16;
    while ((int64_t)nb < 2 * n && nb < 0x80000000u) nb <<= 1;
    DevPtr<int> table, group;
    DevPtr<unsigned> first;
    if (int rc = dev_alloc(table, nb, st)) return rc;
    if (int rc = dev_alloc(group, (size_t)n, st)) return rc;
    if (int rc = dev_alloc(first, (size_t)n, st)) return rc;
    O3DB_CUDA_CHECK(cudaMemsetAsync(table.get(), 0xff, (size_t)nb * sizeof(int), st));   // kEmpty
    O3DB_CUDA_CHECK(cudaMemsetAsync(first.get(), 0xff, (size_t)n * sizeof(unsigned), st));
    const int* keys = reinterpret_cast<const int*>(positions_dev);
    const Table tab{table.get(), nb - 1, keys};
    const unsigned grid = (unsigned)ceil_div(n, kThreads);
    remove_dup_claim_kernel<<<grid, kThreads, 0, st>>>(keys, (int)n, tab, group.get());
    O3DB_LAUNCH_CHECK();
    remove_dup_first_kernel<<<grid, kThreads, 0, st>>>(keys, (int)n, tab, group.get(), first.get());
    O3DB_LAUNCH_CHECK();
    remove_dup_mask_kernel<<<grid, kThreads, 0, st>>>((int)n, group.get(), first.get(), mask_dev);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

int o3db_remove_non_finite_points(const float* positions_dev, int64_t n, int remove_nan, int remove_inf,
                                  uint8_t* mask_dev, void* stream) {
    O3DB_REQUIRE(positions_dev != nullptr && mask_dev != nullptr,
                 "o3db_remove_non_finite_points: null positions or mask");
    O3DB_REQUIRE(n >= 0 && n < INT_MAX, "o3db_remove_non_finite_points: bad point count (%lld)", (long long)n);
    if (n == 0) return O3DB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    remove_non_finite_kernel<<<(unsigned)ceil_div(n, kThreads), kThreads, 0, st>>>(positions_dev, n, remove_nan != 0,
                                                                                    remove_inf != 0, mask_dev);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

}  // extern "C"
