// dbscan.cu — DBSCAN clustering on the device: PointCloud::ClusterDBSCAN (t/geometry/PointCloud.cpp:1634-1644, which
// runs geometry/PointCloudCluster.cpp:21-97 on the host), label for label.  DESIGN.md §4.19.
//
// The cloud is sorted into the cell grid of the hybrid search (grid.cuh) with cells of at least eps.  Every pass below
// runs one thread per sorted slot and visits the slot's neighbours with the exact predicate of upstream's radius search:
//   core     neighbour count (the point itself included) >= min_points, counting stops once it gets there;
//   union    a lock-free union-find over the core slots: every pair of neighbouring core slots is united;
//   flatten  every core slot records its root; each root collects its component's smallest original index;
//   number   a flag at each component's smallest original index, scanned: the cluster ids in upstream's order;
//   label    core points take their component's id, other points the smallest id among their core neighbours, or -1.
#include <cfloat>
#include <climits>
#include <cmath>

#include "common.cuh"
#include "grid.cuh"
#include "scan.cuh"

namespace o3db {

// What the neighbour passes read: the sorted table with its binning radius, and upstream's squared radius.
struct DbscanView {
    RadiusView box;   // box.rr = eps, rounded up a little
    double eps2;      // eps * eps in f64, as KDTreeFlann::SearchRadius passes it to nanoflann
};

// nanoflann's L2_Adaptor::evalMetric for dimension 3 and RadiusResultSet::addPoint: d2 = ((0 + dx dx) + dy dy) + dz dz
// in f64 on the f32 coordinates, dx = q.x - p.x, no FMA, and a neighbour iff d2 < eps^2.  0 + dx dx is dx dx.
__device__ __forceinline__ bool dbscan_neighbour(const float4 q, const float4 p, double eps2) {
    const double dx = __dsub_rn((double)q.x, (double)p.x);
    const double dy = __dsub_rn((double)q.y, (double)p.y);
    const double dz = __dsub_rn((double)q.z, (double)p.z);
    const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
    return d2 < eps2;
}

// radius_visit (grid.cuh) with upstream's predicate: f(slot) for every neighbour of q at a sorted slot >= from.
template <typename F>
__device__ __forceinline__ void dbscan_visit(const DbscanView& v, const float4 q, unsigned from, F&& f) {
    radius_visit(v.box, q, from, [&](const float4 p) { return dbscan_neighbour(q, p, v.eps2); }, f);
}

// The root of x's tree.  Every parent is an ancestor at a lower slot, so path halving (a plain store of the
// grandparent) keeps every tree intact while other threads hook roots; only roots are ever hooked.
__device__ __forceinline__ unsigned dbscan_find(unsigned* parent, unsigned x) {
    volatile unsigned* p = parent;
    unsigned px = p[x];
    while (px != x) {
        const unsigned gp = p[px];
        if (gp != px) p[x] = gp;
        x = px;
        px = gp;
    }
    return x;
}

// Unites the trees of a and b: the larger root is hooked under the smaller with atomicCAS, retried from the new roots
// until the two share a root, so the union is complete when the call returns.
__device__ __forceinline__ void dbscan_unite(unsigned* parent, unsigned a, unsigned b) {
    for (;;) {
        a = dbscan_find(parent, a);
        b = dbscan_find(parent, b);
        if (a == b) return;
        if (a > b) {
            const unsigned t = a;
            a = b;
            b = t;
        }
        if (atomicCAS(&parent[b], b, a) == b) return;
    }
}

// core[s] = the neighbour count of slot s reaches need (PointCloudCluster.cpp:57); parent[s] = s, cmin[s] = none.
__global__ void __launch_bounds__(kThreads) dbscan_core_kernel(DbscanView v, int64_t n, int need,
                                                               uint8_t* __restrict__ core, unsigned* __restrict__ parent,
                                                               unsigned* __restrict__ cmin) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n) return;
    int count = 0;
    if (need > 0)
        dbscan_visit(v, __ldg(&v.box.pts[s]), 0u, [&](unsigned) { return ++count < need; });
    core[s] = count >= need;
    parent[s] = (unsigned)s;
    cmin[s] = 0xffffffffu;
}

// Every pair of neighbouring core slots (s, j), j > s (the relation is symmetric), is united.
__global__ void __launch_bounds__(kThreads) dbscan_union_kernel(DbscanView v, int64_t n,
                                                                const uint8_t* __restrict__ core, unsigned* parent) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n || !core[s]) return;
    dbscan_visit(v, __ldg(&v.box.pts[s]), (unsigned)s + 1u, [&](unsigned j) {
        if (core[j]) dbscan_unite(parent, (unsigned)s, j);
        return true;
    });
}

// root[s] = the root of core slot s, and the root takes the smallest original index of its component.  The root goes
// to its own array: parent[s] may still be rewritten to any ancestor by another thread's path halving.
__global__ void __launch_bounds__(kThreads) dbscan_flatten_kernel(const float4* __restrict__ pts, int64_t n,
                                                                  const uint8_t* __restrict__ core, unsigned* parent,
                                                                  unsigned* __restrict__ root,
                                                                  unsigned* __restrict__ cmin) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n || !core[s]) return;
    const unsigned r = dbscan_find(parent, (unsigned)s);
    root[s] = r;
    atomicMin(&cmin[r], (unsigned)__float_as_int(__ldg(&pts[s]).w));
}

// flag[smallest original index of each component] = 1 (flag is zero on entry)
__global__ void __launch_bounds__(kThreads) dbscan_root_flag_kernel(int64_t n, const uint8_t* __restrict__ core,
                                                                    const unsigned* __restrict__ root,
                                                                    const unsigned* __restrict__ cmin,
                                                                    unsigned* __restrict__ flag) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n || !core[s] || root[s] != (unsigned)s) return;
    flag[cmin[s]] = 1u;
}

// labels[original index] of slot s: a core point's cluster id, a border point's smallest cluster id among its core
// neighbours (the first BFS to reach it labels it, :76), otherwise -1.  id = the scanned flags.
__global__ void __launch_bounds__(kThreads) dbscan_label_kernel(DbscanView v, int64_t n,
                                                                const uint8_t* __restrict__ core,
                                                                const unsigned* __restrict__ root,
                                                                const unsigned* __restrict__ cmin,
                                                                const unsigned* __restrict__ id,
                                                                int32_t* __restrict__ labels) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n) return;
    const float4 q = __ldg(&v.box.pts[s]);
    unsigned best = 0xffffffffu;
    if (core[s]) {
        best = id[cmin[root[s]]];
    } else {
        dbscan_visit(v, q, 0u, [&](unsigned j) {
            if (core[j]) best = min(best, id[cmin[root[j]]]);
            return best != 0u;
        });
    }
    labels[__float_as_int(q.w)] = best == 0xffffffffu ? -1 : (int32_t)best;
}

// nonfinite = 1 when any coordinate is NaN or infinite (grid_index_finite)
__global__ void __launch_bounds__(kThreads) dbscan_finite_kernel(const float* __restrict__ pts, int64_t n,
                                                                 unsigned* __restrict__ nonfinite) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) flag_nonfinite(pts, i, nonfinite);
}

}  // namespace o3db

using namespace o3db;

extern "C" {

int o3db_cluster_dbscan(const float* positions_dev, int64_t n, double eps, int64_t min_points, int32_t* labels_dev,
                        void* stream) {
    O3DB_REQUIRE(positions_dev != nullptr && labels_dev != nullptr, "o3db_cluster_dbscan: null positions or labels");
    O3DB_REQUIRE(n >= 0 && n < INT_MAX, "o3db_cluster_dbscan: bad point count (%lld)", (long long)n);
    O3DB_REQUIRE(std::isfinite(eps) && eps > 0, "ClusterDBSCAN: eps must be positive and finite (got %g)", eps);
    O3DB_REQUIRE(min_points >= 0, "ClusterDBSCAN: min_points must be non-negative (got %lld)", (long long)min_points);
    if (n == 0) return O3DB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    o3db_nns index;
    if (int rc = grid_index_finite(&index, positions_dev, n, eps, dbscan_finite_kernel,
                                   "ClusterDBSCAN: the point cloud has non-finite coordinates", st))
        return rc;
    // rr >= eps after its rounding to f32; an eps beyond the f32 range bins every point into the box
    const double rr = eps * (1.0 + 1e-5);
    const DbscanView v{{index.g, index.pts4.get(), index.cell_start.get(), rr < (double)FLT_MAX ? (float)rr : INFINITY},
                       eps * eps};
    DevPtr<uint8_t> core;
    DevPtr<unsigned> parent, root, cmin, id, scratch;
    if (int rc = dev_alloc(core, (size_t)n, st)) return rc;
    if (int rc = dev_alloc(parent, (size_t)n, st)) return rc;
    if (int rc = dev_alloc(root, (size_t)n, st)) return rc;
    if (int rc = dev_alloc(cmin, (size_t)n, st)) return rc;
    if (int rc = dev_alloc(id, (size_t)n + 1, st)) return rc;
    if (int rc = dev_alloc(scratch, (size_t)ceil_div(n, kScanTile), st)) return rc;
    O3DB_CUDA_CHECK(cudaMemsetAsync(id.get(), 0, ((size_t)n + 1) * sizeof(unsigned), st));
    // a count never exceeds n, so a min_points above n is n + 1: no point is core
    const int need = (int)std::min<int64_t>(min_points, n + 1);
    const unsigned nb = (unsigned)ceil_div(n, kThreads);
    dbscan_core_kernel<<<nb, kThreads, 0, st>>>(v, n, need, core.get(), parent.get(), cmin.get());
    O3DB_LAUNCH_CHECK();
    dbscan_union_kernel<<<nb, kThreads, 0, st>>>(v, n, core.get(), parent.get());
    O3DB_LAUNCH_CHECK();
    dbscan_flatten_kernel<<<nb, kThreads, 0, st>>>(v.box.pts, n, core.get(), parent.get(), root.get(), cmin.get());
    O3DB_LAUNCH_CHECK();
    dbscan_root_flag_kernel<<<nb, kThreads, 0, st>>>(n, core.get(), root.get(), cmin.get(), id.get());
    O3DB_LAUNCH_CHECK();
    if (int rc = exclusive_scan_u32(id.get(), n, scratch.get(), st)) return rc;
    dbscan_label_kernel<<<nb, kThreads, 0, st>>>(v, n, core.get(), root.get(), cmin.get(), id.get(), labels_dev);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

}  // extern "C"
