// knn.cu — exact k-nearest-neighbour search (k <= 32) over a cell-sorted index, and its two consumers on the
// device: PointCloud::RemoveStatisticalOutliers and PointCloud::ComputeMetrics.  See include/open3d_b200.h for the
// reference functions each entry point replaces and DESIGN.md §4.17 for the design.  The same walk with a list of up to
// 128 keys and an optional radius cap gives FPFH its neighbour lists (knn_lists, DESIGN.md §4.24).
#include <cfloat>
#include <cstddef>
#include <climits>
#include <cmath>
#include <new>
#include <vector>

#include "common.cuh"
#include "grid.cuh"
#include "reduce.cuh"

namespace o3db {

static constexpr int kKnnMax = 32;
static_assert(kKnnWideMax == 4 * 32, "knn_lists' list holds four keys per lane");
static constexpr int kBlockShift = 3;           // a coarse block is 8 x 8 x 8 fine cells
static constexpr int kOccLevels = 8;            // cell sizes c0 * 2^L probed for their occupancy
static constexpr unsigned kOccCells = 1u << 24; // cells of probe level 0 at most (a 2 MB bitmap per level)
static constexpr double kTargetOccupancy = 24;  // points per occupied cell the index aims at
static constexpr float kLbShrink = 1.0f - 1e-5f; // covers the f32 rounding of dist^2 and of its lower bounds
static constexpr unsigned kFull = 0xffffffffu;

// ------------------------------------------------------------------ cell size from the data

struct KnnProbe {
    unsigned bbox[6];               // bbox_kernel's output
    unsigned count[kOccLevels];     // occupied cells at each probe level
    unsigned nonfinite;             // a coordinate is NaN (bbox_kernel's fminf / fmaxf skip NaN)
    double c[kOccLevels];           // the probe levels' cell sizes (0: non-finite box)
    float mn[3], inv[kOccLevels];
    int n[kOccLevels][3];
};

// One thread: the probe levels from the bounding box.  Level 0 is the finest cell whose grid over the box has at most
// kOccCells cells; level L has cells 2^L times as large.
__global__ void knn_probe_setup_kernel(KnnProbe* p) {
    double ext[3], emax = 0;
    for (int a = 0; a < 3; ++a) {
        const float mn = ordered_to_float(p->bbox[a]), mx = ordered_to_float(p->bbox[3 + a]);
        p->mn[a] = mn;
        if (!(mn <= mx) || !isfinite(mn) || !isfinite(mx)) {
            for (int l = 0; l < kOccLevels; ++l) p->c[l] = 0;
            return;
        }
        ext[a] = (double)mx - (double)mn;
        emax = fmax(emax, ext[a]);
    }
    double c = 1.0;
    if (emax > 0) {
        double vol = 1;
        for (int a = 0; a < 3; ++a) vol *= fmax(ext[a], emax * 1e-3);
        c = cbrt(vol / kOccCells);
        for (;;) {
            double cells = 1;
            for (int a = 0; a < 3; ++a) cells *= floor(ext[a] / c) + 1;
            if (cells <= kOccCells) break;
            c *= 1.25;
        }
    }
    for (int l = 0; l < kOccLevels; ++l) {
        const double cl = c * (double)(1 << l);
        p->c[l] = cl;
        p->inv[l] = (float)(1.0 / cl);
        for (int a = 0; a < 3; ++a) p->n[l][a] = (int)(floor(ext[a] / cl) + 1);
    }
}

// Marks every point's cell at every probe level in that level's bitmap and counts the cells marked first.
__global__ void knn_probe_kernel(const float* __restrict__ pts, int64_t m, const KnnProbe* __restrict__ p,
                                 unsigned* __restrict__ bits, unsigned* __restrict__ count,
                                 unsigned* __restrict__ nonfinite) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= m || !(p->c[0] > 0)) return;
    const float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
    if (!isfinite(x) || !isfinite(y) || !isfinite(z)) {
        atomicOr(nonfinite, 1u);
        return;
    }
#pragma unroll
    for (int l = 0; l < kOccLevels; ++l) {
        const int ix = cell1(x, p->mn[0], p->inv[l], p->n[l][0]);
        const int iy = cell1(y, p->mn[1], p->inv[l], p->n[l][1]);
        const int iz = cell1(z, p->mn[2], p->inv[l], p->n[l][2]);
        const unsigned key = (unsigned)((iz * p->n[l][1] + iy) * p->n[l][0] + ix);
        const unsigned bit = 1u << (key & 31);
        if (!(atomicOr(&bits[(size_t)l * (kOccCells / 32) + (key >> 5)], bit) & bit)) atomicAdd(&count[l], 1u);
    }
}

// The cell size: the probe levels L-1, L around the target occupancy give a local dimension
// d = log2(K[L-1] / K[L]) in [1, 3] (K = occupied cells; a surface has d ~ 2, a volume 3), and
// c = c[L-1] (T / occ[L-1])^(1/d) interpolates between them (DESIGN.md §4.17).
static double knn_cell_size(const KnnProbe& p, int64_t m) {
    int l = 0;
    while (l < kOccLevels && (double)m < kTargetOccupancy * p.count[l]) ++l;
    if (l == kOccLevels) return p.c[kOccLevels - 1];
    const double occ_hi = (double)m / p.count[l];
    if (l == 0) return p.c[0] * std::pow(kTargetOccupancy / occ_hi, 1.0 / 3.0);
    const double occ_lo = (double)m / p.count[l - 1];
    const double d = std::min(3.0, std::max(1.0, std::log2((double)p.count[l - 1] / p.count[l])));
    const double c = p.c[l - 1] * std::pow(kTargetOccupancy / occ_lo, 1.0 / d);
    return std::min(p.c[l], std::max(p.c[l - 1], c));
}

// flag[coarse block] = 1 when any of its fine cells holds a point
__global__ void knn_block_flags_kernel(const unsigned* __restrict__ cs, Grid g, int nbx, int nby,
                                       unsigned* __restrict__ flag) {
    const int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (c >= (int64_t)g.nx * g.ny * g.nz || cs[c + 1] == cs[c]) return;
    const int ix = (int)(c % g.nx), iy = (int)((c / g.nx) % g.ny), iz = (int)(c / ((int64_t)g.nx * g.ny));
    flag[((iz >> kBlockShift) * nby + (iy >> kBlockShift)) * nbx + (ix >> kBlockShift)] = 1u;
}

// ------------------------------------------------------------------ search

struct KnnView {
    Grid g;
    const float4* pts;
    const unsigned* cs;
    const unsigned* flag;
    int nbx, nby, nbz;
};

// The query in grid axis order with the slack of each axis: binning round-off (g.tol) plus 2 ulp of the query
// coordinate for the f32 subtraction.
struct KnnQuery {
    float x, y, z;       // real axes, for the canonical distance
    float gx, gy, gz;    // grid axes
    float sx, sy, sz;
};

struct CellBox {
    int x0, x1, y0, y1, z0, z1;
};

// Lower bound on |p - q| along one axis for every point binned into cells [i0, i1].
__device__ __forceinline__ float axis_gap(float q, float o, float c, int i0, int i1, float slack) {
    const float lo = o + (float)i0 * c, hi = o + (float)(i1 + 1) * c;
    return fmaxf(fmaxf(lo - q, q - hi) - slack, 0.f);
}
// Lower bound on |p - q| along one axis for every point binned OUTSIDE cells [i0, i1] of n; +inf when none can be.
__device__ __forceinline__ float axis_clearance(float q, float o, float c, int i0, int i1, int n, float slack) {
    float r = __int_as_float(0x7f800000);
    if (i0 > 0) r = fminf(r, q - (o + (float)i0 * c));
    if (i1 < n - 1) r = fminf(r, (o + (float)(i1 + 1) * c) - q);
    return fmaxf(r - slack, 0.f);
}
// dist^2 lower bound for every point outside box b (+inf when b spans the grid)
__device__ __forceinline__ float box_clearance2(const Grid& g, const KnnQuery& q, const CellBox& b) {
    const float r = fminf(axis_clearance(q.gx, g.ox, g.cx, b.x0, b.x1, g.nx, q.sx),
                          fminf(axis_clearance(q.gy, g.oy, g.c, b.y0, b.y1, g.ny, q.sy),
                                axis_clearance(q.gz, g.oz, g.c, b.z0, b.z1, g.nz, q.sz)));
    return r * r * kLbShrink;
}

// The running list: lane j holds the j-th smallest key (dist^2 bits : original index) seen so far, ~0 = none.
// Lanes >= kp may hold larger keys; only lanes < kp are reported.
__device__ __forceinline__ float kth_dist2(unsigned long long key, int kp) {
    // while fewer than kp points are held this is the NaN 0xffffffff: every "kth < bound" test is false
    return __uint_as_float((unsigned)(__shfl_sync(kFull, key, kp - 1) >> 32));
}

// Offers each lane's candidate key; inserts the ones below the current k-th key, one at a time, by ballot and shuffle.
__device__ __forceinline__ void knn_offer(unsigned long long& key, int kp, unsigned long long cand) {
    const int lane = threadIdx.x & 31;
    unsigned long long kth = __shfl_sync(kFull, key, kp - 1);
    unsigned pend = __ballot_sync(kFull, cand < kth);
    while (pend) {
        const int src = __ffs(pend) - 1;
        pend &= pend - 1;
        const unsigned long long c = __shfl_sync(kFull, cand, src);
        if (c < kth) {
            const int pos = __popc(__ballot_sync(kFull, key < c));
            const unsigned long long up = __shfl_up_sync(kFull, key, 1);
            key = lane > pos ? up : (lane == pos ? c : key);
            kth = __shfl_sync(kFull, key, kp - 1);
        }
    }
}

// The list of knn_search_kernel: one key per lane, k <= 32.
struct KnnList {
    unsigned long long key = ~0ull;
    int kp;
    __device__ __forceinline__ float bound() const { return kth_dist2(key, kp); }
    __device__ __forceinline__ bool accept(float) const { return true; }
    __device__ __forceinline__ void offer(unsigned long long cand) { knn_offer(key, kp, cand); }
};

// The list of knn_lists_kernel: four keys per lane, k <= 128.  Slot s of lane j holds the (32 s + j)-th smallest key;
// slots above `last` = (kp - 1) / 32 stay ~0 and are never read.  A candidate beyond the cap (dist^2 > thr, +inf for
// none) is not offered, and the pruning bound is min(k-th dist^2, thr): while fewer than kp keys are held the k-th is
// the NaN 0xffffffff, and fminf then gives thr.  The slots are four named registers: an array indexed by `last` would
// be placed in local memory.
struct KnnWideList {
    unsigned long long k0 = ~0ull, k1 = ~0ull, k2 = ~0ull, k3 = ~0ull;
    int kp, last;
    float thr;
    __device__ __forceinline__ KnnWideList(int kp_, float thr_) : kp(kp_), last((kp_ - 1) >> 5), thr(thr_) {}
    __device__ __forceinline__ unsigned long long kth_key() const {
        return __shfl_sync(kFull, last == 0 ? k0 : (last == 1 ? k1 : (last == 2 ? k2 : k3)), (kp - 1) & 31);
    }
    __device__ __forceinline__ float bound() const { return fminf(__uint_as_float((unsigned)(kth_key() >> 32)), thr); }
    __device__ __forceinline__ bool accept(float d) const { return d <= thr; }
    // slot s (base 32 s) after inserting c at position pos; carry is lane 31 of slot s - 1 before the insertion
    static __device__ __forceinline__ void shift(unsigned long long& k, int base, unsigned long long carry,
                                                 unsigned long long c, int pos) {
        const int lane = threadIdx.x & 31;
        const unsigned long long up = __shfl_up_sync(kFull, k, 1);
        const int g = base + lane;
        k = g > pos ? (lane == 0 ? carry : up) : (g == pos ? c : k);
    }
    // knn_offer over the slots up to `last`: the position is the number of smaller keys in all of them, and the shift
    // carries lane 31 of each slot into lane 0 of the next.
    __device__ __forceinline__ void offer(unsigned long long cand) {
        unsigned long long kth = kth_key();
        unsigned pend = __ballot_sync(kFull, cand < kth);
        while (pend) {
            const int src = __ffs(pend) - 1;
            pend &= pend - 1;
            const unsigned long long c = __shfl_sync(kFull, cand, src);
            if (c < kth) {
                int pos = __popc(__ballot_sync(kFull, k0 < c));
                if (last >= 1) pos += __popc(__ballot_sync(kFull, k1 < c));
                if (last >= 2) pos += __popc(__ballot_sync(kFull, k2 < c));
                if (last >= 3) pos += __popc(__ballot_sync(kFull, k3 < c));
                if (last >= 3) shift(k3, 96, __shfl_sync(kFull, k2, 31), c, pos);
                if (last >= 2) shift(k2, 64, __shfl_sync(kFull, k1, 31), c, pos);
                if (last >= 1) shift(k1, 32, __shfl_sync(kFull, k0, 31), c, pos);
                shift(k0, 0, 0ull, c, pos);
                kth = kth_key();
            }
        }
    }
};

// The sorted points [s, e), 32 at a time.
template <typename List>
__device__ __forceinline__ void knn_scan(const float4* __restrict__ pts, unsigned s, unsigned e, const KnnQuery& q,
                                         List& list) {
    const unsigned lane = threadIdx.x & 31;
    for (unsigned b = s; b < e; b += 32) {
        unsigned long long cand = ~0ull;
        if (b + lane < e) {
            const float4 t = __ldg(&pts[b + lane]);
            const float d = dist2_canonical(t, q.x, q.y, q.z);
            if (list.accept(d)) cand = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)__float_as_int(t.w);
        }
        list.offer(cand);
    }
}

// Every cell of box b that is not in box `skip`, one (grid-y, grid-z) row per lane: a row's cells are one contiguous
// run of pts4 (two when `skip` cuts it).  A row whose lower bound exceeds the k-th distance is not read.
template <typename List>
__device__ __forceinline__ void knn_visit_box(const KnnView& v, const KnnQuery& q, const CellBox& b, const CellBox& skip,
                                              List& list) {
    const Grid& g = v.g;
    const int lane = threadIdx.x & 31;
    const int wy = b.y1 - b.y0 + 1;
    const int rows = wy * (b.z1 - b.z0 + 1);
    const float ex = axis_gap(q.gx, g.ox, g.cx, b.x0, b.x1, q.sx);
    for (int base = 0; base < rows; base += 32) {
        const float kth = list.bound();
        unsigned s1 = 0, e1 = 0, s2 = 0, e2 = 0;
        float lb = 0.f;
        if (base + lane < rows) {
            const int iy = b.y0 + (base + lane) % wy, iz = b.z0 + (base + lane) / wy;
            const float ey = axis_gap(q.gy, g.oy, g.c, iy, iy, q.sy), ez = axis_gap(q.gz, g.oz, g.c, iz, iz, q.sz);
            lb = fmaf(ez, ez, fmaf(ey, ey, ex * ex)) * kLbShrink;
            if (!(kth < lb)) {
                const unsigned* row = v.cs + (size_t)(iz * g.ny + iy) * g.nx;
                int a1 = b.x0, b1 = b.x1, a2 = 1, b2 = 0;
                if (iy >= skip.y0 && iy <= skip.y1 && iz >= skip.z0 && iz <= skip.z1) {
                    b1 = min(b.x1, skip.x0 - 1);
                    a2 = max(b.x0, skip.x1 + 1);
                    b2 = b.x1;
                }
                if (a1 <= b1) {
                    s1 = __ldg(&row[a1]);
                    e1 = __ldg(&row[b1 + 1]);
                }
                if (a2 <= b2) {
                    s2 = __ldg(&row[a2]);
                    e2 = __ldg(&row[b2 + 1]);
                }
            }
        }
        unsigned todo = __ballot_sync(kFull, e1 > s1 || e2 > s2);
        while (todo) {
            const int src = __ffs(todo) - 1;
            todo &= todo - 1;
            const float rlb = __shfl_sync(kFull, lb, src);
            if (list.bound() < rlb) continue;   // the list tightened since the row was tested
            knn_scan(v.pts, __shfl_sync(kFull, s1, src), __shfl_sync(kFull, e1, src), q, list);
            knn_scan(v.pts, __shfl_sync(kFull, s2, src), __shfl_sync(kFull, e2, src), q, list);
        }
    }
}

// Exact k nearest points of one query, one warp per query.
//   1. the 3 x 3 x 3 cells around the query's cell; done when the k-th distance is below the bound on every point
//      outside them (the common case);
//   2. otherwise rounds over the coarse blocks around the query's block, Chebyshev radius 0, 1, 2, 4, ...: each
//      round visits the non-empty blocks of its shell whose lower bound does not exceed the k-th distance, and the
//      search ends after the first round whose box bounds every point outside it beyond the k-th distance, or
//      which covers the grid.  Empty blocks cost one flag load, 32 per warp step.
template <typename List>
__device__ __forceinline__ void knn_query(const KnnView& v, const KnnQuery& q, List& list) {
    const Grid& g = v.g;
    const int lane = threadIdx.x & 31;
    const int cx = cell1(q.gx, g.ox, g.inv_cx, g.nx), cy = cell1(q.gy, g.oy, g.inv_c, g.ny),
              cz = cell1(q.gz, g.oz, g.inv_c, g.nz);
    const CellBox near{max(cx - 1, 0), min(cx + 1, g.nx - 1), max(cy - 1, 0),
                       min(cy + 1, g.ny - 1), max(cz - 1, 0), min(cz + 1, g.nz - 1)};
    const CellBox none{0, -1, 0, -1, 0, -1};
    knn_visit_box(v, q, near, none, list);
    if (list.bound() < box_clearance2(g, q, near)) return;

    const int bx = cx >> kBlockShift, by = cy >> kBlockShift, bz = cz >> kBlockShift;
    int done = -1;   // blocks within this Chebyshev radius are visited
    for (int r = 0;; r = r ? 2 * r : 1) {
        const int x0 = max(bx - r, 0), x1 = min(bx + r, v.nbx - 1), y0 = max(by - r, 0), y1 = min(by + r, v.nby - 1);
        const int z0 = max(bz - r, 0), z1 = min(bz + r, v.nbz - 1);
        const int wx = x1 - x0 + 1, wxy = wx * (y1 - y0 + 1);
        const int total = wxy * (z1 - z0 + 1);
        for (int base = 0; base < total; base += 32) {
            const int t = base + lane;
            int ix = 0, iy = 0, iz = 0;
            float lb = 0.f;
            bool visit = false;
            if (t < total) {
                ix = x0 + t % wx;
                iy = y0 + (t % wxy) / wx;
                iz = z0 + t / wxy;
                const int cheb = max(abs(ix - bx), max(abs(iy - by), abs(iz - bz)));
                if (cheb > done && __ldg(&v.flag[(iz * v.nby + iy) * v.nbx + ix])) {
                    const float gx = axis_gap(q.gx, g.ox, g.cx, ix << kBlockShift,
                                              min(((ix + 1) << kBlockShift) - 1, g.nx - 1), q.sx);
                    const float gy = axis_gap(q.gy, g.oy, g.c, iy << kBlockShift,
                                              min(((iy + 1) << kBlockShift) - 1, g.ny - 1), q.sy);
                    const float gz = axis_gap(q.gz, g.oz, g.c, iz << kBlockShift,
                                              min(((iz + 1) << kBlockShift) - 1, g.nz - 1), q.sz);
                    lb = fmaf(gz, gz, fmaf(gy, gy, gx * gx)) * kLbShrink;
                    visit = true;
                }
            }
            const float kth = list.bound();   // every lane shuffles: not inside the short-circuit below
            unsigned todo = __ballot_sync(kFull, visit && !(kth < lb));
            while (todo) {
                const int src = __ffs(todo) - 1;
                todo &= todo - 1;
                if (list.bound() < __shfl_sync(kFull, lb, src)) continue;
                const int px = __shfl_sync(kFull, ix, src), py = __shfl_sync(kFull, iy, src),
                          pz = __shfl_sync(kFull, iz, src);
                const CellBox blk{px << kBlockShift, min(((px + 1) << kBlockShift) - 1, g.nx - 1),
                                  py << kBlockShift, min(((py + 1) << kBlockShift) - 1, g.ny - 1),
                                  pz << kBlockShift, min(((pz + 1) << kBlockShift) - 1, g.nz - 1)};
                knn_visit_box(v, q, blk, near, list);
            }
        }
        done = r;
        const CellBox seen{x0 << kBlockShift, min(((x1 + 1) << kBlockShift) - 1, g.nx - 1),
                           y0 << kBlockShift, min(((y1 + 1) << kBlockShift) - 1, g.ny - 1),
                           z0 << kBlockShift, min(((z1 + 1) << kBlockShift) - 1, g.nz - 1)};
        if ((x0 == 0 && y0 == 0 && z0 == 0 && x1 == v.nbx - 1 && y1 == v.nby - 1 && z1 == v.nbz - 1) ||
            list.bound() < box_clearance2(g, q, seen))
            return;
    }
}

// The grid coordinates and slacks of a query whose real coordinates are set.
__device__ __forceinline__ void knn_query_setup(const Grid& g, KnnQuery& q) {
    to_grid(g, q.x, q.y, q.z, q.gx, q.gy, q.gz);
    q.sx = g.tol + fabsf(q.gx) * 2.4e-7f;
    q.sy = g.tol + fabsf(q.gy) * 2.4e-7f;
    q.sz = g.tol + fabsf(q.gz) * 2.4e-7f;
}

// One warp per query: lane j writes the j-th neighbour.  A query with a non-finite coordinate gets -1 / 0.
// No __launch_bounds__: with one, ptxas caps the kernel below the 76 registers it needs and spills; without, it fits
// 80 registers, 3 CTAs of 256 threads per SM (tests/test_knn_resources.py).
template <typename IndexT>
__global__ void knn_search_kernel(KnnView v, const float* __restrict__ queries, int64_t nq,
                                                              int kp, IndexT* __restrict__ idx, float* __restrict__ d2) {
    const int64_t qi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (qi >= nq) return;
    KnnQuery q;
    q.x = queries[3 * qi];
    q.y = queries[3 * qi + 1];
    q.z = queries[3 * qi + 2];
    KnnList list;
    list.kp = kp;
    if (isfinite(q.x) && isfinite(q.y) && isfinite(q.z)) {
        knn_query_setup(v.g, q);
        knn_query(v, q, list);
    }
    const unsigned long long key = list.key;
    if (lane < kp) {
        const bool ok = key != ~0ull;
        if (idx) idx[qi * kp + lane] = ok ? (IndexT)(int)(unsigned)key : (IndexT)-1;
        if (d2) d2[qi * kp + lane] = ok ? __uint_as_float((unsigned)(key >> 32)) : 0.f;
    }
}

// One warp per query, up to four keys per lane: the kp nearest points with dist^2 <= thr (+inf: no cap),
// ascending by (dist^2, index).  Slot g = 32 s + lane of row qi gets the g-th neighbour, -1 / 0 past cnt[qi].  With
// thr = +inf this is knn_search_kernel's list; with thr = (float)r * (float)r and kp <= 32 it is the hybrid search's,
// whose distance is the same dist2_canonical and whose order is the same key.  Queries are finite (the callers
// check; a guard here costs the kernel its fit in 80 registers).
__global__ void __launch_bounds__(kThreads) knn_lists_kernel(KnnView v, const float* __restrict__ queries, int64_t nq,
                                                             int kp, float thr, int32_t* __restrict__ idx,
                                                             float* __restrict__ d2, int32_t* __restrict__ cnt) {
    const int64_t qi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (qi >= nq) return;
    KnnQuery q;
    q.x = queries[3 * qi];
    q.y = queries[3 * qi + 1];
    q.z = queries[3 * qi + 2];
    knn_query_setup(v.g, q);
    KnnWideList list(kp, thr);
    knn_query(v, q, list);
    const unsigned long long keys[4] = {list.k0, list.k1, list.k2, list.k3};
    int c = 0;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        const int g = 32 * s + lane;
        const bool ok = g < kp && keys[s] != ~0ull;
        c += __popc(__ballot_sync(kFull, ok));
        if (g < kp) {
            idx[qi * kp + g] = ok ? (int32_t)(unsigned)keys[s] : -1;
            d2[qi * kp + g] = ok ? __uint_as_float((unsigned)(keys[s] >> 32)) : 0.f;
        }
    }
    if (lane == 0) cnt[qi] = c;
}

// *bad = 1 when a query coordinate is NaN or infinite
__global__ void knn_finite_kernel(const float* __restrict__ q, int64_t n, unsigned* __restrict__ bad) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) flag_nonfinite(q, i, bad);
}

// ------------------------------------------------------------------ deterministic sums

// Fixed launch shape for a given n, so that every sum below is taken in one order on every call.
static unsigned sum_blocks(int64_t n) { return (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, kThreads), 1024)); }

// Sum of one double per thread over the block, in a fixed order.
__device__ __forceinline__ double block_sum(double v) {
    __shared__ double s_part[kThreads / 32];
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0;
    if (threadIdx.x == 0)
        for (int w = 0; w < kThreads / 32; ++w) t += s_part[w];
    __syncthreads();
    return t;
}

// PASS 0: avg[i] = fl32(sum_j sqrtf(d2[i, j])) * inv_k, and the block partials of sum avg[i];
// PASS 1: the block partials of sum (avg[i] - mean)^2 (the difference and its square in f32).
template <int PASS>
__global__ void __launch_bounds__(kThreads) outlier_pass_kernel(const float* __restrict__ d2, int64_t n, int kp,
                                                                float inv_k, float mean, float* __restrict__ avg,
                                                                double* __restrict__ partial) {
    double acc = 0;
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        if (PASS == 0) {
            float s = 0.f;
            for (int j = 0; j < kp; ++j) s += sqrtf(d2[i * kp + j]);
            const float a = s * inv_k;
            avg[i] = a;
            acc += (double)a;
        } else {
            const float c = avg[i] - mean;
            acc += (double)(c * c);
        }
    }
    const double t = block_sum(acc);
    if (threadIdx.x == 0) partial[blockIdx.x] = t;
}

__global__ void outlier_mask_kernel(const float* __restrict__ avg, int64_t n, float thr, uint8_t* __restrict__ mask) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) mask[i] = avg[i] <= thr;
}

// Per block: sum of sqrtf(d2) (f64), its max, and per radius the count of sqrtf(d2) < radius.
__global__ void __launch_bounds__(kThreads) metric_pass_kernel(const float* __restrict__ d2, int64_t n,
                                                               const float* __restrict__ radius, int nr,
                                                               double* __restrict__ psum, float* __restrict__ pmax,
                                                               double* __restrict__ pcnt) {
    double acc = 0;
    float mx = 0.f;
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        const float d = sqrtf(d2[i]);
        acc += (double)d;
        mx = fmaxf(mx, d);
    }
    const double t = block_sum(acc);
    __shared__ float s_max[kThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(kFull, mx, o));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 0; w < kThreads / 32; ++w) mx = fmaxf(mx, s_max[w]);
        psum[blockIdx.x] = t;
        pmax[blockIdx.x] = mx;
    }
    for (int r = 0; r < nr; ++r) {
        const float rad = radius[r];
        double cnt = 0;   // integer-valued: exact below 2^53
        for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
            cnt += sqrtf(d2[i]) < rad ? 1.0 : 0.0;
        const double c = block_sum(cnt);
        if (threadIdx.x == 0) pcnt[(size_t)r * gridDim.x + blockIdx.x] = c;
    }
}

}  // namespace o3db

using namespace o3db;

struct o3db_knn {
    o3db_nns grid;
    int nbx = 0, nby = 0, nbz = 0;
    DevPtr<unsigned> flag;   // [nbx * nby * nbz] coarse block non-empty
};

namespace o3db {

using KnnPtr = std::unique_ptr<o3db_knn, HandleDestroy<o3db_knn_destroy>>;

static KnnView knn_view(const o3db_knn* h) {
    return KnnView{h->grid.g, h->grid.pts4.get(), h->grid.cell_start.get(), h->flag.get(), h->nbx, h->nby, h->nbz};
}

// The k' = min(k, M) nearest neighbours' dist^2 of every point of `pts` among `pts` or, with a separate index, of the
// queries; a temporary index is built and destroyed.
static int knn_dist2(const float* data, int64_t m, const float* queries, int64_t nq, int k, DevPtr<float>& d2,
                     cudaStream_t st) {
    o3db_knn* raw = nullptr;
    int rc = o3db_knn_create(data, m, st, &raw);
    if (rc) return rc;
    const KnnPtr index(raw);
    const int kp = (int)std::min<int64_t>(k, m);
    if ((rc = dev_alloc(d2, (size_t)nq * kp, st))) return rc;
    return o3db_knn_search(index.get(), queries, nq, k, O3DB_INDEX_INT32, nullptr, d2.get(), st);
}

int knn_lists(const o3db_knn* knn, const float* queries, int64_t nq, int k, float thr, int32_t* idx, float* d2,
              int32_t* cnt, cudaStream_t st) {
    O3DB_REQUIRE(knn != nullptr, "knn_lists: null index");
    O3DB_REQUIRE(k >= 1 && k <= kKnnWideMax, "knn_lists: k = %d is not in 1..%d", k, kKnnWideMax);
    if (nq == 0) return O3DB_OK;
    const int kp = (int)std::min<int64_t>(k, knn->grid.m);
    knn_lists_kernel<<<(unsigned)ceil_div(nq, kThreads / 32), kThreads, 0, st>>>(
            knn_view(knn), queries, nq, kp, thr, idx, d2, cnt);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

// Sum of the per-block partials, in block order, after a synchronise.
template <typename T>
static int read_partials(const T* dev, size_t count, std::vector<T>& host, cudaStream_t st) {
    host.resize(count);
    O3DB_CUDA_CHECK(cudaMemcpyAsync(host.data(), dev, count * sizeof(T), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    return O3DB_OK;
}

}  // namespace o3db

extern "C" {

int o3db_knn_create(const float* points_dev, int64_t num_points, void* stream, o3db_knn** out) {
    O3DB_REQUIRE(out != nullptr, "o3db_knn_create: out is null");
    *out = nullptr;
    O3DB_REQUIRE(points_dev != nullptr && num_points > 0, "o3db_knn_create: empty dataset");
    O3DB_REQUIRE(num_points < INT_MAX, "o3db_knn_create: too many points");
    KnnPtr h(new (std::nothrow) o3db_knn());
    O3DB_REQUIRE(h != nullptr, "out of host memory");
    configure_memory_pool();
    cudaStream_t st = (cudaStream_t)stream;
    o3db_nns* s = &h->grid;
    s->stream = st;
    s->m = num_points;
    KnnProbe probe;
    {
        DevPtr<KnnProbe> d_probe;
        DevPtr<unsigned> bits;
        if (int rc = dev_alloc(d_probe, 1, st)) return rc;
        if (int rc = dev_alloc(bits, (size_t)kOccLevels * (kOccCells / 32), st)) return rc;
        O3DB_CUDA_CHECK(cudaMemsetAsync(d_probe.get(), 0, sizeof(KnnProbe), st));
        O3DB_CUDA_CHECK(cudaMemsetAsync(bits.get(), 0, (size_t)kOccLevels * (kOccCells / 8), st));
        char* base = reinterpret_cast<char*>(d_probe.get());
        if (int rc = bbox_launch(points_dev, num_points, reinterpret_cast<unsigned*>(base + offsetof(KnnProbe, bbox)), st))
            return rc;
        knn_probe_setup_kernel<<<1, 1, 0, st>>>(d_probe.get());
        O3DB_LAUNCH_CHECK();
        knn_probe_kernel<<<(unsigned)ceil_div(num_points, kThreads), kThreads, 0, st>>>(points_dev, num_points,
                                                                                        d_probe.get(), bits.get(),
            reinterpret_cast<unsigned*>(base + offsetof(KnnProbe, count)),
            reinterpret_cast<unsigned*>(base + offsetof(KnnProbe, nonfinite)));
        O3DB_LAUNCH_CHECK();
        O3DB_CUDA_CHECK(cudaMemcpyAsync(&probe, d_probe.get(), sizeof(KnnProbe), cudaMemcpyDeviceToHost, st));
        O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    }
    float mn[3], mx[3];
    if (bbox_decode(probe.bbox, mn, mx) || probe.nonfinite) {
        set_last_error("o3db_knn_create: the dataset has non-finite coordinates");
        return O3DB_ERR_INVALID;
    }
    grid_from_bbox(mn, mx, knn_cell_size(probe, num_points), false, num_points, &s->g, &s->ncell);
    if (int rc = grid_sort(s, points_dev, nullptr, num_points, st)) return rc;
    h->nbx = ((s->g.nx - 1) >> kBlockShift) + 1;
    h->nby = ((s->g.ny - 1) >> kBlockShift) + 1;
    h->nbz = ((s->g.nz - 1) >> kBlockShift) + 1;
    const size_t nblk = (size_t)h->nbx * h->nby * h->nbz;
    if (int rc = dev_alloc(h->flag, nblk, st)) return rc;
    O3DB_CUDA_CHECK(cudaMemsetAsync(h->flag.get(), 0, nblk * sizeof(unsigned), st));
    knn_block_flags_kernel<<<(unsigned)ceil_div(s->ncell, kThreads), kThreads, 0, st>>>(s->cell_start.get(), s->g,
                                                                                       h->nbx, h->nby, h->flag.get());
    O3DB_LAUNCH_CHECK();
    *out = h.release();
    return O3DB_OK;
}

void o3db_knn_destroy(o3db_knn* knn) {
    if (!knn) return;
    // searches may still be in flight on the creation stream, and it waits for those on other streams
    cudaStreamSynchronize(knn->grid.stream);
    delete knn;
}

int o3db_knn_index_stats(const o3db_knn* knn, double* cell_size, int64_t* num_cells, int64_t* num_blocks) {
    O3DB_REQUIRE(knn != nullptr, "o3db_knn_index_stats: null index");
    if (cell_size) *cell_size = knn->grid.g.c;
    if (num_cells) *num_cells = knn->grid.ncell;
    if (num_blocks) *num_blocks = (int64_t)knn->nbx * knn->nby * knn->nbz;
    return O3DB_OK;
}

int o3db_knn_search(const o3db_knn* knn, const float* queries_dev, int64_t num_queries, int knn_k, int index_dtype,
                    void* indices_dev, float* distances_dev, void* stream) {
    O3DB_REQUIRE(knn != nullptr, "Index is not set.");
    O3DB_REQUIRE(knn_k >= 1, "knn should be larger than 0.");
    O3DB_REQUIRE(knn_k <= kKnnMax, "knn = %d exceeds the largest k this search supports (%d)", knn_k, kKnnMax);
    O3DB_REQUIRE(index_dtype == O3DB_INDEX_INT32 || index_dtype == O3DB_INDEX_INT64,
                 "o3db_knn_search: index_dtype must be O3DB_INDEX_INT32 or O3DB_INDEX_INT64");
    O3DB_REQUIRE(num_queries >= 0, "o3db_knn_search: negative query count");
    if (num_queries == 0) return O3DB_OK;
    O3DB_REQUIRE(queries_dev != nullptr, "o3db_knn_search: null queries");
    const int kp = (int)std::min<int64_t>(knn_k, knn->grid.m);
    const unsigned nb = (unsigned)ceil_div(num_queries, kThreads / 32);
    cudaStream_t st = (cudaStream_t)stream;
    const HandleUse use(knn->grid.events, knn->grid.stream, st);
    if (use.status()) return use.status();
    if (index_dtype == O3DB_INDEX_INT32)
        knn_search_kernel<int32_t><<<nb, kThreads, 0, st>>>(knn_view(knn), queries_dev, num_queries, kp,
                                                            static_cast<int32_t*>(indices_dev), distances_dev);
    else
        knn_search_kernel<int64_t><<<nb, kThreads, 0, st>>>(knn_view(knn), queries_dev, num_queries, kp,
                                                            static_cast<int64_t*>(indices_dev), distances_dev);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

int o3db_knn_search_lists(const o3db_knn* knn, const float* queries_dev, int64_t num_queries, int knn_k, double radius,
                          int32_t* indices_dev, float* distances_dev, int32_t* counts_dev, void* stream) {
    O3DB_REQUIRE(knn != nullptr, "Index is not set.");
    O3DB_REQUIRE(knn_k >= 1 && knn_k <= kKnnWideMax, "knn = %d is not in 1..%d", knn_k, kKnnWideMax);
    O3DB_REQUIRE(radius >= 0 && std::isfinite(radius), "o3db_knn_search_lists: radius must be finite and >= 0 (got %g)",
                 radius);
    O3DB_REQUIRE(num_queries >= 0, "o3db_knn_search_lists: negative query count");
    if (num_queries == 0) return O3DB_OK;
    O3DB_REQUIRE(queries_dev && indices_dev && distances_dev && counts_dev, "o3db_knn_search_lists: null argument");
    cudaStream_t st = (cudaStream_t)stream;
    const HandleUse use(knn->grid.events, knn->grid.stream, st);
    if (use.status()) return use.status();
    DevPtr<unsigned> bad;
    if (int rc = dev_alloc(bad, 1, st)) return rc;
    O3DB_CUDA_CHECK(cudaMemsetAsync(bad.get(), 0, sizeof(unsigned), st));
    knn_finite_kernel<<<(unsigned)ceil_div(num_queries, kThreads), kThreads, 0, st>>>(queries_dev, num_queries, bad.get());
    O3DB_LAUNCH_CHECK();
    unsigned h_bad = 0;
    O3DB_CUDA_CHECK(cudaMemcpyAsync(&h_bad, bad.get(), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    O3DB_REQUIRE(h_bad == 0, "o3db_knn_search_lists: the queries have non-finite coordinates");
    const float thr = radius > 0 ? (float)radius * (float)radius : INFINITY;
    return knn_lists(knn, queries_dev, num_queries, knn_k, thr, indices_dev, distances_dev, counts_dev, st);
}

int o3db_remove_statistical_outliers(const float* positions_dev, int64_t n, int nb_neighbors, double std_ratio,
                                     uint8_t* mask_dev, float* avg_dev, void* stream) {
    O3DB_REQUIRE(nb_neighbors >= 1 && std_ratio > 0,
                 "Illegal input parameters, the number of neighbors and standard deviation ratio must be positive.");
    O3DB_REQUIRE(nb_neighbors <= kKnnMax, "nb_neighbors = %d exceeds the largest k the search supports (%d)",
                 nb_neighbors, kKnnMax);
    O3DB_REQUIRE(n >= 0 && n < INT_MAX, "o3db_remove_statistical_outliers: bad point count");
    if (n == 0) return O3DB_OK;
    O3DB_REQUIRE(positions_dev != nullptr && mask_dev != nullptr, "o3db_remove_statistical_outliers: null argument");
    cudaStream_t st = (cudaStream_t)stream;
    DevPtr<float> d2, avg_own;
    int rc = knn_dist2(positions_dev, n, positions_dev, n, nb_neighbors, d2, st);
    if (rc) return rc;
    float* avg = avg_dev;
    if (!avg) {
        if ((rc = dev_alloc(avg_own, (size_t)n, st))) return rc;
        avg = avg_own.get();
    }
    const int kp = (int)std::min<int64_t>(nb_neighbors, n);
    const unsigned G = sum_blocks(n);
    DevPtr<double> partial;
    if ((rc = dev_alloc(partial, G, st))) return rc;
    std::vector<double> h;
    // cloud_mean: the f64 sum rounded to f32 times (float)(1 / n), as upstream's Mean (Sum x factor) in f32
    outlier_pass_kernel<0><<<G, kThreads, 0, st>>>(d2.get(), n, kp, (float)(1.0 / kp), 0.f, avg, partial.get());
    O3DB_LAUNCH_CHECK();
    if ((rc = read_partials(partial.get(), G, h, st))) return rc;
    double s = 0;
    for (double v : h) s += v;
    const float mean_f = (float)s * (float)(1.0 / (double)n);
    const double cloud_mean = (double)mean_f;
    outlier_pass_kernel<1><<<G, kThreads, 0, st>>>(d2.get(), n, kp, 0.f, (float)cloud_mean, avg, partial.get());
    O3DB_LAUNCH_CHECK();
    if ((rc = read_partials(partial.get(), G, h, st))) return rc;
    double sq_sum = 0;
    for (double v : h) sq_sum += v;
    const double std_dev = std::sqrt(sq_sum / (double)(n - 1));
    const double thr = cloud_mean + std_ratio * std_dev;
    outlier_mask_kernel<<<(unsigned)ceil_div(n, kThreads), kThreads, 0, st>>>(avg, n, (float)thr, mask_dev);
    O3DB_LAUNCH_CHECK();
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));   // avg_own is freed on return
    return O3DB_OK;
}

int o3db_compute_metrics(const float* points1_dev, int64_t n1, const float* points2_dev, int64_t n2,
                         const int* metrics, int num_metrics, const float* fscore_radius, int num_radius,
                         float* values_host, int64_t num_values, void* stream) {
    O3DB_REQUIRE(n1 > 0 && n2 > 0 && points1_dev && points2_dev, "One or both input point clouds are empty!");
    O3DB_REQUIRE(n1 < INT_MAX && n2 < INT_MAX, "o3db_compute_metrics: too many points");
    O3DB_REQUIRE(num_metrics >= 0 && (metrics || num_metrics == 0), "o3db_compute_metrics: bad metric list");
    O3DB_REQUIRE(num_radius >= 0 && (fscore_radius || num_radius == 0), "o3db_compute_metrics: bad F-score radii");
    int64_t want = 0;
    for (int i = 0; i < num_metrics; ++i) {
        O3DB_REQUIRE(metrics[i] == O3DB_METRIC_CHAMFER || metrics[i] == O3DB_METRIC_HAUSDORFF ||
                             metrics[i] == O3DB_METRIC_FSCORE,
                     "o3db_compute_metrics: unknown metric %d", metrics[i]);
        want += metrics[i] == O3DB_METRIC_FSCORE ? num_radius : 1;
    }
    O3DB_REQUIRE(num_values >= want && (values_host || want == 0),
                 "o3db_compute_metrics: the output holds %lld values, the metrics give %lld", (long long)num_values,
                 (long long)want);
    cudaStream_t st = (cudaStream_t)stream;
    DevPtr<float> d12, d21, rad;
    int rc = knn_dist2(points2_dev, n2, points1_dev, n1, 1, d12, st);
    if (rc) return rc;
    if ((rc = knn_dist2(points1_dev, n1, points2_dev, n2, 1, d21, st))) return rc;
    if ((rc = dev_alloc(rad, (size_t)std::max(num_radius, 1), st))) return rc;
    if (num_radius)
        O3DB_CUDA_CHECK(cudaMemcpyAsync(rad.get(), fscore_radius, num_radius * sizeof(float), cudaMemcpyHostToDevice, st));
    struct Dir {
        double sum;
        float max;
        std::vector<double> count;
    } dir[2];
    const float* d[2] = {d12.get(), d21.get()};
    const int64_t n[2] = {n1, n2};
    for (int k = 0; k < 2; ++k) {
        const unsigned G = sum_blocks(n[k]);
        DevPtr<double> psum, pcnt;
        DevPtr<float> pmax;
        if ((rc = dev_alloc(psum, G, st))) return rc;
        if ((rc = dev_alloc(pmax, G, st))) return rc;
        if ((rc = dev_alloc(pcnt, (size_t)G * std::max(num_radius, 1), st))) return rc;
        metric_pass_kernel<<<G, kThreads, 0, st>>>(d[k], n[k], rad.get(), num_radius, psum.get(), pmax.get(), pcnt.get());
        O3DB_LAUNCH_CHECK();
        std::vector<double> hs, hc;
        std::vector<float> hm;
        if ((rc = read_partials(psum.get(), G, hs, st))) return rc;
        if ((rc = read_partials(pmax.get(), G, hm, st))) return rc;
        if ((rc = read_partials(pcnt.get(), (size_t)G * num_radius, hc, st))) return rc;
        dir[k].sum = 0;
        dir[k].max = 0.f;
        for (unsigned b = 0; b < G; ++b) {
            dir[k].sum += hs[b];
            dir[k].max = std::max(dir[k].max, hm[b]);
        }
        dir[k].count.assign(num_radius, 0.0);
        for (int r = 0; r < num_radius; ++r)
            for (unsigned b = 0; b < G; ++b) dir[k].count[r] += hc[(size_t)r * G + b];
    }
    // Metrics.cpp, in f32 as upstream; means as Sum x (float)(1 / n), the sum taken in f64
    const float mean12 = (float)dir[0].sum * (float)(1.0 / (double)n1);
    const float mean21 = (float)dir[1].sum * (float)(1.0 / (double)n2);
    int64_t o = 0;
    for (int i = 0; i < num_metrics; ++i) {
        if (metrics[i] == O3DB_METRIC_CHAMFER) {
            values_host[o++] = mean21 + mean12;
        } else if (metrics[i] == O3DB_METRIC_HAUSDORFF) {
            values_host[o++] = std::max(dir[0].max, dir[1].max);
        } else {
            for (int r = 0; r < num_radius; ++r) {
                const float precision = (float)(dir[0].count[r] * (100.0 / (double)n1));
                const float recall = (float)(dir[1].count[r] * (100.0 / (double)n2));
                float fscore = 0.0f;
                if (precision + recall > 0) fscore = 2 * precision * recall / (precision + recall);
                values_host[o++] = fscore;
            }
        }
    }
    return O3DB_OK;
}

}  // extern "C"
