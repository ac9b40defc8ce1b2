// icp.cu — correspondence search, pose reduction and the fused device-resident
// ICP loop (point-to-plane, coloured, point-to-point) for sm_90a.  See include/open3d_b200.h for the
// reference interfaces each entry point replaces and DESIGN.md for the design.
//
// No CPU fallback: every entry point needs a CUDA device.
#include <cfloat>
#include <cstddef>
#include <algorithm>
#include <climits>
#include <cmath>
#include <new>
#include <vector>

#include "comm.h"
#include "common.cuh"
#include "grid.cuh"
#include "reduce.cuh"
#include "scan.cuh"

namespace o3db {

static constexpr int64_t kMaxCells = int64_t(1) << 26;  // 256 MB of u32 CSR offsets at most
static constexpr int kMaxCellsPerAxis = 4096;
static constexpr double kThinFactor = 8;   // grid-x (thin axis) cells are this much coarser
static constexpr double kDefaultCellScale = 0.5;   // see icp_create_impl

// --------------------------------------------------------------------- bbox

__global__ void bbox_kernel(const float* __restrict__ pts, int64_t n, unsigned* __restrict__ bbox /*6*/) {
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
         i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float v = pts[3 * i + a];
            mn[a] = fminf(mn[a], v);
            mx[a] = fmaxf(mx[a], v);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
            mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            atomicMin(&bbox[a], float_to_ordered(mn[a]));
            atomicMax(&bbox[3 + a], float_to_ordered(mx[a]));
        }
    }
}

// ------------------------------------------------------------ counting sort

struct Affine {  // row-major 3x4 + projective row, f32 (TransformImpl.h:20-45)
    float m[16];
};

__device__ __forceinline__ void apply_transform(const float* __restrict__ T, float& x, float& y, float& z) {
    const float px = x, py = y, pz = z;
    const float ox = T[0] * px + T[1] * py + T[2] * pz + T[3];
    const float oy = T[4] * px + T[5] * py + T[6] * pz + T[7];
    const float oz = T[8] * px + T[9] * py + T[10] * pz + T[11];
    const float ow = T[12] * px + T[13] * py + T[14] * pz + T[15];
    if (ow == 1.0f) {   // rigid transforms: x / 1 == x exactly, skip three IEEE divisions
        x = ox;
        y = oy;
        z = oz;
    } else {
        x = ox / ow;
        y = oy / ow;
        z = oz / ow;
    }
}

// Sort key of the working source: tile-major (16 x 16 x 4 cells per tile, cells row-major
// inside), so that 256 consecutive sorted queries occupy a compact 3-D box whose candidate
// rows can be staged in shared memory.  Only locality depends on it, never correctness.
static constexpr int kTileX = 16, kTileY = 16, kTileZ = 4;
__host__ __device__ inline int64_t tiled_key_space(int nx, int ny, int nz) {
    return (int64_t)((nx + kTileX - 1) / kTileX) * ((ny + kTileY - 1) / kTileY) * ((nz + kTileZ - 1) / kTileZ) *
           (kTileX * kTileY * kTileZ);
}
__device__ __forceinline__ unsigned cell_key_tiled(const Grid& g, float rx, float ry, float rz) {
    float x, y, z;
    to_grid(g, rx, ry, rz, x, y, z);
    const int ix = cell1(x, g.ox, g.inv_cx, g.nx), iy = cell1(y, g.oy, g.inv_c, g.ny), iz = cell1(z, g.oz, g.inv_c, g.nz);
    const int ntx = (g.nx + kTileX - 1) / kTileX, nty = (g.ny + kTileY - 1) / kTileY;
    const int tile = ((iz / kTileZ) * nty + iy / kTileY) * ntx + ix / kTileX;
    const int local = ((iz % kTileZ) * kTileY + iy % kTileY) * kTileX + ix % kTileX;
    return (unsigned)tile * (unsigned)(kTileX * kTileY * kTileZ) + (unsigned)local;
}

// key[i] = cell of (optionally transformed) point i, rank[i] = arrival order in the cell.
// TRANSFORM = true is the source path (tile-major key); false the target (row-major key).
template <bool TRANSFORM>
__global__ void count_kernel(const float* __restrict__ pts, int64_t n, Grid g, Affine T,
                             unsigned* __restrict__ count, unsigned* __restrict__ key,
                             unsigned* __restrict__ rank) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
    if (TRANSFORM) apply_transform(T.m, x, y, z);
    const unsigned k = TRANSFORM ? cell_key_tiled(g, x, y, z) : cell_key(g, x, y, z);
    key[i] = k;
    rank[i] = atomicAdd(&count[k], 1u);
}

// Stable order inside a cell.  count_kernel's atomic rank is the ARRIVAL order of the points of a cell, which
// differs from run to run; these two passes replace it by the canonical one (ascending original index), so that
// the sorted arrays — and with them every sum taken over them — are bit-reproducible.  Cells hold a handful
// of points, so ranking a point against its cell mates is cheaper than any general stable sort.
__global__ void scatter_index_kernel(int64_t n, const unsigned* __restrict__ start, const unsigned* __restrict__ key,
                                     const unsigned* __restrict__ rank, unsigned* __restrict__ idx_sorted) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) idx_sorted[start[key[i]] + rank[i]] = (unsigned)i;
}
static constexpr unsigned kCanonMaxRun = 2048;   // longer runs (absurd densities) keep the arrival order
__global__ void canonical_rank_kernel(int64_t n, const unsigned* __restrict__ start, const unsigned* __restrict__ key,
                                      const unsigned* __restrict__ idx_sorted, unsigned* __restrict__ rank) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= n) return;
    const unsigned i = idx_sorted[j];
    const unsigned k = key[i];
    const unsigned s = start[k], e = start[k + 1];
    if (e - s == 1 || e - s > kCanonMaxRun) return;
    unsigned below = 0;
    for (unsigned q = s; q < e; ++q) below += __ldg(&idx_sorted[q]) < i ? 1u : 0u;
    rank[i] = below;
}
static int canonical_ranks(int64_t n, const unsigned* start, const unsigned* key, unsigned* rank, cudaStream_t st) {
    unsigned* idx_sorted = nullptr;
    O3DB_CUDA_CHECK(cudaMallocAsync(&idx_sorted, n * sizeof(unsigned), st));
    const unsigned nb = (unsigned)ceil_div(n, 256);
    scatter_index_kernel<<<nb, 256, 0, st>>>(n, start, key, rank, idx_sorted);
    O3DB_LAUNCH_CHECK();
    canonical_rank_kernel<<<nb, 256, 0, st>>>(n, start, key, idx_sorted, rank);
    O3DB_LAUNCH_CHECK();
    O3DB_CUDA_CHECK(cudaFreeAsync(idx_sorted, st));
    return O3DB_OK;
}

// Working source, CHUNK-BLOCKED: chunk c (32 consecutive sorted positions) is one 640-byte record of planes
//   [32 x float x | 32 x float y | 32 x float z | 32 x int seed | 32 x float clearance]
// so that everything a warp needs to start a chunk arrives with ONE bulk copy (it took three with separate arrays: 44
// issue slots per chunk, DESIGN.md 4.1), and a warp stores a plane back with one coalesced store of at most 128 bytes.
// 20 B per point.
// The original index of a sorted position is not in the record: only the evaluation pass (correspondences) and the
// ColoredICP set-up read it, so it lives in a separate array (o3db_icp::src_idx) that the iterations never move.
static constexpr int kSrcChunkBytes = 5 * 32 * 4;
struct SrcBlocked {
    char* base;
    __host__ __device__ static size_t bytes(int64_t n_pad) { return (size_t)(n_pad / 32) * kSrcChunkBytes; }
    __device__ __forceinline__ char* chunk(int i) const { return base + (size_t)(i >> 5) * kSrcChunkBytes; }
    // coordinate `axis` (0 = x, 1 = y, 2 = z) of point i
    __device__ __forceinline__ float* coord(int axis, int i) const {
        return reinterpret_cast<float*>(chunk(i) + 128 * axis) + (i & 31);
    }
    __device__ __forceinline__ int* seed(int i) const { return reinterpret_cast<int*>(chunk(i) + 384) + (i & 31); }
    __device__ __forceinline__ float* clearance(int i) const { return reinterpret_cast<float*>(chunk(i) + 512) + (i & 31); }
};

// no seeds, no clearances (and zeroed padding points)
__global__ void src_blocked_init_kernel(SrcBlocked sb, int64_t n, int64_t n_pad, bool clear_points) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_pad) return;
    *sb.seed((int)i) = -1;
    *sb.clearance((int)i) = 0.f;
    if (clear_points && i >= n)
        for (int axis = 0; axis < 3; ++axis) *sb.coord(axis, (int)i) = 0.f;
}

// scatter of the caller's source into the blocked working copy (clone + initial transform); src_idx[sorted position]
// receives the original index
__global__ void scatter_source_kernel(const float* __restrict__ pts, int64_t n, Affine T, const unsigned* __restrict__ start,
                                      const unsigned* __restrict__ key, const unsigned* __restrict__ rank, SrcBlocked sb,
                                      int* __restrict__ src_idx) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
    apply_transform(T.m, x, y, z);
    const unsigned p = start[key[i]] + rank[i];
    *sb.coord(0, (int)p) = x;
    *sb.coord(1, (int)p) = y;
    *sb.coord(2, (int)p) = z;
    src_idx[p] = (int)i;
}

template <bool TRANSFORM>
__global__ void scatter_kernel(const float* __restrict__ pts, const float* __restrict__ nrm, int64_t n,
                               Affine T, const unsigned* __restrict__ start,
                               const unsigned* __restrict__ key, const unsigned* __restrict__ rank,
                               float4* __restrict__ pts4, float4* __restrict__ nrm4) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
    if (TRANSFORM) apply_transform(T.m, x, y, z);
    const unsigned p = start[key[i]] + rank[i];
    pts4[p] = make_float4(x, y, z, __int_as_float((int)i));
    if (nrm4) nrm4[p] = make_float4(nrm[3 * i], nrm[3 * i + 1], nrm[3 * i + 2], 0.f);
}

// Exclusive scan of u32 data[0..n) in place; data[n] receives the total (scan.cuh).

__device__ __forceinline__ unsigned block_exclusive_scan(unsigned v, unsigned& total) {
    __shared__ unsigned s_w[kThreads / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    unsigned inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) s_w[w] = inc;
    __syncthreads();
    if (w == 0) {
        unsigned x = lane < kThreads / 32 ? s_w[lane] : 0u;
#pragma unroll
        for (int o = 1; o < kThreads / 32; o <<= 1) {
            const unsigned t = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += t;
        }
        if (lane < kThreads / 32) s_w[lane] = x;  // inclusive over warps
    }
    __syncthreads();
    total = s_w[kThreads / 32 - 1];
    const unsigned base = w ? s_w[w - 1] : 0u;
    __syncthreads();
    return base + inc - v;
}

__global__ void scan_tile_sums(const unsigned* __restrict__ data, int64_t n, unsigned* __restrict__ tile_sums) {
    const int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
    unsigned s = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k)
        if (base + k < n) s += data[base + k];
    unsigned total;
    block_exclusive_scan(s, total);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}

__global__ void scan_tile_offsets(unsigned* __restrict__ tile_sums, int64_t ntiles, unsigned* __restrict__ grand_total) {
    unsigned carry = 0;
    for (int64_t b = 0; b < ntiles; b += kThreads) {
        const int64_t i = b + threadIdx.x;
        const unsigned v = i < ntiles ? tile_sums[i] : 0u;
        unsigned total;
        const unsigned ex = block_exclusive_scan(v, total);
        if (i < ntiles) tile_sums[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) *grand_total = carry;
}

__global__ void scan_apply(unsigned* __restrict__ data, int64_t n, const unsigned* __restrict__ tile_offsets) {
    const int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
    unsigned v[kScanItems];
    unsigned s = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        v[k] = base + k < n ? data[base + k] : 0u;
        s += v[k];
    }
    unsigned total;
    unsigned ex = block_exclusive_scan(s, total) + tile_offsets[blockIdx.x];
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        if (base + k < n) data[base + k] = ex;
        ex += v[k];
    }
}

// data has n+1 entries; scratch has ceil(n/kScanTile) entries.
int exclusive_scan_u32(unsigned* data, int64_t n, unsigned* scratch, cudaStream_t st) {
    const int64_t ntiles = ceil_div(n, kScanTile);
    scan_tile_sums<<<(unsigned)ntiles, kThreads, 0, st>>>(data, n, scratch);
    O3DB_LAUNCH_CHECK();
    scan_tile_offsets<<<1, kThreads, 0, st>>>(scratch, ntiles, data + n);
    O3DB_LAUNCH_CHECK();
    scan_apply<<<(unsigned)ntiles, kThreads, 0, st>>>(data, n, scratch);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}


// ------------------------------------- reference-layout CSR table (interop)

// core/nns/NeighborSearchCommon.h:31-52 + FixedRadiusSearchImpl.cuh:63-134.
__device__ __forceinline__ unsigned ref_bucket(const float* __restrict__ p, float inv_voxel, unsigned table_size) {
    const int vx = (int)floorf(p[0] * inv_voxel), vy = (int)floorf(p[1] * inv_voxel), vz = (int)floorf(p[2] * inv_voxel);
    const unsigned h32 = ((unsigned)vx * 73856096u) ^ ((unsigned)vy * 193649663u) ^ ((unsigned)vz * 83492791u);
    const uint64_t h = (uint64_t)(int64_t)(int)h32;   // int -> size_t sign-extends
    return (unsigned)(h % (uint64_t)table_size);
}

__global__ void ref_count_kernel(const float* __restrict__ pts, int64_t n, float inv_voxel, unsigned table_size,
                                 unsigned* __restrict__ count, unsigned* __restrict__ rank) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    rank[i] = atomicAdd(&count[ref_bucket(pts + 3 * i, inv_voxel, table_size)], 1u);
}

__global__ void ref_scatter_kernel(const float* __restrict__ pts, int64_t n, float inv_voxel, unsigned table_size,
                                   const unsigned* __restrict__ start, const unsigned* __restrict__ rank,
                                   unsigned* __restrict__ index) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    index[start[ref_bucket(pts + 3 * i, inv_voxel, table_size)] + rank[i]] = (unsigned)i;
}

// ------------------------------------------------------------------ index

}  // namespace o3db

using namespace o3db;

struct o3db_nns {
    cudaStream_t stream = 0;   // creation stream (buffers are freed on it)
    Grid g{};
    double radius = 0;
    int64_t m = 0;
    int64_t ncell = 0;
    float4* pts4 = nullptr;
    float4* nrm4 = nullptr;
    unsigned* cell_start = nullptr;
};

namespace o3db {

static void nns_free(o3db_nns* s, cudaStream_t st) {
    if (!s) return;
    if (s->pts4) cudaFreeAsync(s->pts4, st);
    if (s->nrm4) cudaFreeAsync(s->nrm4, st);
    if (s->cell_start) cudaFreeAsync(s->cell_start, st);
    s->pts4 = s->nrm4 = nullptr;
    s->cell_start = nullptr;
}

static constexpr double kThinMergeMax = 8.0;   // merge the whole thin axis into ONE cell while a (y, z) column holds at most this many points on average
static int grid_from_bbox(const float mn[3], const float mx[3], double radius, double cell_scale, int64_t m, Grid* g,
                          int64_t* ncell) {
    double c = radius * (cell_scale > 0 ? cell_scale : 1.0) * (1.0 + 1e-4);
    if (!(c > 0) || !std::isfinite(c)) c = 1.0;
    double ext[3];
    double maxabs = 0;
    for (int a = 0; a < 3; ++a) {
        ext[a] = std::max(0.0, (double)mx[a] - (double)mn[a]);
        maxabs = std::max(maxabs, std::max(std::fabs((double)mn[a]), std::fabs((double)mx[a])));
    }
    // grid axis order: fastest = the real axis with the smallest extent (ties: z, then y),
    // slowest = the one with the largest
    int order[3] = {2, 1, 0};
    std::stable_sort(order, order + 3, [&](int a, int b) { return ext[a] < ext[b]; });
    for (int k = 0; k < 3; ++k) g->ax[k] = order[k];
    double cx = c * kThinFactor;
    for (;;) {
        double n[3];
        bool ok = true;
        double prod = 1;
        // Surface-like clouds: when a (y, z) column of cells holds only a handful of points over the WHOLE thin
        // extent, the thin axis becomes a single cell (slab scans cross all of it anyway): the CSR table
        // shrinks by nx and a slab boundary is one multiply-free lookup.  Volumetric clouds keep thin cells.
        const double cols = (std::floor(ext[order[1]] / c) + 1) * (std::floor(ext[order[2]] / c) + 1);
        cx = c * kThinFactor;
        if ((double)m <= kThinMergeMax * cols) cx = std::max(cx, ext[order[0]] * (1.0 + 1e-3) + c);
        for (int k = 0; k < 3; ++k) {
            n[k] = std::floor(ext[order[k]] / (k == 0 ? cx : c)) + 1;
            ok = ok && n[k] <= kMaxCellsPerAxis;
            prod *= n[k];
        }
        if (ok && prod <= (double)kMaxCells) {
            g->nx = (int)n[0];
            g->ny = (int)n[1];
            g->nz = (int)n[2];
            break;
        }
        c *= 1.25;
    }
    g->c = (float)c;
    g->inv_c = 1.0f / g->c;
    g->cx = (float)cx;
    g->inv_cx = 1.0f / g->cx;
    g->ox = mn[order[0]];
    g->oy = mn[order[1]];
    g->oz = mn[order[2]];
    g->tol = (float)(c * 2e-3 + maxabs * 1e-6);
    for (int k = 0; k < 3; ++k) {
        g->bmin[k] = mn[order[k]];
        g->bmax[k] = mx[order[k]];
    }
    *ncell = (int64_t)g->nx * g->ny * g->nz;
    return O3DB_OK;
}

// Builds pts4 / nrm4 / cell_start for `pts` (device).  Synchronises `st` once
// (the grid dimensions depend on the bounding box).
static int nns_build(o3db_nns* s, const float* pts, const float* nrm, int64_t m, double radius,
                     double cell_scale, cudaStream_t st) {
    configure_memory_pool();
    s->stream = st;
    s->m = m;
    s->radius = radius;
    unsigned* d_bbox = nullptr;
    O3DB_CUDA_CHECK(cudaMallocAsync(&d_bbox, 6 * sizeof(unsigned), st));
    const unsigned init[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};
    O3DB_CUDA_CHECK(cudaMemcpyAsync(d_bbox, init, sizeof(init), cudaMemcpyHostToDevice, st));
    const int blocks = (int)std::min<int64_t>(ceil_div(m, kThreads), (int64_t)num_sms() * 8);
    bbox_kernel<<<blocks, kThreads, 0, st>>>(pts, m, d_bbox);
    O3DB_LAUNCH_CHECK();
    unsigned h_bbox[6];
    O3DB_CUDA_CHECK(cudaMemcpyAsync(h_bbox, d_bbox, sizeof(h_bbox), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    O3DB_CUDA_CHECK(cudaFreeAsync(d_bbox, st));
    float mn[3], mx[3];
    for (int a = 0; a < 3; ++a) {
        mn[a] = ordered_to_float(h_bbox[a]);
        mx[a] = ordered_to_float(h_bbox[3 + a]);
        if (!(mn[a] <= mx[a]) || !std::isfinite(mn[a]) || !std::isfinite(mx[a])) {
            set_last_error("target point cloud has non-finite coordinates");
            return O3DB_ERR_INVALID;
        }
    }
    grid_from_bbox(mn, mx, radius, cell_scale, m, &s->g, &s->ncell);

    unsigned *key = nullptr, *rank = nullptr, *scratch = nullptr;
    O3DB_CUDA_CHECK(cudaMallocAsync(&s->cell_start, (s->ncell + 1) * sizeof(unsigned), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&s->pts4, m * sizeof(float4), st));
    if (nrm) O3DB_CUDA_CHECK(cudaMallocAsync(&s->nrm4, m * sizeof(float4), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&key, m * sizeof(unsigned), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&rank, m * sizeof(unsigned), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&scratch, ceil_div(s->ncell, kScanTile) * sizeof(unsigned), st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(s->cell_start, 0, (s->ncell + 1) * sizeof(unsigned), st));
    Affine id{};
    const unsigned nb = (unsigned)ceil_div(m, kThreads);
    count_kernel<false><<<nb, kThreads, 0, st>>>(pts, m, s->g, id, s->cell_start, key, rank);
    O3DB_LAUNCH_CHECK();
    int rc = exclusive_scan_u32(s->cell_start, s->ncell, scratch, st);
    if (rc) return rc;
    rc = canonical_ranks(m, s->cell_start, key, rank, st);
    if (rc) return rc;
    scatter_kernel<false><<<nb, kThreads, 0, st>>>(pts, nrm, m, id, s->cell_start, key, rank, s->pts4, s->nrm4);
    O3DB_LAUNCH_CHECK();
    O3DB_CUDA_CHECK(cudaFreeAsync(key, st));
    O3DB_CUDA_CHECK(cudaFreeAsync(rank, st));
    O3DB_CUDA_CHECK(cudaFreeAsync(scratch, st));
    return O3DB_OK;
}

// ------------------------------------------------------- stand-alone search

template <bool PRUNE>
__global__ void __launch_bounds__(kThreads)
hybrid_search_k1_kernel(Grid g, const float4* __restrict__ pts, const unsigned* __restrict__ cs,
                        const float* __restrict__ q, int64_t n, float rr, float thr,
                        int32_t* __restrict__ idx, float* __restrict__ dist, int32_t* __restrict__ cnt) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    Best b;
    nn_search<PRUNE>(g, pts, cs, q[3 * i], q[3 * i + 1], q[3 * i + 2], rr, thr, b);
    if (idx) idx[i] = b.j >= 0 ? b.idx : -1;
    if (dist) dist[i] = b.j >= 0 ? b.d : 0.f;
    if (cnt) cnt[i] = b.j >= 0 ? 1 : 0;
}

static constexpr int kMaxKnn = 32;

// General max_knn (small): per-thread sorted list, same visiting scheme without pruning.
__global__ void __launch_bounds__(kThreads)
hybrid_search_knn_kernel(Grid g, const float4* __restrict__ pts, const unsigned* __restrict__ cs,
                         const float* __restrict__ q, int64_t n, float rr, float thr, int k,
                         int32_t* __restrict__ idx, float* __restrict__ dist, int32_t* __restrict__ cnt) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float qx = q[3 * i], qy = q[3 * i + 1], qz = q[3 * i + 2];
    int bi[kMaxKnn];
    float bd[kMaxKnn];
    int c = 0;
    float gx, gy, gz;
    to_grid(g, qx, qy, qz, gx, gy, gz);
    const float lx = lo_bound(gx, rr), hx = hi_bound(gx, rr);
    const float ly = lo_bound(gy, rr), hy = hi_bound(gy, rr);
    const float lz = lo_bound(gz, rr), hz = hi_bound(gz, rr);
    const bool outside = hx < g.bmin[0] || lx > g.bmax[0] || hy < g.bmin[1] || ly > g.bmax[1] ||
                         hz < g.bmin[2] || lz > g.bmax[2] || !(qx == qx) || !(qy == qy) || !(qz == qz);
    if (!outside) {
        const int x0 = cell1(lx, g.ox, g.inv_cx, g.nx), x1 = cell1(hx, g.ox, g.inv_cx, g.nx);
        const int y0 = cell1(ly, g.oy, g.inv_c, g.ny), y1 = cell1(hy, g.oy, g.inv_c, g.ny);
        const int z0 = cell1(lz, g.oz, g.inv_c, g.nz), z1 = cell1(hz, g.oz, g.inv_c, g.nz);
        for (int iz = z0; iz <= z1; ++iz)
            for (int iy = y0; iy <= y1; ++iy) {
                const int row = (iz * g.ny + iy) * g.nx;
                const unsigned s = cs[row + x0], e = cs[row + x1 + 1];
                for (unsigned j = s; j < e; ++j) {
                    const float4 t = __ldg(&pts[j]);
                    const float dx = t.x - qx, dy = t.y - qy, dz = t.z - qz;
                    const float d = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
                    if (!(d <= thr)) continue;
                    const int id = __float_as_int(t.w);
                    int m = c;
                    if (m == k) {
                        if (d > bd[m - 1] || (d == bd[m - 1] && id > bi[m - 1])) continue;
                        m = k - 1;
                    }
                    int pos = m;
                    while (pos > 0 && (bd[pos - 1] > d || (bd[pos - 1] == d && bi[pos - 1] > id))) {
                        bd[pos] = bd[pos - 1];
                        bi[pos] = bi[pos - 1];
                        --pos;
                    }
                    bd[pos] = d;
                    bi[pos] = id;
                    c = m + 1;
                }
            }
    }
    for (int j = 0; j < k; ++j) {
        if (idx) idx[i * k + j] = j < c ? bi[j] : -1;
        if (dist) dist[i * k + j] = j < c ? bd[j] : 0.f;
    }
    if (cnt) cnt[i] = c;
}

// --------------------------------------------------------- robust kernels

struct Robust {
    int method;
    float scale;
    double shape;
};

// RobustKernelImpl.h:35-115 for scalar_t = float (double literals promote as upstream).
__device__ __forceinline__ float robust_weight(const Robust& k, float r) {
    switch (k.method) {
        case O3DB_ROBUST_L2: return 1.0f;
        case O3DB_ROBUST_L1: return (float)(1.0 / fabsf(r));
        case O3DB_ROBUST_HUBER: return k.scale / fmaxf(fabsf(r), k.scale);
        case O3DB_ROBUST_CAUCHY: {
            const float q = r / k.scale;
            return (float)(1.0 / (1.0 + (double)(q * q)));
        }
        case O3DB_ROBUST_GM: {
            const float s = k.scale + r * r;
            return k.scale / (s * s);
        }
        case O3DB_ROBUST_TUKEY: {
            const float q = fminf(1.0f, fabsf(r) / k.scale);
            const double v = 1.0 - (double)(q * q);
            return (float)(v * v);
        }
        default: {  // generalized
            const float s2 = k.scale * k.scale;
            // open3d::IsClose (GeometryMacros.h:58-63) is relative: the shape ~ 0 branch of
            // RobustKernelImpl.h:85-91 can never be taken; only shape ~ 2 is special-cased.
            if (k.shape > (1.0 - 1e-3) * 2.0 && k.shape < (1.0 + 1e-3) * 2.0) return (float)(1.0 / (double)s2);
            const float q = r / k.scale;
            if (k.shape < -1e7) return (float)(exp((double)(q * q) / (-2.0)) / (double)s2);
            return (float)(pow((double)(q * q) / fabs(k.shape - 2.0) + 1, (k.shape / 2.0) - 1.0) / (double)s2);
        }
    }
}

// ------------------------------------------------- 29(+1)-scalar reduction (reduce.cuh)

// RegistrationImpl.h:251-287 + RegistrationCUDA.cu:29-79 slot layout.
template <bool L2LOSS, int NACC>
__device__ __forceinline__ void accumulate_p2plane(float (&acc)[NACC], const Robust& rk, float sx, float sy,
                                                   float sz, float tx, float ty, float tz, float nx, float ny,
                                                   float nz) {
    // r and J are evaluated without FMA contraction, in the reference's operation order, so
    // that residual-dependent robust weights (e.g. L1: 1/|r|) see the same r as the CPU path
    // even when (s - t).n cancels to ~0; the accumulation below may fuse.
    const float r = __fadd_rn(__fadd_rn(__fmul_rn(__fsub_rn(sx, tx), nx), __fmul_rn(__fsub_rn(sy, ty), ny)),
                              __fmul_rn(__fsub_rn(sz, tz), nz));
    float J[6];
    J[0] = __fsub_rn(__fmul_rn(nz, sy), __fmul_rn(ny, sz));
    J[1] = __fsub_rn(__fmul_rn(nx, sz), __fmul_rn(nz, sx));
    J[2] = __fsub_rn(__fmul_rn(ny, sx), __fmul_rn(nx, sy));
    J[3] = nx;
    J[4] = ny;
    J[5] = nz;
    const float w = L2LOSS ? 1.0f : robust_weight(rk, r);
    int s = 0;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        const float jw = J[j] * w;
#pragma unroll
        for (int k = 0; k <= j; ++k) acc[s++] += jw * J[k];
        acc[21 + j] += jw * r;
    }
    acc[27] += r;
    acc[28] += 1.0f;
}

// ComputePoseColoredICP per-correspondence body (RegistrationImpl.h:337-425 / RegistrationCUDA.cu:119-183):
// geometric + photometric Jacobian rows, two robust weights, same 29-slot layout.
template <bool L2LOSS, int NACC>
__device__ __forceinline__ void accumulate_colored(float (&acc)[NACC], const Robust& rk, const float (&vs)[3],
                                                   const float (&vt)[3], const float (&nt)[3], float is, float it,
                                                   const float (&dit)[3], float sqrt_lg, float sqrt_lp) {
    const float d = (vs[0] - vt[0]) * nt[0] + (vs[1] - vt[1]) * nt[1] + (vs[2] - vt[2]) * nt[2];
    float JG[6], JI[6];
    JG[0] = sqrt_lg * (-vs[2] * nt[1] + vs[1] * nt[2]);
    JG[1] = sqrt_lg * (vs[2] * nt[0] - vs[0] * nt[2]);
    JG[2] = sqrt_lg * (-vs[1] * nt[0] + vs[0] * nt[1]);
    JG[3] = sqrt_lg * nt[0];
    JG[4] = sqrt_lg * nt[1];
    JG[5] = sqrt_lg * nt[2];
    const float rG = sqrt_lg * d;
    const float vp[3] = {vs[0] - d * nt[0], vs[1] - d * nt[1], vs[2] - d * nt[2]};
    const float is_proj = dit[0] * (vp[0] - vt[0]) + dit[1] * (vp[1] - vt[1]) + dit[2] * (vp[2] - vt[2]) + it;
    const float sd = dit[0] * nt[0] + dit[1] * nt[1] + dit[2] * nt[2];
    const float dM[3] = {sd * nt[0] - dit[0], sd * nt[1] - dit[1], sd * nt[2] - dit[2]};
    JI[0] = sqrt_lp * (-vs[2] * dM[1] + vs[1] * dM[2]);
    JI[1] = sqrt_lp * (vs[2] * dM[0] - vs[0] * dM[2]);
    JI[2] = sqrt_lp * (-vs[1] * dM[0] + vs[0] * dM[1]);
    JI[3] = sqrt_lp * dM[0];
    JI[4] = sqrt_lp * dM[1];
    JI[5] = sqrt_lp * dM[2];
    const float rI = sqrt_lp * (is - is_proj);
    const float wG = L2LOSS ? 1.0f : robust_weight(rk, rG);
    const float wI = L2LOSS ? 1.0f : robust_weight(rk, rI);
    int p = 0;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
#pragma unroll
        for (int k = 0; k <= j; ++k) acc[p++] += JG[j] * wG * JG[k] + JI[j] * wI * JI[k];
        acc[21 + j] += JG[j] * wG * rG + JI[j] * wI * rI;
    }
    acc[27] += rG * rG + rI * rI;
    acc[28] += 1.0f;
}

// intensity of an RGB triple exactly as upstream: float sum, divided by the double literal 3.0
__device__ __forceinline__ float color_intensity(float r, float g, float b) { return (float)((r + g + b) / 3.0); }

// -------------------------------------------- stand-alone pose reductions

struct PoseOut {
    double* sums29;
    double* pose;
    int* status;  // device int: 0 ok, 1 singular
};

// Last block of a pose reduction: the sums out, the f64 solve by one thread, the pose (zero for a singular system)
// and its status.
__device__ __forceinline__ void pose_epilogue(const double* s_final, const PoseOut& out) {
    if (threadIdx.x < 29 && out.sums29) out.sums29[threadIdx.x] = s_final[threadIdx.x];
    if (threadIdx.x == 0) {
        double pose[6] = {0, 0, 0, 0, 0, 0};
        const bool ok = solve6x6(s_final, pose);
        if (!ok)
            for (int k = 0; k < 6; ++k) pose[k] = 0.0;
        if (out.pose)
            for (int k = 0; k < 6; ++k) out.pose[k] = pose[k];
        if (out.status) *out.status = ok ? 0 : 1;
    }
}

// ComputePosePointToPlaneKernelCUDA (RegistrationCUDA.cu:29-79) with int64 correspondences.
template <bool L2LOSS>
__global__ void __launch_bounds__(kThreads)
pose_p2plane_kernel(const float* __restrict__ src, const float* __restrict__ tgt, const float* __restrict__ nrm,
                    const int64_t* __restrict__ corr, int64_t n, Robust rk, double* __restrict__ partials,
                    unsigned* ticket, PoseOut out) {
    __shared__ double s_warp[kThreads / 32][kSumStride];
    __shared__ double s_final[kSumStride];
    if (!reduce_sums(n, s_warp, partials, ticket, s_final, [&](int64_t i, float (&acc)[kNumSums]) {
            const int64_t c = corr[i];
            if (c == -1) return;
            const float* t = tgt + 3 * c;
            const float* m = nrm + 3 * c;
            accumulate_p2plane<L2LOSS, kNumSums>(acc, rk, src[3 * i], src[3 * i + 1], src[3 * i + 2], t[0], t[1], t[2],
                                                 m[0], m[1], m[2]);
        }))
        return;
    pose_epilogue(s_final, out);
}

// ComputePoseColoredICPKernelCUDA (RegistrationCUDA.cu:119-180), RegistrationImpl.h:413-493.
template <bool L2LOSS>
__global__ void __launch_bounds__(kThreads)
pose_colored_kernel(const float* __restrict__ src, const float* __restrict__ src_c, const float* __restrict__ tgt,
                    const float* __restrict__ nrm, const float* __restrict__ tgt_c,
                    const float* __restrict__ tgt_g, const int64_t* __restrict__ corr, int64_t n, float sqrt_lg,
                    float sqrt_lp, Robust rk, double* __restrict__ partials, unsigned* ticket, PoseOut out) {
    __shared__ double s_warp[kThreads / 32][kSumStride];
    __shared__ double s_final[kSumStride];
    if (!reduce_sums(n, s_warp, partials, ticket, s_final, [&](int64_t i, float (&acc)[kNumSums]) {
            if (corr[i] == -1) return;
            const int64_t t = 3 * corr[i], s = 3 * i;
            const float vs[3] = {src[s], src[s + 1], src[s + 2]};
            const float vt[3] = {tgt[t], tgt[t + 1], tgt[t + 2]};
            const float nt[3] = {nrm[t], nrm[t + 1], nrm[t + 2]};
            const float is = color_intensity(src_c[s], src_c[s + 1], src_c[s + 2]);
            const float it = color_intensity(tgt_c[t], tgt_c[t + 1], tgt_c[t + 2]);
            const float dit[3] = {tgt_g[t], tgt_g[t + 1], tgt_g[t + 2]};
            accumulate_colored<L2LOSS, kNumSums>(acc, rk, vs, vt, nt, is, it, dit, sqrt_lg, sqrt_lp);
        }))
        return;
    pose_epilogue(s_final, out);
}

// ComputeRtPointToPointCPU (RegistrationCPU.cpp:619-653) with int64 correspondences: Get3x3SxyLinearSystem as one
// pass of raw moments about a pivot (reduce.cuh; here the first target point, which lies within the cloud's extent of
// every matched point), then the Kabsch step by warp 0 of the last block.  out[0, 16): the row-major 4 x 4 [R t; 0 1]
// (unwritten without a valid correspondence), out[16]: the number of valid correspondences.
__global__ void __launch_bounds__(kThreads)
rt_p2point_kernel(const float* __restrict__ src, const float* __restrict__ tgt, const int64_t* __restrict__ corr, int64_t n,
                  double* __restrict__ partials, unsigned* ticket, double* __restrict__ out) {
    __shared__ double s_warp[kThreads / 32][kSumStride];
    __shared__ double s_final[kSumStride];
    __shared__ float s_pivot[3];
    const float pivot[3] = {__ldg(&tgt[0]), __ldg(&tgt[1]), __ldg(&tgt[2])};
    if (!reduce_sums(n, s_warp, partials, ticket, s_final, [&](int64_t i, float (&acc)[kNumSums]) {
            const int64_t c = corr[i];
            if (c == -1) return;
            const float* t = tgt + 3 * c;
            const float vs[3] = {src[3 * i] - pivot[0], src[3 * i + 1] - pivot[1], src[3 * i + 2] - pivot[2]};
            const float vt[3] = {t[0] - pivot[0], t[1] - pivot[1], t[2] - pivot[2]};
            accumulate_p2point<kNumSums>(acc, vs, vt);
        }))
        return;
    if (threadIdx.x >= 32) return;
    if (threadIdx.x < 3) s_pivot[threadIdx.x] = pivot[threadIdx.x];
    __syncwarp();
    if (s_final[kCountSlot] > 0) {
        double* scratch = &s_warp[0][0];   // (dead: the sums are in s_final)
        kabsch_step_warp(s_final, s_pivot, scratch);
        if (threadIdx.x < 16) out[threadIdx.x] = scratch[16 + threadIdx.x];
    }
    if (threadIdx.x == 0) out[16] = s_final[kCountSlot];
}

// ComputeInformationMatrixKernelCUDA (RegistrationCUDA.cu:492-533) with GetInformationJacobians (RegistrationImpl.h:686-715):
// the 21 lower-triangle terms of GTG per matched target point (f32, upstream's expression), reduced like the pose sums
// (f32 per thread over a few terms, then f64: deterministic, and closer to the exact sum than upstream's f32 atomics).
// corr_i32: the hybrid search's own Int32 index column (-1 = none); corr_i64: a caller's Int64 correspondence set.
__global__ void __launch_bounds__(kThreads)
information_matrix_kernel(const float* __restrict__ tgt, const int32_t* __restrict__ corr_i32, const int64_t* __restrict__ corr_i64,
                          int64_t n, double* __restrict__ partials, unsigned* ticket, double* __restrict__ sums_out) {
    __shared__ double s_warp[kThreads / 32][kSumStride];
    __shared__ double s_final[kSumStride];
    if (!reduce_sums(n, s_warp, partials, ticket, s_final, [&](int64_t i, float (&acc)[kNumSums]) {
            const int64_t c = corr_i32 ? (int64_t)corr_i32[i] : corr_i64[i];
            if (c == -1) return;
            const float* p = tgt + 3 * c;
            const float px = p[0], py = p[1], pz = p[2];
            const float Jx[6] = {0.f, pz, -py, 1.f, 0.f, 0.f};
            const float Jy[6] = {-pz, 0.f, px, 0.f, 1.f, 0.f};
            const float Jz[6] = {py, -px, 0.f, 0.f, 0.f, 1.f};
            int q = 0;
#pragma unroll
            for (int j = 0; j < 6; ++j)
#pragma unroll
                for (int k = 0; k <= j; ++k)
                    acc[q++] += __fadd_rn(__fadd_rn(__fmul_rn(Jx[j], Jx[k]), __fmul_rn(Jy[j], Jy[k])), __fmul_rn(Jz[j], Jz[k]));
            acc[28] += 1.0f;
        }))
        return;
    if (threadIdx.x < kNumSums) sums_out[threadIdx.x] = s_final[threadIdx.x];
}

// ------------------------------------------------------ transform kernels

__global__ void transform_points_kernel(float* __restrict__ p, int64_t n, Affine T) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
    apply_transform(T.m, x, y, z);
    p[3 * i] = x;
    p[3 * i + 1] = y;
    p[3 * i + 2] = z;
}

__global__ void transform_normals_kernel(float* __restrict__ p, int64_t n, Affine T) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
    p[3 * i] = T.m[0] * x + T.m[1] * y + T.m[2] * z;
    p[3 * i + 1] = T.m[4] * x + T.m[5] * y + T.m[6] * z;
    p[3 * i + 2] = T.m[8] * x + T.m[9] * y + T.m[10] * z;
}

// ColoredICP side arrays, in the sort order of the working clouds (orig index = .w of the target's float4, src_idx of
// the source)
__global__ void pack_target_color_kernel(const float4* __restrict__ pts4, const float* __restrict__ col,
                                         const float* __restrict__ grad, int64_t m, float4* __restrict__ tcg) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= m) return;
    const int64_t o = 3 * (int64_t)__float_as_int(pts4[j].w);
    tcg[j] = make_float4(grad[o], grad[o + 1], grad[o + 2], color_intensity(col[o], col[o + 1], col[o + 2]));
}

__global__ void pack_source_intensity_kernel(const int* __restrict__ src_idx, const float* __restrict__ col,
                                             int64_t n, float* __restrict__ sint) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t o = 3 * (int64_t)src_idx[i];
    sint[i] = color_intensity(col[o], col[o + 1], col[o + 2]);
}

// ------------------------------------------------------------ fused ICP loop

// The estimator of a handle: which per-query terms an iteration adds and which step turns the totals into an update.
enum : int { kEstPlane = 0, kEstColored = 1, kEstPoint = 2 };

struct IcpState {        // lives in device memory; read back once at the end
    double T[16];        // cumulative source->target transformation (f64)
    double sums[kSumStride];
    double prev_fitness, prev_rmse, fitness, rmse;
    double count;        // correspondences of the last search
    float Uf[16];        // pending update to apply to the working source (f32)
    int iter;            // == reference's iteration_count
    int executed;        // iterations whose (fitness, rmse) were logged
    int done;            // loop left (converged / no correspondences / singular)
    int converged;
    int status;          // 0 ok, 1 singular
    unsigned ticket;
    int sums_cached;     // chunk_sums holds every chunk's line for the working source as it is now (see IcpArgs)
};

struct IcpArgs {
    Grid g;
    const float4* tgt;
    const float4* nrm;
    const unsigned* cs;
    SrcBlocked src;       // working source, sorted, chunk-blocked: point, seed = sorted target position of its last
                          // winner (-1 = none), clearance of that winner (lower bound on the distance to every OTHER
                          // target point, minus the motion since it was established; 0 = unknown)
    const int* src_idx;   // sorted source position -> original index (read in evaluate mode with corr_out only)
    float* chunk_sums;    // per 32-query chunk, the 32 f32 sums its last iteration added to the warp's totals (128 B)
    int64_t n;            // local source points
    double n_total;       // source points over all ranks (fitness denominator)
    float rr, thr;
    float r1, r1_accept2;   // pass-1 radius of the two-pass search (= cell size) and its acceptance bound
    Robust rk;
    double* partials;
    IcpState* st;
    double* per_iter;
    int64_t* corr_out;    // evaluate mode only
    double rel_fitness, rel_rmse;
    int max_iteration;
    int fuse_finalize;    // 0: leave the totals in st->sums (multi-GPU all-reduce follows)
    // ColoredICP only (null otherwise)
    const float4* tcg;    // per sorted target point: colour gradient xyz, .w = intensity
    const float* sint;    // per sorted source point: intensity
    float sqrt_lg, sqrt_lp;
    // multi-GPU, in-kernel exchange (use_peer != 0): every rank's mailbox as mapped into this process
    PeerView peer;
    int use_peer;
    // point-to-point only: the pivot the moments are taken about (centre of the target's bounding box, world axes)
    int point_to_point;
    float pivot[3];
};

__device__ void set_identity(double* T, float* Uf) {
    for (int i = 0; i < 16; ++i) {
        const double v = (i % 5 == 0) ? 1.0 : 0.0;
        if (T) T[i] = v;
        if (Uf) Uf[i] = (float)v;
    }
}

// Threads per block of the iteration kernel: ONE fat block of 24 warps per SM (80 registers x 768 threads fills the
// register file): a third of the per-block partial rows for the last block to add up (one per SM instead of three)
// and a third of the block prologues / epilogues; the loop itself has no block-wide barrier either way.  On an H100
// it is 3-6 % faster than three 256-thread blocks per SM (profiles/h100_reduce_ab.jsonl).
static constexpr int kIcpThreads = 768;

// Host part of DoSingleScaleICPIterations (Registration.cpp:293-358), on device, run by ONE WARP once per
// iteration (all 32 lanes must call it): gauss_newton_step_warp and left_multiply_warp (reduce.cuh) spread the
// step over lanes, lane 0 keeps the books.  `s_scratch`: the step's scratch.
template <bool POINT>
__device__ void icp_finalize_iteration(const IcpArgs& a, const double* sums, double* s_scratch) {
    IcpState* st = a.st;
    const int lane = threadIdx.x & 31;
    const double count = sums[28];
    const double fitness = count / a.n_total;                       // Registration.cpp:47-50
    const double rmse = count > 0 ? sqrt(sums[29] / count) : 0.0;
    if (!(fitness > DBL_MIN)) {  // :51-60, :300-306 — no correspondences
        if (lane == 0) {
            st->fitness = fitness;
            st->rmse = rmse;
            st->count = count;
            set_identity(st->T, st->Uf);
            st->converged = 0;
            st->done = 1;
        }
        return;
    }
    if (POINT) {   // ComputeRtPointToPoint (kernel/Registration.cpp:365-404): no singular case
        kabsch_step_warp(sums, a.pivot, s_scratch);
    } else if (!gauss_newton_step_warp(sums, s_scratch)) {  // TransformationConverter.cpp:219-225 — the reference raises
        if (lane == 0) {
            st->fitness = fitness;
            st->rmse = rmse;
            st->count = count;
            set_identity(nullptr, st->Uf);
            st->status = 1;
            st->done = 1;
        }
        return;
    }
    const double* U = s_scratch + 16;
    if (lane < 16) {                     // :319  T <- U * T
        left_multiply_warp(U, st->T);
        st->Uf[lane] = (float)U[lane];   // :322 applied by the next kernel's load
    }
    if (lane == 0) {
        st->fitness = fitness;
        st->rmse = rmse;
        st->count = count;
        if (a.per_iter) {
            a.per_iter[2 * st->executed] = fitness;
            a.per_iter[2 * st->executed + 1] = rmse;
        }
        st->executed += 1;
        if (st->iter != 0 && fabs(st->prev_fitness - fitness) < a.rel_fitness &&
            fabs(st->prev_rmse - rmse) < a.rel_rmse) {  // :348-355
            st->converged = 1;
            st->done = 1;
        } else {
            st->prev_fitness = fitness;
            st->prev_rmse = rmse;
            st->iter += 1;
            if (st->iter >= a.max_iteration) st->done = 1;
        }
    }
}

// Final ComputeRegistrationResult (Registration.cpp:424-431).
__device__ void icp_finalize_evaluate(const IcpArgs& a, const double* sums) {
    IcpState* st = a.st;
    const double count = sums[28];
    st->count = count;
    if (count > 0) {
        st->fitness = count / a.n_total;
        st->rmse = sqrt(sums[29] / count);
    } else {
        st->fitness = 0.0;
        st->rmse = 0.0;
        set_identity(st->T, nullptr);
        st->converged = 0;
    }
    set_identity(nullptr, st->Uf);
}

// ------------------------------------------------------- one query of one iteration

// Everything one working source point does in one iteration: apply the pending update (the reference's
// separate PointCloud::Transform pass, Registration.cpp:322) and store it back, exact 1-NN within the radius
// (seeded by last iteration's winner `jp` when there is one: ts / nn / cg are that target point, its normal and
// its colour row, fetched by the caller; point-to-point has neither), the estimator's terms + count and sum of d^2,
// new seed.
// MODE 0 = iterate, MODE 1 = evaluate (no Jacobian; writes correspondences in the caller's order).
template <bool L2LOSS, int MODE, int EST>
__device__ __forceinline__ bool icp_process_query(const IcpArgs& a, const float* s_U, int i, float px, float py, float pz,
                                                  int jp, float clear_prev, const float4* seed_ts, const float4* seed_nn,
                                                  const float4* seed_cg, float (&acc)[32]) {
    const float ox = px, oy = py, oz = pz;
    apply_transform(s_U, px, py, pz);
    // Only values whose bits changed are stored back: a store marks its 32-byte sector dirty, and the sector goes back
    // to HBM, even when it rewrites the bits already there.  Once the clouds are aligned, the pending update leaves
    // most coordinates (and with them the clearance) bit-for-bit where they were, and a sector of a plane (8 lanes)
    // whose lanes all skip their store stays clean.
    if (__float_as_uint(px) != __float_as_uint(ox)) *a.src.coord(0, i) = px;
    if (__float_as_uint(py) != __float_as_uint(oy)) *a.src.coord(1, i) = py;
    if (__float_as_uint(pz) != __float_as_uint(oz)) *a.src.coord(2, i) = pz;
    unsigned bj = kNoPoint;
    bool handled = false;
    float clear_new = 0.f;      // what is known about the distance to every point other than the winner
    float4 ts = make_float4(0.f, 0.f, 0.f, 0.f);
    if (jp >= 0) {
        // "Still the winner" certificate (the Elkan / Hamerly bound of accelerated k-means, applied to ICP
        // correspondences): when this query was last searched, every target point other than its winner was at
        // least `clearance` away; since then the query has moved by at most the accumulated |p_new - p_old|
        // (triangle inequality), which clear_prev already has subtracted.  If the old winner is now strictly
        // closer than that bound, it is the exact nearest neighbour — no table lookup, no candidate scan.
        // All roundings go against the certificate (round-down subtraction, 1e-5 margins on both roots).
        ts = *seed_ts;
        const float sd = dist2_canonical(ts, px, py, pz);
        const float mx = px - ox, my = py - oy, mz = pz - oz;
        const float m2 = fmaf(mz, mz, fmaf(my, my, mx * mx));
        const float moved = m2 > 0.f ? __fmul_ru(m2 * rsqrtf(m2), 1.00001f) : 0.f;
        const float clear = __fsub_rd(clear_prev, moved);
        const float r1 = sd > 0.f ? __fmul_ru(sd * rsqrtf(sd), 1.00001f) : 0.f;
        if (sd <= a.thr) {
            if (r1 < clear) {
                bj = (unsigned)jp;
                clear_new = clear;
                handled = true;
            } else {
                bj = nn_search_seeded_fast(a.g, a.tgt, a.cs, px, py, pz, a.r1, a.r1_accept2, a.rr, a.thr, sd, handled,
                                           clear_new);
            }
        }
    }
    if (!handled) {
        bj = nn_search_slow(&a.g, a.tgt, a.cs, px, py, pz, a.r1, a.r1_accept2, a.rr, a.thr, jp);
        clear_new = 0.f;
    }
    if ((int)bj != jp) *a.src.seed(i) = (int)bj;
    if (__float_as_uint(clear_new) != __float_as_uint(clear_prev)) *a.src.clearance(i) = clear_new;
    int widx = -1;
    if (bj != kNoPoint) {
        const float4 t = (int)bj == jp ? ts : __ldg(&a.tgt[bj]);   // (just scanned: an L1 hit)
        const float d = dist2_canonical(t, px, py, pz);   // the same arithmetic as inside the scan: same bits
        widx = __float_as_int(t.w);
        if (MODE == 0 && EST == kEstPoint) {
            // the pivot is subtracted in f32 first: the products stay at the cloud's extent, not its distance
            const float vs[3] = {px - a.pivot[0], py - a.pivot[1], pz - a.pivot[2]};
            const float vt[3] = {t.x - a.pivot[0], t.y - a.pivot[1], t.z - a.pivot[2]};
            accumulate_p2point<32>(acc, vs, vt);
        } else if (MODE == 0) {
            // the seed's normal / colour row were fetched ahead (the winner rarely changes once the clouds
            // are roughly aligned); they are only read now, so that they hold no registers during the search
            const float4 nn = (int)bj == jp ? *seed_nn : __ldg(&a.nrm[bj]);
            if (EST == kEstColored) {
                const float4 cg = (int)bj == jp ? *seed_cg : __ldg(&a.tcg[bj]);
                const float vs[3] = {px, py, pz}, vt[3] = {t.x, t.y, t.z}, nt[3] = {nn.x, nn.y, nn.z};
                const float dit[3] = {cg.x, cg.y, cg.z};
                accumulate_colored<L2LOSS, 32>(acc, a.rk, vs, vt, nt, __ldg(&a.sint[i]), cg.w, dit, a.sqrt_lg, a.sqrt_lp);
            } else {
                accumulate_p2plane<L2LOSS, 32>(acc, a.rk, px, py, pz, t.x, t.y, t.z, nn.x, nn.y, nn.z);
            }
        } else {
            acc[28] += 1.0f;
        }
        acc[29] += d;
    }
    if (MODE == 1 && a.corr_out) a.corr_out[a.src_idx[i]] = (int64_t)widx;
    return bj != kNoPoint;
}

// One chunk's contribution to the 30 sums: transposed warp reduction of the lanes' terms (f32 tree over 32
// queries), added to the warp's running totals — one f64 per lane, lane l = slot l.  Returns what lane l added:
// +0.0 when no lane matched, and adding +0.0 to acc64, which starts at +0.0 and so is never -0.0, leaves its bits
// as they are.  A replayed chunk may therefore add its cached line unconditionally.
__device__ __forceinline__ float icp_accumulate_chunk(float (&term)[32], bool matched, double& acc64) {
    float line = 0.f;
    if (__any_sync(0xffffffffu, matched)) {
        line = warp_transpose_sum32(term);
        acc64 += (double)line;
    }
    return line;
}

// The exchange step of the source-sharded loop (SURVEY.md 8e), done INSIDE the iteration kernel over NVLink /
// NVSwitch peer memory instead of kernel -> ncclAllReduce -> finalize kernel.  Flag-in-data protocol (what NCCL
// calls LL): warp 0 of each rank's last block stores its 30 local sums into slot [parity][rank] of EVERY rank's
// mailbox as 8-byte words (32 data bits : 32-bit sequence number) — an aligned 8-byte store arrives whole, so a
// reader that sees the sequence number in a word has its data bits too, and no fence / release round trip is
// needed: the exchange costs one NVLink one-way latency.  Each rank then waits until the `world` slots of its OWN
// mailbox carry the sequence number and adds them in rank order, so every rank computes bit-identical totals and
// the identical pose update, with no broadcast.  Two slot parities suffice: rank r reuses a slot two collectives
// later, which it can only reach after every peer has published the collective in between, i.e. after every peer
// has finished reading the older one.  All 32 lanes of the warp must call it.  Returns false on a timeout (a peer
// died): the caller flags a communication error instead of hanging the GPU.
__device__ __forceinline__ bool peer_all_reduce(const PeerView& pv, double* s_final) {
    const int lane = threadIdx.x & 31;
    unsigned long long seq = 0;
    if (lane == 0) seq = *pv.seq + 1;
    seq = __shfl_sync(0xffffffffu, seq, 0);
    const unsigned tag = (unsigned)seq;                       // (0 never appears: the mailboxes start zeroed)
    const size_t par = (size_t)(seq & 1ull) * pv.world;
    if (lane < kNumSums) {
        const unsigned long long bits = (unsigned long long)__double_as_longlong(s_final[lane]);
        const unsigned long long w0 = ((unsigned long long)tag << 32) | (bits & 0xffffffffull);
        const unsigned long long w1 = ((unsigned long long)tag << 32) | (bits >> 32);
        for (int p = 0; p < pv.world; ++p) {
            double* dst = pv.box[p] + (par + pv.rank) * kBoxDoubles + 2 * lane;
            asm volatile("st.volatile.global.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"(w0), "l"(w1) : "memory");
        }
    }
    double acc = 0.0;
    bool ok = true;
    const long long t0 = global_ns();
    // collect in batches of 8 ranks: all loads of a batch are in flight together (one memory round trip per batch when
    // the peers have already published, instead of one per rank), the sum stays in rank order
    constexpr int kBatch = 8;
    for (int r0 = 0; r0 < pv.world && ok; r0 += kBatch) {
        unsigned long long w0[kBatch], w1[kBatch];
        if (lane < kNumSums) {
            unsigned pending = 0;
#pragma unroll
            for (int u = 0; u < kBatch; ++u)
                if (r0 + u < pv.world) pending |= 1u << u;
            while (pending) {
#pragma unroll
                for (int u = 0; u < kBatch; ++u)
                    if (pending & (1u << u)) {
                        const double* src = pv.box[pv.rank] + (par + r0 + u) * kBoxDoubles + 2 * lane;
                        asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0[u]), "=l"(w1[u]) : "l"(src) : "memory");
                    }
#pragma unroll
                for (int u = 0; u < kBatch; ++u)
                    if ((pending & (1u << u)) && (unsigned)(w0[u] >> 32) == tag && (unsigned)(w1[u] >> 32) == tag) pending &= ~(1u << u);
                if (pending) {
                    if (global_ns() - t0 > 4000000000ll) {   // 4 s
                        ok = false;
                        break;
                    }
                }
            }
            if (ok) {
#pragma unroll
                for (int u = 0; u < kBatch; ++u)
                    if (r0 + u < pv.world) acc += __longlong_as_double((long long)((w1[u] << 32) | (w0[u] & 0xffffffffull)));
            }
        }
        ok = __all_sync(0xffffffffu, ok);
    }
    if (lane < kNumSums) s_final[lane] = acc;
    if (lane == 0) *pv.seq = seq;
    __syncwarp();
    return ok;
}

// Block epilogue of the iteration kernel: block partial -> (last block) grand total, solve, pose update,
// convergence test.
template <int MODE, bool POINT>
__device__ __forceinline__ void icp_block_epilogue(const IcpArgs& a, double (*s_warp)[kSumStride], double* s_final) {
    if (!block_reduce_to_global<kIcpThreads>(s_warp, a.partials, &a.st->ticket, s_final)) return;
    // Every other block has read sums_cached by now.  An iteration has just written or replayed the line of every
    // chunk against the coordinates it left; the evaluation pass moves the coordinates and writes no line.
    if (threadIdx.x == 0) a.st->sums_cached = MODE == 0;
    if (a.fuse_finalize) {
        if (threadIdx.x < 32) {
            if (a.use_peer && !peer_all_reduce(a.peer, s_final)) {
                if (threadIdx.x == 0) {        // a peer never answered: stop the loop, the host reports O3DB_ERR_COMM
                    a.st->status = 2;
                    a.st->done = 1;
                }
                return;
            }
            if (MODE == 0) icp_finalize_iteration<POINT>(a, s_final, &s_warp[0][0]);   // (s_warp is dead: reused as scratch)
            else if (threadIdx.x == 0) icp_finalize_evaluate(a, s_final);
        }
    } else if (threadIdx.x < kNumSums) {
        a.st->sums[threadIdx.x] = s_final[threadIdx.x];
    }
}

// ------------------------------------------------ iteration kernel: TMA + cp.async ring

// Per warp, a two-slot ring in shared memory holds what a 32-query chunk needs before its search can
// start, fetched while the PREVIOUS chunk is being searched:
//   A  the chunk's record of the working source (points, seeds, clearances): one TMA bulk copy
//      (cp.async.bulk, completion on the slot's mbarrier) of 640 B issued by lane 0 two chunks ahead;
//   B  the seeds' target points, normals (and colour rows; point-to-point: the points alone): one 16-byte cp.async gather per lane and
//      array, issued one chunk ahead as soon as A has landed (the gather address IS the seed).
// A query therefore starts with p, seed, seed point and seed normal already on chip, and its dependent
// chain shrinks from four global round trips (source -> seed point -> CSR offsets -> candidates) to two.
// There is no block-wide barrier in the loop: slots are private to a warp (lane 0 produces, __syncwarp
// hands a consumed slot back), accumulator flushes are warp-local.
template <int EST>
struct __align__(16) IcpStage {
    // A: one chunk record of the working source (SrcBlocked): 640 contiguous bytes, ONE bulk copy
    float px[32];      // working source points, one plane per coordinate
    float py[32];
    float pz[32];
    int jp[32];        // seeds
    float d2[32];      // clearances
    // B: gathered per lane from the seeds
    float4 ts[32];     // the seeds' target points
    float4 ns[EST == kEstPoint ? 1 : 32];     // their normals
    float4 cg[EST == kEstColored ? 32 : 1];   // their colour rows
};

__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* b) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                         smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(b))
                 : "memory");
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
// through L2 only: for data an earlier launch wrote, which no L1 may hold a stale copy of
__device__ __forceinline__ void cp_async16_cg(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

template <int EST>
struct IcpStagedSmem {   // dynamic shared memory of the iteration kernels
    IcpStage<EST> stage[kIcpThreads / 32][2];
};

// The body of every iteration kernel below: one source for the ring, the search, the replay and the epilogue.
template <bool L2LOSS, int MODE, int EST>
__device__ __forceinline__ void icp_iteration(const IcpArgs& a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    IcpStagedSmem<EST>& sm = *reinterpret_cast<IcpStagedSmem<EST>*>(smem_raw);
    __shared__ double s_warp[kIcpThreads / 32][kSumStride];
    __shared__ double s_final[kSumStride];
    __shared__ float s_U[16];
    __shared__ int s_done, s_reverse, s_cached;
    __shared__ __align__(8) unsigned long long s_mbar[kIcpThreads / 32][2];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int k = threadIdx.x; k < (kIcpThreads / 32) * kSumStride; k += kIcpThreads) (&s_warp[0][0])[k] = 0.0;
    if (threadIdx.x < 2 * (kIcpThreads / 32)) mbar_init(&s_mbar[0][0] + threadIdx.x, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    // Programmatic dependent launch: this grid may become resident while the previous iteration's last
    // block is still in its serial epilogue; nothing produced by that kernel is read before the wait.
    pdl_wait();
    pdl_launch_dependents();
    if (threadIdx.x == 0) {
        s_done = *(volatile int*)&a.st->done;
        s_reverse = a.st->executed & 1;
        s_cached = MODE == 0 && a.st->sums_cached;
    }
    if (threadIdx.x < 16) s_U[threadIdx.x] = a.st->Uf[threadIdx.x];
    __syncthreads();
    if (MODE == 0 && s_done) return;

    // The warp owns the chunks starting at first, first + stride, ... below n (the arrays are padded to a multiple
    // of 256 entries, so a chunk that starts below n can always be copied whole).  It visits them in ascending
    // order when an even number of iterations has run and in descending order otherwise, so the evaluation pass
    // sweeps opposite to the iteration before it.  An iteration touches about twice the L2 in records, seed rows
    // and stores; walking the same order every time puts the whole working set between two uses of a line, while
    // a reversed walk starts on what the previous launch touched last.  The order depends only on device state,
    // never on how the host batches launches, and the per-chunk work is the same either way: only the order of the
    // warp's f64 running sums changes.
    const int n = (int)a.n;
    const int stride = gridDim.x * kIcpThreads;
    const int first = blockIdx.x * kIcpThreads + w * 32;
    const int steps = first < n ? (n - 1 - first) / stride + 1 : 0;
    const int step = s_reverse ? -stride : stride;
    const int start = s_reverse ? first + (steps - 1) * stride : first;
    constexpr unsigned kBytesA = kSrcChunkBytes;
    static_assert(offsetof(IcpStage<EST>, py) == 128 && offsetof(IcpStage<EST>, pz) == 256 &&
                  offsetof(IcpStage<EST>, jp) == 384 && offsetof(IcpStage<EST>, d2) == 512 &&
                  offsetof(IcpStage<EST>, ts) == kBytesA, "stage A mirrors a chunk record");
    // chunk c (the warp's c-th step) covers working-source positions [start + c * step, ... + 32)
    auto issue_a = [&](int c) {                // lane 0: ONE TMA bulk copy of chunk c's record into slot c & 1
        if (lane == 0 && c < steps) {
            IcpStage<EST>& sl = sm.stage[w][c & 1];
            unsigned long long* mb = &s_mbar[w][c & 1];
            mbar_arrive_expect_tx(mb, kBytesA);
            bulk_g2s(sl.px, a.src.chunk(start + c * step), kBytesA, mb);
        }
    };
    // Sum replay (iterations only).  When the pending update leaves all of a chunk's points bit-for-bit where they
    // were, every input of the chunk's sums is what the previous iteration used: the points, hence their exact
    // nearest neighbours (every search path returns the exhaustive-search winner), hence the winners' rows and the
    // per-handle constants.  Its 32 sums are then the line the previous iteration stored in a.chunk_sums, bit for
    // bit, and adding that line to acc64 at the same place in the sweep gives the same totals.  Such a chunk fetches
    // its 128-byte line instead of the seed rows, and does no search, no Jacobian, no reduction and no store.  Its
    // seeds already hold the winners; only a clearance that a search would have re-established stays as it was,
    // which can send a later search down another (equally exact) path.
    bool replay_b = false;   // the decision of the last issue_b, warp-uniform
    auto issue_b = [&](int c) {                // every lane: gather its seed's rows of chunk c (needs A(c))
        if (c < steps) {
            IcpStage<EST>& sl = sm.stage[w][c & 1];
            mbar_wait(&s_mbar[w][c & 1], (unsigned)(c >> 1) & 1u);
            const int q0 = start + c * step;
            bool unchanged = true;   // (positions past n count as unchanged: the update moves padding points)
            if (MODE == 0 && s_cached && q0 + lane < n) {
                float x = sl.px[lane], y = sl.py[lane], z = sl.pz[lane];
                const float ox = x, oy = y, oz = z;
                apply_transform(s_U, x, y, z);   // the expression icp_process_query applies
                unchanged = __float_as_uint(x) == __float_as_uint(ox) && __float_as_uint(y) == __float_as_uint(oy) &&
                            __float_as_uint(z) == __float_as_uint(oz);
            }
            replay_b = MODE == 0 && s_cached && __all_sync(0xffffffffu, unchanged);
            if (replay_b) {
                if (lane < 8)
                    cp_async16_cg(&sl.ts[lane], reinterpret_cast<const float4*>(a.chunk_sums + q0) + lane);
            } else {
                const int jp = sl.jp[lane];
                if (jp >= 0) {
                    cp_async16(&sl.ts[lane], a.tgt + jp);
                    if (MODE == 0 && EST != kEstPoint) cp_async16(&sl.ns[lane], a.nrm + jp);
                    if (MODE == 0 && EST == kEstColored) cp_async16(&sl.cg[lane], a.tcg + jp);
                }
            }
        }
        cp_async_commit();
    };

    double acc64 = 0.0;      // lane l: running total of slot l over this warp's queries
    issue_a(0);
    issue_a(1);
    issue_b(0);
    for (int c = 0; c < steps; ++c) {
        const int q0 = start + c * step;
        IcpStage<EST>& sl = sm.stage[w][c & 1];
        const bool replay = replay_b;
        // A(c) has landed: every lane waited on its mbarrier in issue_b(c), one trip ago (or in the prologue)
        cp_async_wait_all();                                       // B(c), or the cached line of chunk c
        const float px = sl.px[lane], py = sl.py[lane], pz = sl.pz[lane];
        const int jp = sl.jp[lane];
        const float clear_prev = sl.d2[lane];
        __syncwarp();          // every lane has read its point / jp / d2 of slot c & 1: hand that part back to the producer
        issue_a(c + 2);
        issue_b(c + 1);
        // (ts / ns / cg of slot c & 1 are rewritten by issue_b(c + 2), i.e. in the NEXT trip: still valid below)
        if (replay) {
            acc64 += (double)reinterpret_cast<const float*>(sl.ts)[lane];
            continue;
        }
        const int i = q0 + lane;
        float term[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) term[k] = 0.f;
        bool matched = false;
        if (i < n)
            matched = icp_process_query<L2LOSS, MODE, EST>(a, s_U, i, px, py, pz, jp, clear_prev, &sl.ts[lane],
                                                           &sl.ns[EST == kEstPoint ? 0 : lane],
                                                           &sl.cg[EST == kEstColored ? lane : 0], term);
        const float line = icp_accumulate_chunk(term, matched, acc64);
        if (MODE == 0) a.chunk_sums[q0 + lane] = line;   // one coalesced 128-byte store
    }
    if (lane < kNumSums) s_warp[w][lane] = acc64;
    icp_block_epilogue<MODE, EST == kEstPoint>(a, s_warp, s_final);
}

template <bool L2LOSS, int MODE, bool COLORED = false>
__global__ void __launch_bounds__(kIcpThreads, 1)
icp_iteration_kernel(const __grid_constant__ IcpArgs a) {
    icp_iteration<L2LOSS, MODE, COLORED ? kEstColored : kEstPlane>(a);
}

// The point-to-point iteration (L2 only: TransformationEstimationPointToPoint has no robust kernel).  Its evaluation
// pass is icp_iteration_kernel<true, 1>: evaluation reads no normal and adds no estimator term.
__global__ void __launch_bounds__(kIcpThreads, 1)
icp_point_iteration_kernel(const __grid_constant__ IcpArgs a) {
    icp_iteration<true, 0, kEstPoint>(a);
}

// Multi-GPU: runs after the all-reduce of st->sums.
template <int MODE>
__global__ void icp_finalize_kernel(IcpArgs a) {   // <<<1, 32>>>
    __shared__ double s_scratch[64];
    if (MODE == 0) {
        if (a.st->done) return;
        if (a.point_to_point) icp_finalize_iteration<true>(a, a.st->sums, s_scratch);
        else icp_finalize_iteration<false>(a, a.st->sums, s_scratch);
    } else if (threadIdx.x == 0) {
        icp_finalize_evaluate(a, a.st->sums);
    }
}

// Gather the caller's source into the sorted working copy (clone + initial transform).
// (scatter_kernel<true> does the work; this is the reset path reusing key/rank.)

}  // namespace o3db

struct o3db_icp {
    o3db_nns nns;
    o3db_icp_options opt{};
    cudaStream_t stream = 0;         // creation stream: allocations are freed on it (o3db_icp_destroy)
    const float* src_user = nullptr;
    int64_t n = 0;
    int64_t n_pad = 0;               // n rounded up to whole 256-entry chunks (allocation size of src_blk / src_idx)
    double n_total = 0;
    double init_T[16];
    char* src_blk = nullptr;         // chunk-blocked working source: points, seeds, clearances (SrcBlocked)
    int* src_idx = nullptr;          // sorted source position -> original index
    float* chunk_sums = nullptr;     // n_pad floats: one 128-byte line of cached sums per 32-query chunk (IcpArgs)
    unsigned* src_key = nullptr;     // cell key of every source point (sort order)
    unsigned* src_rank = nullptr;
    unsigned* src_start = nullptr;   // CSR offsets of the source sort
    double* partials = nullptr;
    double* per_iter = nullptr;
    IcpState* st = nullptr;
    IcpState* h_st = nullptr;        // pinned
    o3db_comm* comm = nullptr;
    int grid_blocks = 0;
    int64_t src_keys = 0;            // size of the source sort key space
    int launched = 0;
    bool l2loss = true;
    // ColoredICP (TransformationEstimationForColoredICP); null / unused for point-to-plane
    bool colored = false;
    const float* src_colors_user = nullptr;
    float4* tcg4 = nullptr;          // sorted target: colour gradient xyz + intensity
    float* sint = nullptr;           // sorted source: intensity
    double lambda_geometric = 0.968;
    // TransformationEstimationPointToPoint: no target normals (nns.nrm4 stays null), no robust kernel
    bool point = false;
    float pivot[3] = {0.f, 0.f, 0.f};
};

namespace o3db {

typedef void (*IcpKernel)(IcpArgs);
// mode 0 = iterate (loss / colour of the handle), 1 = final evaluation (no Jacobian)
static IcpKernel icp_kernel_for(const o3db_icp* c, int mode) {
    if (mode == 1) return icp_iteration_kernel<true, 1, false>;
    if (c->point) return icp_point_iteration_kernel;
    if (c->colored) return c->l2loss ? icp_iteration_kernel<true, 0, true> : icp_iteration_kernel<false, 0, true>;
    return c->l2loss ? icp_iteration_kernel<true, 0, false> : icp_iteration_kernel<false, 0, false>;
}

// dynamic shared memory of the handle's iteration kernels (the stage ring)
static size_t icp_smem_bytes(const o3db_icp* c, int mode) {
    if (mode == 1) return sizeof(IcpStagedSmem<kEstPlane>);
    return c->colored ? sizeof(IcpStagedSmem<kEstColored>) : c->point ? sizeof(IcpStagedSmem<kEstPoint>) : sizeof(IcpStagedSmem<kEstPlane>);
}

// The kernel's griddepcontrol.wait orders it after the previous kernel on the stream; everything before that wait
// may overlap the predecessor's tail.
static cudaError_t launch_icp(const o3db_icp* c, int mode, cudaStream_t st, const IcpArgs& a) {
    return launch_pdl_ex(icp_kernel_for(c, mode), {(unsigned)c->grid_blocks, kIcpThreads, icp_smem_bytes(c, mode)}, st, a);
}
static IcpArgs make_args(o3db_icp* c) {
    IcpArgs a{};
    a.g = c->nns.g;
    a.tgt = c->nns.pts4;
    a.nrm = c->nns.nrm4;
    a.cs = c->nns.cell_start;
    a.src = SrcBlocked{c->src_blk};
    a.src_idx = c->src_idx;
    a.chunk_sums = c->chunk_sums;
    a.n = c->n;
    a.n_total = c->n_total;
    const float r = (float)c->opt.max_correspondence_distance;
    a.thr = r * r;                       // FixedRadiusSearchImpl.cuh:692: T(radius) * T(radius)
    a.rr = r * (1.0f + 1e-6f);
    // unseeded first pass: a box of at least half the radius (and at least one cell)
    a.r1 = fminf(fmaxf(c->nns.g.c, 0.5f * (1.0f + 1e-4f) * r), a.rr);
    a.r1_accept2 = (a.r1 * (1.0f - 1e-4f)) * (a.r1 * (1.0f - 1e-4f));
    a.rk.method = c->opt.kernel.method;
    a.rk.scale = (float)c->opt.kernel.scale;
    a.rk.shape = c->opt.kernel.shape;
    a.partials = c->partials;
    a.st = c->st;
    a.per_iter = c->per_iter;
    a.corr_out = nullptr;
    a.rel_fitness = c->opt.relative_fitness;
    a.rel_rmse = c->opt.relative_rmse;
    a.max_iteration = c->opt.max_iteration;
    const PeerView* pv = o3db_comm_peer_view(c->comm);
    a.use_peer = pv ? 1 : 0;
    if (pv) a.peer = *pv;
    a.fuse_finalize = (c->comm && !pv) ? 0 : 1;   // NCCL transport: all-reduce + finalize kernel follow the launch
    a.tcg = c->tcg4;
    a.sint = c->sint;
    a.sqrt_lg = (float)sqrt(c->lambda_geometric);          // RegistrationCUDA.cu:205-208
    a.sqrt_lp = (float)sqrt(1.0 - c->lambda_geometric);
    a.point_to_point = c->point ? 1 : 0;
    for (int k = 0; k < 3; ++k) a.pivot[k] = c->pivot[k];
    return a;
}

static int icp_init_state(o3db_icp* c, cudaStream_t st) {
    IcpState h{};   // (sums_cached = 0: o3db_icp_reset has just gathered the caller's source again, which may differ)
    for (int i = 0; i < 16; ++i) {
        h.T[i] = c->init_T[i];
        h.Uf[i] = (i % 5 == 0) ? 1.f : 0.f;   // the initial transform is applied by the gather
    }
    memcpy(c->h_st, &h, sizeof(h));
    O3DB_CUDA_CHECK(cudaMemcpyAsync(c->st, c->h_st, sizeof(IcpState), cudaMemcpyHostToDevice, st));
    src_blocked_init_kernel<<<(unsigned)ceil_div(c->n_pad, kThreads), kThreads, 0, st>>>(SrcBlocked{c->src_blk}, c->n, c->n_pad,
                                                                                         false);   // no seeds, no clearances
    O3DB_LAUNCH_CHECK();
    c->launched = 0;
    return O3DB_OK;
}

static int icp_gather_source(o3db_icp* c, cudaStream_t st) {
    Affine T0;
    for (int i = 0; i < 16; ++i) T0.m[i] = (float)c->init_T[i];   // Transform.cpp:29-31: T cast to the point dtype
    if (c->n == 0) return O3DB_OK;
    scatter_source_kernel<<<(unsigned)ceil_div(c->n, kThreads), kThreads, 0, st>>>(c->src_user, c->n, T0, c->src_start,
                                                                                  c->src_key, c->src_rank, SrcBlocked{c->src_blk},
                                                                                  c->src_idx);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

}  // namespace o3db

extern "C" {

int o3db_nns_create(const float* points_dev, int64_t num_points, double radius, void* stream, o3db_nns** out) {
    O3DB_REQUIRE(out != nullptr, "o3db_nns_create: out is null");
    *out = nullptr;
    O3DB_REQUIRE(points_dev != nullptr && num_points > 0, "o3db_nns_create: empty point set");
    O3DB_REQUIRE(num_points < INT_MAX, "o3db_nns_create: too many points");
    O3DB_REQUIRE(radius > 0 && std::isfinite(radius), "o3db_nns_create: radius must be positive");
    o3db_nns* s = new (std::nothrow) o3db_nns();
    O3DB_REQUIRE(s != nullptr, "out of host memory");
    const int rc = nns_build(s, points_dev, nullptr, num_points, radius, 1.0, (cudaStream_t)stream);
    if (rc != O3DB_OK) {
        nns_free(s, (cudaStream_t)stream);
        delete s;
        return rc;
    }
    *out = s;
    return O3DB_OK;
}

void o3db_nns_destroy(o3db_nns* nns) {
    if (!nns) return;
    cudaStreamSynchronize(nns->stream);   // searches may still be in flight on the creation stream
    nns_free(nns, nns->stream);
    delete nns;
}

int o3db_nns_hybrid_search(const o3db_nns* nns, const float* queries_dev, int64_t num_queries, double radius,
                           int max_knn, int32_t* indices_dev, float* distances_dev, int32_t* counts_dev,
                           void* stream) {
    O3DB_REQUIRE(nns != nullptr, "o3db_nns_hybrid_search: null index");
    O3DB_REQUIRE(max_knn >= 1 && max_knn <= kMaxKnn, "o3db_nns_hybrid_search: max_knn must be in 1..%d", kMaxKnn);
    O3DB_REQUIRE(radius > 0 && radius <= nns->radius * (1 + 1e-12),
                 "o3db_nns_hybrid_search: radius %g exceeds the index radius %g", radius, nns->radius);
    if (num_queries == 0) return O3DB_OK;
    O3DB_REQUIRE(queries_dev != nullptr && num_queries > 0, "o3db_nns_hybrid_search: bad queries");
    const float r = (float)radius;
    const float thr = r * r, rr = r * (1.0f + 1e-6f);
    const unsigned nb = (unsigned)ceil_div(num_queries, kThreads);
    cudaStream_t st = (cudaStream_t)stream;
    if (max_knn == 1)
        hybrid_search_k1_kernel<true><<<nb, kThreads, 0, st>>>(nns->g, nns->pts4, nns->cell_start, queries_dev,
                                                               num_queries, rr, thr, indices_dev, distances_dev,
                                                               counts_dev);
    else
        hybrid_search_knn_kernel<<<nb, kThreads, 0, st>>>(nns->g, nns->pts4, nns->cell_start, queries_dev,
                                                          num_queries, rr, thr, max_knn, indices_dev,
                                                          distances_dev, counts_dev);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

int o3db_build_spatial_hash_table(const float* points_dev, int64_t num_points, double radius,
                                  uint32_t hash_table_size, uint32_t* hash_table_index_dev,
                                  uint32_t* hash_table_cell_splits_dev, void* stream) {
    O3DB_REQUIRE(points_dev && hash_table_index_dev && hash_table_cell_splits_dev && num_points > 0 &&
                         num_points < INT_MAX && hash_table_size > 0 && radius > 0,
                 "o3db_build_spatial_hash_table: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    const float voxel = 2 * (float)radius;          // FixedRadiusSearchImpl.cuh:760-761 (T arithmetic)
    const float inv_voxel = 1 / voxel;
    unsigned *rank = nullptr, *scratch = nullptr;
    O3DB_CUDA_CHECK(cudaMallocAsync(&rank, num_points * sizeof(unsigned), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&scratch, ceil_div(hash_table_size, kScanTile) * sizeof(unsigned), st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(hash_table_cell_splits_dev, 0, ((size_t)hash_table_size + 1) * sizeof(unsigned), st));
    const unsigned nb = (unsigned)ceil_div(num_points, kThreads);
    ref_count_kernel<<<nb, kThreads, 0, st>>>(points_dev, num_points, inv_voxel, hash_table_size,
                                              hash_table_cell_splits_dev, rank);
    O3DB_LAUNCH_CHECK();
    int rc = exclusive_scan_u32(hash_table_cell_splits_dev, hash_table_size, scratch, st);
    if (rc) return rc;
    ref_scatter_kernel<<<nb, kThreads, 0, st>>>(points_dev, num_points, inv_voxel, hash_table_size,
                                                hash_table_cell_splits_dev, rank, hash_table_index_dev);
    O3DB_LAUNCH_CHECK();
    O3DB_CUDA_CHECK(cudaFreeAsync(rank, st));
    O3DB_CUDA_CHECK(cudaFreeAsync(scratch, st));
    return O3DB_OK;
}

void o3db_pose_to_transformation(const double pose_host[6], double transformation_host[16]) {
    pose_to_T(pose_host, transformation_host);
}

int o3db_transform_points(const double T[16], float* points_dev, int64_t n, void* stream) {
    O3DB_REQUIRE(T != nullptr && (points_dev != nullptr || n == 0) && n >= 0, "o3db_transform_points: bad arguments");
    if (n == 0) return O3DB_OK;
    Affine A;
    for (int i = 0; i < 16; ++i) A.m[i] = (float)T[i];
    transform_points_kernel<<<(unsigned)ceil_div(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(points_dev, n, A);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

int o3db_transform_normals(const double T[16], float* normals_dev, int64_t n, void* stream) {
    O3DB_REQUIRE(T != nullptr && (normals_dev != nullptr || n == 0) && n >= 0, "o3db_transform_normals: bad arguments");
    if (n == 0) return O3DB_OK;
    Affine A;
    for (int i = 0; i < 16; ++i) A.m[i] = (float)T[i];
    transform_normals_kernel<<<(unsigned)ceil_div(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(normals_dev, n, A);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

}  // extern "C"

namespace o3db {

struct PoseScratch {
    double* partials = nullptr;
    unsigned* ticket = nullptr;
    int* status = nullptr;
    double* sums = nullptr;
    int blocks = 0;
};

static int pose_scratch_alloc(PoseScratch* s, int64_t n, cudaStream_t st) {
    s->blocks = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, kThreads), (int64_t)num_sms() * 4));
    char* base = nullptr;
    const size_t bytes = (size_t)s->blocks * kSumStride * sizeof(double) + kSumStride * sizeof(double) + 64;
    O3DB_CUDA_CHECK(cudaMallocAsync(&base, bytes, st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(base, 0, bytes, st));
    s->partials = (double*)base;
    s->sums = s->partials + (size_t)s->blocks * kSumStride;
    s->ticket = (unsigned*)(s->sums + kSumStride);
    s->status = (int*)(s->ticket + 4);
    return O3DB_OK;
}

static int pose_finish(PoseScratch* s, double* sums29_dev, float* residual_host, int* inlier_count_host,
                       cudaStream_t st) {
    int rc = O3DB_OK;
    if (sums29_dev)
        O3DB_CUDA_CHECK(cudaMemcpyAsync(sums29_dev, s->sums, 29 * sizeof(double), cudaMemcpyDeviceToDevice, st));
    if (residual_host || inlier_count_host) {
        double h[kSumStride];
        int status = 0;
        O3DB_CUDA_CHECK(cudaMemcpyAsync(h, s->sums, sizeof(h), cudaMemcpyDeviceToHost, st));
        O3DB_CUDA_CHECK(cudaMemcpyAsync(&status, s->status, sizeof(int), cudaMemcpyDeviceToHost, st));
        O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
        if (status) {  // TransformationConverter.cpp:219-225
            set_last_error("Singular 6x6 linear system detected, tracking failed.");
            if (residual_host) *residual_host = 0;
            if (inlier_count_host) *inlier_count_host = 0;
            rc = O3DB_ERR_SINGULAR;
        } else {
            if (residual_host) *residual_host = (float)h[27];
            if (inlier_count_host) *inlier_count_host = (int)h[28];
        }
    }
    O3DB_CUDA_CHECK(cudaFreeAsync(s->partials, st));
    return rc;
}

// The pose entry points' launch: `l2` for the L2 loss, `robust` for every other kernel, both taking `args` followed by
// the robust kernel, the scratch and the outputs.
template <typename Kernel, typename... Args>
static int pose_run(Kernel l2, Kernel robust, const o3db_robust_kernel* kernel, int64_t n, double* sums29_dev,
                    double* pose_dev, float* residual_host, int* inlier_count_host, cudaStream_t st, Args... args) {
    PoseScratch s;
    int rc = pose_scratch_alloc(&s, n, st);
    if (rc) return rc;
    const Robust rk{kernel ? kernel->method : 0, kernel ? (float)kernel->scale : 1.f, kernel ? kernel->shape : 1.0};
    (rk.method == O3DB_ROBUST_L2 ? l2 : robust)<<<s.blocks, kThreads, 0, st>>>(args..., rk, s.partials, s.ticket,
                                                                                PoseOut{s.sums, pose_dev, s.status});
    O3DB_LAUNCH_CHECK();
    return pose_finish(&s, sums29_dev, residual_host, inlier_count_host, st);
}

// information_matrix_kernel over n correspondences, given as corr_i32 or as corr_i64; its sums are read back into h.
static int information_sums(const float* tgt, const int32_t* corr_i32, const int64_t* corr_i64, int64_t n,
                            double (&h)[kSumStride], cudaStream_t st) {
    PoseScratch s;
    int rc = pose_scratch_alloc(&s, n, st);
    if (rc) return rc;
    information_matrix_kernel<<<s.blocks, kThreads, 0, st>>>(tgt, corr_i32, corr_i64, n, s.partials, s.ticket, s.sums);
    O3DB_LAUNCH_CHECK();
    O3DB_CUDA_CHECK(cudaMemcpyAsync(h, s.sums, sizeof(h), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    O3DB_CUDA_CHECK(cudaFreeAsync(s.partials, st));
    return O3DB_OK;
}

// The 21 lower-triangle sums -> the symmetric 6x6 information matrix (RegistrationCUDA.cu:565-571).
static void unpack_information(const double* h, double information[36]) {
    int q = 0;
    for (int j = 0; j < 6; ++j)
        for (int k = 0; k <= j; ++k) information[j * 6 + k] = information[k * 6 + j] = h[q++];
}

}  // namespace o3db

extern "C" {

int o3db_compute_pose_point_to_plane(const float* source_dev, const float* target_dev,
                                     const float* target_normals_dev, const int64_t* correspondences_dev,
                                     int64_t n, const o3db_robust_kernel* kernel, double* sums29_dev,
                                     double* pose_dev, float* residual_host, int* inlier_count_host,
                                     void* stream) {
    O3DB_REQUIRE(n >= 0 && (n == 0 || (source_dev && target_dev && target_normals_dev && correspondences_dev)),
                 "o3db_compute_pose_point_to_plane: bad arguments");
    return pose_run(pose_p2plane_kernel<true>, pose_p2plane_kernel<false>, kernel, n, sums29_dev, pose_dev,
                    residual_host, inlier_count_host, (cudaStream_t)stream, source_dev, target_dev, target_normals_dev,
                    correspondences_dev, n);
}

int o3db_compute_pose_colored_icp(const float* source_dev, const float* source_colors_dev, const float* target_dev,
                                  const float* target_normals_dev, const float* target_colors_dev,
                                  const float* target_color_gradients_dev, const int64_t* correspondences_dev,
                                  int64_t n, const o3db_robust_kernel* kernel, double lambda_geometric,
                                  double* sums29_dev, double* pose_dev, float* residual_host,
                                  int* inlier_count_host, void* stream) {
    O3DB_REQUIRE(n >= 0 && (n == 0 || (source_dev && source_colors_dev && target_dev && target_normals_dev &&
                                       target_colors_dev && target_color_gradients_dev && correspondences_dev)),
                 "o3db_compute_pose_colored_icp: bad arguments");
    const float sl = (float)sqrt(lambda_geometric), sp = (float)sqrt(1.0 - lambda_geometric);  // RegistrationCUDA.cu:205-208
    return pose_run(pose_colored_kernel<true>, pose_colored_kernel<false>, kernel, n, sums29_dev, pose_dev,
                    residual_host, inlier_count_host, (cudaStream_t)stream, source_dev, source_colors_dev, target_dev,
                    target_normals_dev, target_colors_dev, target_color_gradients_dev, correspondences_dev, n, sl, sp);
}

int o3db_compute_rt_point_to_point(const float* source_dev, const float* target_dev, const int64_t* correspondences_dev,
                                   int64_t n, double R_host[9], double t_host[3], int* inlier_count_host, void* stream) {
    O3DB_REQUIRE(source_dev && target_dev && correspondences_dev && R_host && t_host && n > 0,
                 "o3db_compute_rt_point_to_point: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    PoseScratch s;
    int rc = pose_scratch_alloc(&s, n, st);
    if (rc) return rc;
    rt_p2point_kernel<<<s.blocks, kThreads, 0, st>>>(source_dev, target_dev, correspondences_dev, n, s.partials, s.ticket,
                                                     s.sums);
    O3DB_LAUNCH_CHECK();
    double h[kSumStride];
    O3DB_CUDA_CHECK(cudaMemcpyAsync(h, s.sums, sizeof(h), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    O3DB_CUDA_CHECK(cudaFreeAsync(s.partials, st));
    if (inlier_count_host) *inlier_count_host = (int)h[16];
    if (h[16] == 0) {   // RegistrationCPU.cpp:547-549
        set_last_error("No valid correspondence present.");
        return O3DB_ERR_INVALID;
    }
    for (int j = 0; j < 3; ++j) {
        for (int k = 0; k < 3; ++k) R_host[3 * j + k] = h[4 * j + k];
        t_host[j] = h[4 * j + 3];
    }
    return O3DB_OK;
}

int o3db_compute_information_matrix(const float* target_dev, const int64_t* correspondences_dev, int64_t n,
                                    double information_host[36], int64_t* num_correspondences_host, void* stream) {
    O3DB_REQUIRE(target_dev && correspondences_dev && information_host && n > 0, "o3db_compute_information_matrix: bad arguments");
    double h[kSumStride];
    const int rc = information_sums(target_dev, nullptr, correspondences_dev, n, h, (cudaStream_t)stream);
    if (rc) return rc;
    unpack_information(h, information_host);
    if (num_correspondences_host) *num_correspondences_host = (int64_t)h[28];
    return O3DB_OK;
}

int o3db_get_information_matrix(const float* source_dev, int64_t n, const float* target_dev, int64_t m,
                                double max_correspondence_distance, const double transformation_host[16],
                                double information_host[36], void* stream) {
    O3DB_REQUIRE(source_dev && target_dev && n > 0 && m > 0, "Source and/or Target pointcloud is empty.");   // Registration.cpp:450-452
    O3DB_REQUIRE(transformation_host && information_host && max_correspondence_distance > 0,
                 "o3db_get_information_matrix: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    // :460-472: transform a clone of the source, hybrid search (k = 1) on the target
    float* moved = nullptr;
    int32_t* idx = nullptr;
    O3DB_CUDA_CHECK(cudaMallocAsync(&moved, (size_t)n * 3 * sizeof(float), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&idx, (size_t)n * sizeof(int32_t), st));
    O3DB_CUDA_CHECK(cudaMemcpyAsync(moved, source_dev, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    o3db_nns* index = nullptr;
    int rc = o3db_transform_points(transformation_host, moved, n, stream);
    if (rc == O3DB_OK) rc = o3db_nns_create(target_dev, m, max_correspondence_distance, stream, &index);
    if (rc == O3DB_OK) rc = o3db_nns_hybrid_search(index, moved, n, max_correspondence_distance, 1, idx, nullptr, nullptr, stream);
    double h[kSumStride] = {0};
    if (rc == O3DB_OK)
        rc = information_sums(target_dev, idx, nullptr, n, h, st);
    else
        cudaStreamSynchronize(st);
    cudaFreeAsync(moved, st);
    cudaFreeAsync(idx, st);
    if (index) o3db_nns_destroy(index);
    if (rc) return rc;
    if ((int64_t)h[28] == 0) {   // :476-480
        set_last_error("0 correspondence present between the pointclouds. Try increasing the max_correspondence_distance parameter.");
        return O3DB_ERR_INVALID;
    }
    unpack_information(h, information_host);
    return O3DB_OK;
}

// ------------------------------------------------------------- fused ICP API

void o3db_icp_destroy(o3db_icp* c) {
    if (!c) return;
    // Every buffer was allocated, and all work on it enqueued, on the handle's stream: drain it, then
    // free in stream order on the same stream (the pinned block may still be the target of a D2H copy).
    cudaStream_t st = c->stream;
    cudaStreamSynchronize(st);
    nns_free(&c->nns, st);
    if (c->src_blk) cudaFreeAsync(c->src_blk, st);
    if (c->src_idx) cudaFreeAsync(c->src_idx, st);
    if (c->chunk_sums) cudaFreeAsync(c->chunk_sums, st);
    if (c->src_key) cudaFreeAsync(c->src_key, st);
    if (c->src_rank) cudaFreeAsync(c->src_rank, st);
    if (c->src_start) cudaFreeAsync(c->src_start, st);
    if (c->partials) cudaFreeAsync(c->partials, st);
    if (c->per_iter) cudaFreeAsync(c->per_iter, st);
    if (c->st) cudaFreeAsync(c->st, st);
    if (c->tcg4) cudaFreeAsync(c->tcg4, st);
    if (c->sint) cudaFreeAsync(c->sint, st);
    if (c->h_st) pinned_release(c->h_st);
    delete c;
}

}  // extern "C"

namespace o3db {
struct EstimatorInputs {   // all device pointers; null source_colors and no point_to_point = plain point-to-plane
    bool point_to_point = false;   // no target normals wanted
    const float* source_colors = nullptr;
    const float* target_colors = nullptr;
    const float* target_color_gradients = nullptr;
    double lambda_geometric = 0.968;
};
}  // namespace o3db

static int icp_create_impl(const float* source_dev, int64_t n, const float* target_dev, const float* target_normals_dev,
                           int64_t m, const double init_T[16], const o3db_icp_options* options, o3db_comm* comm,
                           const o3db::EstimatorInputs& col, void* stream, o3db_icp** out,
                           cudaEvent_t source_ready = nullptr) {
    O3DB_REQUIRE(out != nullptr, "o3db_icp_create: out is null");
    *out = nullptr;
    O3DB_REQUIRE(options != nullptr && init_T != nullptr, "o3db_icp_create: null options / init");
    // Registration.cpp:119-219 AssertInputMultiScaleICP
    O3DB_REQUIRE(source_dev && target_dev && n > 0 && m > 0, "Source and/or Target pointcloud is empty.");
    O3DB_REQUIRE(col.point_to_point || target_normals_dev != nullptr, "Target pointcloud missing normals attribute.");
    O3DB_REQUIRE(n < INT_MAX - 2048 && m < INT_MAX - 2048, "o3db_icp_create: too many points");
    O3DB_REQUIRE(options->max_correspondence_distance > 0, "max_correspondence_distance must be positive");
    O3DB_REQUIRE(options->max_iteration >= 0, "max_iteration must be non-negative");
    cudaStream_t st = (cudaStream_t)stream;
    o3db_icp* c = new (std::nothrow) o3db_icp();
    O3DB_REQUIRE(c != nullptr, "out of host memory");
    c->opt = *options;
    c->stream = st;
    c->src_user = source_dev;
    c->n = n;
    c->comm = comm;
    c->point = col.point_to_point;
    c->l2loss = c->point || options->kernel.method == O3DB_ROBUST_L2;
    c->colored = col.source_colors != nullptr;
    c->src_colors_user = col.source_colors;
    c->lambda_geometric = col.lambda_geometric;
    memcpy(c->init_T, init_T, sizeof(c->init_T));
    // fine cells (half the radius) by default: pass 1 of the two-pass search then covers the
    // +-1 cell box, which holds the nearest neighbour of every already roughly aligned point
    int rc = nns_build(&c->nns, target_dev, c->point ? nullptr : target_normals_dev, m, options->max_correspondence_distance,
                       options->cell_scale > 0 ? options->cell_scale : kDefaultCellScale, st);
    if (rc) {
        o3db_icp_destroy(c);
        return rc;
    }
#define ICP_TRY(expr)                         \
    do {                                      \
        int rc__ = (expr);                    \
        if (rc__ != O3DB_OK) {                \
            o3db_icp_destroy(c);              \
            return rc__;                      \
        }                                     \
    } while (0)
#define ICP_CUDA(expr)                                                                           \
    do {                                                                                         \
        cudaError_t e__ = (expr);                                                                \
        if (e__ != cudaSuccess) {                                                                \
            set_last_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
            o3db_icp_destroy(c);                                                                 \
            return O3DB_ERR_CUDA;                                                                \
        }                                                                                        \
    } while (0)
    for (int k = 0; k < 3; ++k)   // (Grid::bmin / bmax are in grid-axis order: grid axis k is world axis ax[k])
        c->pivot[c->nns.g.ax[k]] = 0.5f * c->nns.g.bmin[k] + 0.5f * c->nns.g.bmax[k];
    // fitness denominator over all ranks
    c->n_total = (double)n;
    int occ = 1;
    for (int mode = 0; mode < 2; ++mode)
        ICP_CUDA(cudaFuncSetAttribute(icp_kernel_for(c, mode), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)icp_smem_bytes(c, mode)));
    ICP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, icp_kernel_for(c, 0), kIcpThreads, icp_smem_bytes(c, 0)));
    c->grid_blocks = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, kIcpThreads), (int64_t)num_sms() * std::max(occ, 1)));
    const int64_t ncell = tiled_key_space(c->nns.g.nx, c->nns.g.ny, c->nns.g.nz);   // tile-major source keys
    c->src_keys = ncell;
    // padded to whole 256-entry chunks: the staged kernel copies 32-entry chunks with TMA bulk copies
    c->n_pad = ceil_div(n, 256) * 256;
    ICP_CUDA(cudaMallocAsync(&c->src_blk, SrcBlocked::bytes(c->n_pad), st));
    ICP_CUDA(cudaMallocAsync(&c->src_idx, c->n_pad * sizeof(int), st));
    // (no initial contents: IcpState::sums_cached starts at 0, so the first iteration writes every line)
    ICP_CUDA(cudaMallocAsync(&c->chunk_sums, c->n_pad * sizeof(float), st));
    src_blocked_init_kernel<<<(unsigned)ceil_div(c->n_pad, kThreads), kThreads, 0, st>>>(SrcBlocked{c->src_blk}, n, c->n_pad, true);
    count_launch();
    ICP_CUDA(cudaGetLastError());
    ICP_CUDA(cudaMallocAsync(&c->src_key, n * sizeof(unsigned), st));
    ICP_CUDA(cudaMallocAsync(&c->src_rank, n * sizeof(unsigned), st));
    ICP_CUDA(cudaMallocAsync(&c->src_start, (ncell + 1) * sizeof(unsigned), st));
    ICP_CUDA(cudaMallocAsync(&c->partials, (size_t)c->grid_blocks * kSumStride * sizeof(double), st));
    ICP_CUDA(cudaMallocAsync(&c->per_iter, (size_t)std::max(1, options->max_iteration) * 2 * sizeof(double), st));
    ICP_CUDA(cudaMallocAsync(&c->st, sizeof(IcpState), st));
    static_assert(sizeof(IcpState) <= 4096, "IcpState must fit a pinned block");
    c->h_st = (IcpState*)pinned_acquire(sizeof(IcpState));
    if (!c->h_st) {
        set_last_error("pinned host allocation failed");
        o3db_icp_destroy(c);
        return O3DB_ERR_CUDA;
    }
    ICP_CUDA(cudaMemsetAsync(c->partials, 0, (size_t)c->grid_blocks * kSumStride * sizeof(double), st));
    ICP_CUDA(cudaMemsetAsync(c->per_iter, 0, (size_t)std::max(1, options->max_iteration) * 2 * sizeof(double), st));
    // sort order of the source: target-grid cell of the initially transformed point
    unsigned* scratch = nullptr;
    ICP_CUDA(cudaMallocAsync(&scratch, ceil_div(ncell, kScanTile) * sizeof(unsigned), st));
    ICP_CUDA(cudaMemsetAsync(c->src_start, 0, (ncell + 1) * sizeof(unsigned), st));
    Affine T0;
    for (int i = 0; i < 16; ++i) T0.m[i] = (float)init_T[i];
    // (host-buffer entry point: the source is still arriving on a copy stream while the target index is built)
    if (source_ready) ICP_CUDA(cudaStreamWaitEvent(st, source_ready, 0));
    count_kernel<true><<<(unsigned)ceil_div(n, kThreads), kThreads, 0, st>>>(source_dev, n, c->nns.g, T0, c->src_start,
                                                                            c->src_key, c->src_rank);
    count_launch();
    ICP_CUDA(cudaGetLastError());
    ICP_TRY(exclusive_scan_u32(c->src_start, ncell, scratch, st));
    ICP_CUDA(cudaFreeAsync(scratch, st));
    ICP_TRY(canonical_ranks(n, c->src_start, c->src_key, c->src_rank, st));
    ICP_TRY(icp_gather_source(c, st));
    if (c->colored) {
        ICP_CUDA(cudaMallocAsync(&c->tcg4, m * sizeof(float4), st));
        ICP_CUDA(cudaMallocAsync(&c->sint, n * sizeof(float), st));
        pack_target_color_kernel<<<(unsigned)ceil_div(m, kThreads), kThreads, 0, st>>>(
                c->nns.pts4, col.target_colors, col.target_color_gradients, m, c->tcg4);
        count_launch();
        ICP_CUDA(cudaGetLastError());
        // the source sort order is fixed at creation (o3db_icp_reset re-gathers into the same slots)
        pack_source_intensity_kernel<<<(unsigned)ceil_div(n, kThreads), kThreads, 0, st>>>(c->src_idx, col.source_colors, n,
                                                                                          c->sint);
        count_launch();
        ICP_CUDA(cudaGetLastError());
    }
    ICP_TRY(icp_init_state(c, st));
    if (comm) {
        double* d = nullptr;
        ICP_CUDA(cudaMallocAsync(&d, sizeof(double), st));
        ICP_CUDA(cudaMemcpyAsync(d, &c->n_total, sizeof(double), cudaMemcpyHostToDevice, st));
        ICP_TRY(o3db_comm_allreduce_f64(comm, d, 1, st));
        ICP_CUDA(cudaMemcpyAsync(&c->n_total, d, sizeof(double), cudaMemcpyDeviceToHost, st));
        ICP_CUDA(cudaStreamSynchronize(st));
        ICP_CUDA(cudaFreeAsync(d, st));
    }
    *out = c;
    return O3DB_OK;
}

extern "C" {

int o3db_icp_create(const float* source_dev, int64_t n, const float* target_dev, const float* target_normals_dev,
                    int64_t m, const double init_T[16], const o3db_icp_options* options, o3db_comm* comm,
                    void* stream, o3db_icp** out) {
    return icp_create_impl(source_dev, n, target_dev, target_normals_dev, m, init_T, options, comm,
                           o3db::EstimatorInputs{}, stream, out);
}

int o3db_icp_create_colored(const float* source_dev, const float* source_colors_dev, int64_t n,
                            const float* target_dev, const float* target_normals_dev, const float* target_colors_dev,
                            const float* target_color_gradients_dev, int64_t m, const double init_T[16],
                            const o3db_icp_options* options, double lambda_geometric, o3db_comm* comm, void* stream,
                            o3db_icp** out) {
    O3DB_REQUIRE(out != nullptr, "o3db_icp_create_colored: out is null");
    *out = nullptr;
    // ColoredICP.. TransformationEstimationForColoredICP::ComputeTransformation (TransformationEstimation.cpp:226-262)
    O3DB_REQUIRE(source_colors_dev != nullptr, "Source pointcloud missing colors attribute.");
    O3DB_REQUIRE(target_colors_dev != nullptr, "Target pointcloud missing colors attribute.");
    O3DB_REQUIRE(target_color_gradients_dev != nullptr,
                 "Target pointcloud missing color_gradients attribute (o3db_estimate_color_gradients).");
    O3DB_REQUIRE(lambda_geometric >= 0.0 && lambda_geometric <= 1.0, "lambda_geometric must be in [0, 1]");
    o3db::EstimatorInputs col;
    col.source_colors = source_colors_dev;
    col.target_colors = target_colors_dev;
    col.target_color_gradients = target_color_gradients_dev;
    col.lambda_geometric = lambda_geometric;
    return icp_create_impl(source_dev, n, target_dev, target_normals_dev, m, init_T, options, comm, col, stream, out);
}

int o3db_icp_create_point_to_point(const float* source_dev, int64_t n, const float* target_dev, int64_t m,
                                   const double init_T[16], const o3db_icp_options* options, o3db_comm* comm, void* stream,
                                   o3db_icp** out) {
    o3db::EstimatorInputs est;
    est.point_to_point = true;
    return icp_create_impl(source_dev, n, target_dev, nullptr, m, init_T, options, comm, est, stream, out);
}

int o3db_icp_reset(o3db_icp* c, void* stream) {
    O3DB_REQUIRE(c != nullptr, "o3db_icp_reset: null handle");
    cudaStream_t st = (cudaStream_t)stream;
    int rc = icp_gather_source(c, st);
    if (rc) return rc;
    return icp_init_state(c, st);
}

int o3db_icp_iterate(o3db_icp* c, int iterations, void* stream) {
    O3DB_REQUIRE(c != nullptr, "o3db_icp_iterate: null handle");
    cudaStream_t st = (cudaStream_t)stream;
    const int todo = std::min(iterations, c->opt.max_iteration - c->launched);
    IcpArgs a = make_args(c);
    for (int k = 0; k < todo; ++k) {
        launch_icp(c, 0, st, a);
        O3DB_LAUNCH_CHECK();
        if (!a.fuse_finalize) {
            int rc = o3db_comm_allreduce_f64(c->comm, (double*)((char*)c->st + offsetof(IcpState, sums)), kNumSums, st);
            if (rc) return rc;
            icp_finalize_kernel<0><<<1, 32, 0, st>>>(a);
            O3DB_LAUNCH_CHECK();
        }
        c->launched += 1;
    }
    return O3DB_OK;
}

static int icp_read_state(o3db_icp* c, o3db_icp_result* result, double* per_iteration_host, cudaStream_t st) {
    O3DB_CUDA_CHECK(cudaMemcpyAsync(c->h_st, c->st, sizeof(IcpState), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    const IcpState& h = *c->h_st;
    memcpy(result->transformation, h.T, sizeof(h.T));
    result->fitness = h.fitness;
    result->inlier_rmse = h.rmse;
    result->converged = h.converged;
    result->num_iterations = h.iter;
    result->num_correspondences = (int64_t)h.count;
    if (h.status == 2) {
        set_last_error("multi-GPU exchange timed out: a peer rank did not publish its sums (in-kernel NVLink exchange)");
        return O3DB_ERR_COMM;
    }
    result->status = h.status ? O3DB_ERR_SINGULAR : O3DB_OK;
    if (per_iteration_host && h.executed > 0) {
        O3DB_CUDA_CHECK(cudaMemcpyAsync(per_iteration_host, c->per_iter, (size_t)h.executed * 2 * sizeof(double),
                                        cudaMemcpyDeviceToHost, st));
        O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    }
    if (h.status) {
        set_last_error("Singular 6x6 linear system detected, tracking failed.");
        return O3DB_ERR_SINGULAR;
    }
    return O3DB_OK;
}


int o3db_icp_finish(o3db_icp* c, o3db_icp_result* result, int64_t* correspondences_dev, double* per_iteration_host,
                    void* stream) {
    O3DB_REQUIRE(c != nullptr && result != nullptr, "o3db_icp_finish: null argument");
    cudaStream_t st = (cudaStream_t)stream;
    IcpArgs a = make_args(c);
    a.corr_out = correspondences_dev;
    launch_icp(c, 1, st, a);
    O3DB_LAUNCH_CHECK();
    if (!a.fuse_finalize) {
        int rc = o3db_comm_allreduce_f64(c->comm, (double*)((char*)c->st + offsetof(IcpState, sums)), kNumSums, st);
        if (rc) return rc;
        icp_finalize_kernel<1><<<1, 32, 0, st>>>(a);
        O3DB_LAUNCH_CHECK();
    }
    return icp_read_state(c, result, per_iteration_host, st);
}

int o3db_icp_state(o3db_icp* c, o3db_icp_result* result, double* per_iteration_host, void* stream) {
    O3DB_REQUIRE(c != nullptr && result != nullptr, "o3db_icp_state: null argument");
    return icp_read_state(c, result, per_iteration_host, (cudaStream_t)stream);
}

int o3db_icp_point_to_plane(const float* source_dev, int64_t n, const float* target_dev,
                            const float* target_normals_dev, int64_t m, const double init_T[16],
                            const o3db_icp_options* options, o3db_icp_result* result, int64_t* correspondences_dev,
                            double* per_iteration_host, void* stream) {
    o3db_icp* c = nullptr;
    int rc = o3db_icp_create(source_dev, n, target_dev, target_normals_dev, m, init_T, options, nullptr, stream, &c);
    if (rc) return rc;
    rc = o3db_icp_iterate(c, options->max_iteration, stream);
    if (rc == O3DB_OK) rc = o3db_icp_finish(c, result, correspondences_dev, per_iteration_host, stream);
    cudaStreamSynchronize((cudaStream_t)stream);
    o3db_icp_destroy(c);
    return rc;
}

int o3db_icp_point_to_point(const float* source_dev, int64_t n, const float* target_dev, int64_t m, const double init_T[16],
                            const o3db_icp_options* options, o3db_icp_result* result, int64_t* correspondences_dev,
                            double* per_iteration_host, void* stream) {
    o3db_icp* c = nullptr;
    int rc = o3db_icp_create_point_to_point(source_dev, n, target_dev, m, init_T, options, nullptr, stream, &c);
    if (rc) return rc;
    rc = o3db_icp_iterate(c, options->max_iteration, stream);
    if (rc == O3DB_OK) rc = o3db_icp_finish(c, result, correspondences_dev, per_iteration_host, stream);
    cudaStreamSynchronize((cudaStream_t)stream);
    o3db_icp_destroy(c);
    return rc;
}

int o3db_icp_colored(const float* source_dev, const float* source_colors_dev, int64_t n, const float* target_dev,
                     const float* target_normals_dev, const float* target_colors_dev,
                     const float* target_color_gradients_dev, int64_t m, const double init_T[16],
                     const o3db_icp_options* options, double lambda_geometric, o3db_icp_result* result,
                     int64_t* correspondences_dev, double* per_iteration_host, void* stream) {
    o3db_icp* c = nullptr;
    int rc = o3db_icp_create_colored(source_dev, source_colors_dev, n, target_dev, target_normals_dev,
                                     target_colors_dev, target_color_gradients_dev, m, init_T, options,
                                     lambda_geometric, nullptr, stream, &c);
    if (rc) return rc;
    rc = o3db_icp_iterate(c, options->max_iteration, stream);
    if (rc == O3DB_OK) rc = o3db_icp_finish(c, result, correspondences_dev, per_iteration_host, stream);
    cudaStreamSynchronize((cudaStream_t)stream);
    o3db_icp_destroy(c);
    return rc;
}

int o3db_icp_point_to_plane_host(const float* source_host, int64_t n, const float* target_host,
                                 const float* target_normals_host, int64_t m, const double init_T[16],
                                 const o3db_icp_options* options, o3db_icp_result* result,
                                 int64_t* correspondences_host, double* per_iteration_host) {
    O3DB_REQUIRE(source_host && target_host && n > 0 && m > 0, "Source and/or Target pointcloud is empty.");
    O3DB_REQUIRE(target_normals_host != nullptr, "Target pointcloud missing normals attribute.");
    O3DB_REQUIRE(options != nullptr && result != nullptr, "o3db_icp_point_to_plane_host: null options / result");
    configure_memory_pool();
    cudaStream_t st = 0;
    // Copy order = need order: target and normals first (the index build starts as soon as they are in), the source
    // on a second stream so that its transfer overlaps the target's bounding box / count / scan / scatter; the source
    // sort waits on the copy's event.  The 72 MB over PCIe remain the floor of this entry point.
    struct CopyLane {      // one per device, created on first use (streams and events belong to a device)
        cudaStream_t stream = nullptr;
        cudaEvent_t source_ready = nullptr, buffers_ready = nullptr;
    };
    static CopyLane lanes[64];
    int dev = 0;
    O3DB_CUDA_CHECK(cudaGetDevice(&dev));
    O3DB_REQUIRE(dev >= 0 && dev < 64, "o3db_icp_point_to_plane_host: device index out of range");
    CopyLane& lane = lanes[dev];
    if (!lane.stream) {
        O3DB_CUDA_CHECK(cudaStreamCreateWithFlags(&lane.stream, cudaStreamNonBlocking));
        O3DB_CUDA_CHECK(cudaEventCreateWithFlags(&lane.source_ready, cudaEventDisableTiming));
        O3DB_CUDA_CHECK(cudaEventCreateWithFlags(&lane.buffers_ready, cudaEventDisableTiming));
    }
    cudaStream_t copy_stream = lane.stream;
    cudaEvent_t source_ready = lane.source_ready, buffers_ready = lane.buffers_ready;
    float *d_src = nullptr, *d_tgt = nullptr, *d_nrm = nullptr;
    int64_t* d_corr = nullptr;
    O3DB_CUDA_CHECK(cudaMallocAsync(&d_src, n * 3 * sizeof(float), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&d_tgt, m * 3 * sizeof(float), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&d_nrm, m * 3 * sizeof(float), st));
    if (correspondences_host) O3DB_CUDA_CHECK(cudaMallocAsync(&d_corr, n * sizeof(int64_t), st));
    O3DB_CUDA_CHECK(cudaEventRecord(buffers_ready, st));
    O3DB_CUDA_CHECK(cudaMemcpyAsync(d_tgt, target_host, m * 3 * sizeof(float), cudaMemcpyHostToDevice, st));
    O3DB_CUDA_CHECK(cudaMemcpyAsync(d_nrm, target_normals_host, m * 3 * sizeof(float), cudaMemcpyHostToDevice, st));
    O3DB_CUDA_CHECK(cudaStreamWaitEvent(copy_stream, buffers_ready, 0));      // d_src exists (stream-ordered allocation)
    O3DB_CUDA_CHECK(cudaMemcpyAsync(d_src, source_host, n * 3 * sizeof(float), cudaMemcpyHostToDevice, copy_stream));
    O3DB_CUDA_CHECK(cudaEventRecord(source_ready, copy_stream));
    o3db_icp* c = nullptr;
    int rc = icp_create_impl(d_src, n, d_tgt, d_nrm, m, init_T, options, nullptr, o3db::EstimatorInputs{}, st, &c, source_ready);
    if (rc == O3DB_OK) rc = o3db_icp_iterate(c, options->max_iteration, st);
    if (rc == O3DB_OK) rc = o3db_icp_finish(c, result, d_corr, per_iteration_host, st);
    cudaStreamSynchronize(st);
    cudaStreamSynchronize(copy_stream);
    if (c) o3db_icp_destroy(c);
    if (rc == O3DB_OK && correspondences_host) {
        cudaError_t e = cudaMemcpyAsync(correspondences_host, d_corr, n * sizeof(int64_t), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) {
            set_last_error("D2H copy of correspondences failed: %s", cudaGetErrorString(e));
            rc = O3DB_ERR_CUDA;
        }
    }
    cudaFreeAsync(d_src, st);
    cudaFreeAsync(d_tgt, st);
    cudaFreeAsync(d_nrm, st);
    if (d_corr) cudaFreeAsync(d_corr, st);
    return rc;
}

}  // extern "C"
