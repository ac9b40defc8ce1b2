// projection.cu — point clouds from depth / RGB-D images and back, for sm_90a.
//
// Unproject: PointCloud::CreateFromDepthImage / CreateFromRGBDImage (t/geometry/PointCloud.cpp:1414-1469) ->
// kernel::pointcloud::Unproject (kernel/PointCloudImpl.h:43-144).  One point per strided pixel (x, y) =
// (j * stride, i * stride) with 0 < d < depth_max, d = depth / depth_scale, at RigidTransform(pose, Unproject(x, y, d))
// with pose = InverseTransformation(extrinsics), and the colour pixel at (x, y) as f32 without scaling.  Upstream
// appends rows through an atomic counter; here the order is fixed, row-major over the strided grid, in five launches
// whatever the image:
//   count        one CTA per tile of kPT strided pixels: a ballot per warp, one u32 per tile;
//   scan         exclusive scan of the tile counts (icp.cu's u32 scan, scan.cuh, three launches);
//   emit         the same tiles again: each valid pixel's row is its tile's offset plus its rank in the tile (ballot /
//                popc within the warp, a scan of the warp counts across the CTA).
// The one host synchronisation reads the point count.
//
// Project: PointCloud::ProjectToDepthImage / ProjectToRGBDImage (PointCloud.cpp:1471-1530) -> kernel::pointcloud::
// Project (kernel/PointCloudCUDA.cu:26-162).  Each point goes through RigidTransform(extrinsics), Project and a round
// half away from zero, and is rejected when !InBoundary(u, v) || zc <= 0 || zc > depth_max.  Each pixel keeps the
// point with the least (float bits of d = zc * depth_scale, point index): the reference CUDA kernel's packed 64-bit
// atomicMin, used for depth-only images too so that the result never depends on thread order.  Two launches after a
// fill of the key buffer, no host synchronisation:
//   scatter      one 64-bit atomicMin per accepted point;
//   resolve      one thread per pixel writes 0 or the winner's depth (and colour), so the outputs need no zeroing.
//
// Every f32 expression is evaluated in the reference's source order with round-to-nearest intrinsics (vbg.cuh), so
// the rows and pixels equal the CPU oracle's (oracle/projection) bit for bit.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "scan.cuh"
#include "vbg.cuh"

namespace o3db {

static constexpr int kPT = 256;   // threads per CTA of the projection kernels; strided pixels per unproject tile

struct UnprojectArgs {
    const void* depth;          // [rows][cols] u16 or f32
    const void* color;          // [rows][cols][3] u8 or f32, null: depth only
    int depth_f32, color_f32;
    int cols;                   // row pitch of the images, in pixels
    int stride, cols_strided;
    int npix;                   // (rows / stride) * (cols / stride)
    Cam cam;                    // intrinsics, pose = InverseTransformation(extrinsics), scale 1
    float depth_scale, depth_max;
    unsigned* counts;           // [tiles + 1]: points per tile, then their exclusive scan
    float* points;
    float* colors;
};

// Strided pixel w of the grid: its image coordinates and whether it yields a point (PointCloudImpl.h:96-101).
__device__ __forceinline__ bool unproject_valid(const UnprojectArgs& a, int w, int& x, int& y, float& d) {
    if (w >= a.npix) return false;
    y = (w / a.cols_strided) * a.stride;
    x = (w % a.cols_strided) * a.stride;
    const size_t p = (size_t)y * a.cols + x;
    const float raw = a.depth_f32 ? static_cast<const float*>(a.depth)[p]
                                  : (float)static_cast<const uint16_t*>(a.depth)[p];
    d = dvd(raw, a.depth_scale);
    return d > 0.f && d < a.depth_max;
}

__global__ void __launch_bounds__(kPT) unproject_count_kernel(UnprojectArgs a) {
    __shared__ unsigned s_warp[kPT / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x, y;
    float d;
    const bool ok = unproject_valid(a, blockIdx.x * kPT + threadIdx.x, x, y, d);
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned t = 0;
#pragma unroll
        for (int k = 0; k < kPT / 32; ++k) t += s_warp[k];
        a.counts[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(kPT) unproject_emit_kernel(UnprojectArgs a) {
    __shared__ unsigned s_warp[kPT / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = 0, y = 0;
    float d = 0.f;
    // The depth image was complete before the count pass began, so it is read before waiting for the scan.
    const bool ok = unproject_valid(a, blockIdx.x * kPT + threadIdx.x, x, y, d);
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    unsigned base = 0;
#pragma unroll
    for (int k = 0; k < kPT / 32; ++k) base += k < warp ? s_warp[k] : 0u;
    pdl_wait();
    if (!ok) return;
    const size_t row = (size_t)a.counts[blockIdx.x] + base + __popc(m & ((1u << lane) - 1u));
    float xc, yc, zc;
    unproject(a.cam, (float)x, (float)y, d, xc, yc, zc);   // PointCloudImpl.h:109-116
    float* p = a.points + 3 * row;
    rigid(a.cam, xc, yc, zc, p[0], p[1], p[2]);
    if (a.color) {   // :117-126, the colour image as f32 (CreateFromRGBDImage converts it without scaling)
        const size_t q = 3 * ((size_t)y * a.cols + x);
        float* c = a.colors + 3 * row;
        if (a.color_f32) {
            const float* s = static_cast<const float*>(a.color) + q;
            c[0] = s[0];
            c[1] = s[1];
            c[2] = s[2];
        } else {
            const uint8_t* s = static_cast<const uint8_t*>(a.color) + q;
            c[0] = (float)s[0];
            c[1] = (float)s[1];
            c[2] = (float)s[2];
        }
    }
}

// PointCloudCUDA.cu:86-115: the packed (depth bits, point index) minimum per pixel.
__global__ void __launch_bounds__(kPT) project_scatter_kernel(const float* __restrict__ pts, int n, Cam cam,
                                                              float depth_scale, float depth_max, int rows, int cols,
                                                              unsigned long long* __restrict__ keys) {
    const int i = blockIdx.x * kPT + threadIdx.x;
    if (i >= n) return;
    float xc, yc, zc, u, v;
    rigid(cam, pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2], xc, yc, zc);
    project(cam, xc, yc, zc, u, v);
    u = roundf(u);
    v = roundf(v);
    if (!in_boundary(u, v, rows, cols) || zc <= 0.f || zc > depth_max) return;
    const float d = mul(zc, depth_scale);
    const unsigned long long key = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)i;
    atomicMin(keys + (size_t)(int)v * cols + (int)u, key);
}

__global__ void __launch_bounds__(kPT) project_resolve_kernel(const unsigned long long* __restrict__ keys,
                                                              long long npix, const float* __restrict__ pt_colors,
                                                              float* __restrict__ depth, float* __restrict__ color) {
    pdl_wait();
    const long long p = blockIdx.x * (long long)kPT + threadIdx.x;
    if (p >= npix) return;
    const unsigned long long key = keys[p];
    const bool hit = key != ~0ull;
    depth[p] = hit ? __uint_as_float((unsigned)(key >> 32)) : 0.f;
    if (color) {
        const float* c = pt_colors + 3 * (size_t)(unsigned)key;
        color[3 * p] = hit ? c[0] : 0.f;
        color[3 * p + 1] = hit ? c[1] : 0.f;
        color[3 * p + 2] = hit ? c[2] : 0.f;
    }
}

}  // namespace o3db

using namespace o3db;

extern "C" {

int o3db_unproject(const void* depth_dev, int depth_dtype, int rows, int cols, const void* color_dev, int color_dtype,
                   const double intrinsic_host[9], const double extrinsic_host[16], float depth_scale, float depth_max,
                   int stride, float* points_dev, float* colors_dev, int64_t* num_points, void* stream) {
    O3DB_REQUIRE(num_points != nullptr, "o3db_unproject: null num_points");
    *num_points = 0;
    O3DB_REQUIRE(intrinsic_host && extrinsic_host, "o3db_unproject: null intrinsic / extrinsic");
    O3DB_REQUIRE(rows >= 0 && cols >= 0, "o3db_unproject: negative image size %d x %d", rows, cols);
    O3DB_REQUIRE(stride >= 1, "o3db_unproject: stride must be >= 1 (got %d)", stride);
    O3DB_REQUIRE(std::isfinite(depth_scale) && depth_scale > 0.f,
                 "o3db_unproject: depth_scale must be finite and positive (got %g)", (double)depth_scale);
    O3DB_REQUIRE(depth_dtype == O3DB_DEPTH_U16 || depth_dtype == O3DB_DEPTH_F32,
                 "o3db_unproject: depth must be UInt16 or Float32");
    O3DB_REQUIRE(!color_dev || color_dtype == O3DB_COLOR_U8 || color_dtype == O3DB_COLOR_F32,
                 "o3db_unproject: colour must be UInt8 or Float32");
    const int64_t rs = rows / stride, cs = cols / stride, npix = rs * cs;
    O3DB_REQUIRE(npix < ((int64_t)1 << 31), "o3db_unproject: the strided grid has %lld pixels, 2^31 or more",
                 (long long)npix);
    // an empty strided grid reads and writes nothing
    O3DB_REQUIRE(npix == 0 || (depth_dev && points_dev), "o3db_unproject: null depth / points");
    O3DB_REQUIRE(npix == 0 || !color_dev || colors_dev, "o3db_unproject: null colours output for a colour image");
    cudaStream_t st = (cudaStream_t)stream;
    double pose[16];
    inverse_transformation(extrinsic_host, pose);   // PointCloudImpl.h:63-64
    UnprojectArgs a{};
    a.depth = depth_dev;
    a.color = color_dev;
    a.depth_f32 = depth_dtype == O3DB_DEPTH_F32;
    a.color_f32 = color_dtype == O3DB_COLOR_F32;
    a.cols = cols;
    a.stride = stride;
    a.cols_strided = (int)cs;
    a.npix = (int)npix;
    a.cam = make_cam(intrinsic_host, pose, 1.0f);
    a.depth_scale = depth_scale;
    a.depth_max = depth_max;
    a.points = points_dev;
    a.colors = color_dev ? colors_dev : nullptr;
    // at least one tile, so that an empty grid runs the same launches
    const int64_t tiles = std::max<int64_t>(1, ceil_div(npix, kPT));
    const int64_t scan_tiles = ceil_div(tiles, kScanTile);
    unsigned* buf = nullptr;
    O3DB_CUDA_CHECK(cudaMallocAsync(&buf, (size_t)(tiles + 1 + scan_tiles) * sizeof(unsigned), st));
    a.counts = buf;
    unsigned* h_total = (unsigned*)pinned_acquire(sizeof(unsigned));
    int rc = O3DB_OK;
    cudaError_t e = cudaSuccess;
    if (!h_total) {
        set_last_error("o3db_unproject: out of pinned host memory");
        rc = O3DB_ERR_CUDA;
    }
    if (rc == O3DB_OK) {
        unproject_count_kernel<<<(unsigned)tiles, kPT, 0, st>>>(a);
        count_launch();
        e = cudaGetLastError();
        if (e == cudaSuccess) rc = exclusive_scan_u32(buf, tiles, buf + tiles + 1, st);
        if (e == cudaSuccess && rc == O3DB_OK) {
            e = launch_pdl_ex(unproject_emit_kernel, {(unsigned)tiles, kPT}, st, a);
            count_launch();
        }
        if (e == cudaSuccess && rc == O3DB_OK)
            e = cudaMemcpyAsync(h_total, buf + tiles, sizeof(unsigned), cudaMemcpyDeviceToHost, st);
        if (e != cudaSuccess) {
            set_last_error("o3db_unproject: %s", cudaGetErrorString(e));
            rc = O3DB_ERR_CUDA;
        }
    }
    cudaFreeAsync(buf, st);
    if (rc == O3DB_OK) {
        e = cudaStreamSynchronize(st);   // the one host synchronisation: the point count
        if (e != cudaSuccess) {
            set_last_error("o3db_unproject: %s", cudaGetErrorString(e));
            rc = O3DB_ERR_CUDA;
        } else {
            *num_points = *h_total;
        }
    }
    if (h_total) pinned_release(h_total);
    return rc;
}

int o3db_project(const float* points_dev, const float* colors_dev, int64_t n, const double intrinsic_host[9],
                 const double extrinsic_host[16], float depth_scale, float depth_max, int rows, int cols,
                 float* depth_dev, float* color_dev, void* stream) {
    O3DB_REQUIRE(intrinsic_host && extrinsic_host, "o3db_project: null intrinsic / extrinsic");
    O3DB_REQUIRE(rows >= 0 && cols >= 0, "o3db_project: negative image size %d x %d", rows, cols);
    O3DB_REQUIRE(n >= 0 && n < ((int64_t)1 << 31), "o3db_project: %lld points; the point index must fit in 31 bits",
                 (long long)n);
    O3DB_REQUIRE(std::isfinite(depth_scale) && depth_scale > 0.f,
                 "o3db_project: depth_scale must be finite and positive (got %g)", (double)depth_scale);
    const int64_t npix = (int64_t)rows * cols;
    O3DB_REQUIRE(npix == 0 || depth_dev, "o3db_project: null depth output");
    O3DB_REQUIRE(n == 0 || points_dev, "o3db_project: null points");
    O3DB_REQUIRE(n == 0 || !color_dev || colors_dev, "o3db_project: a colour image needs point colours");
    O3DB_REQUIRE(npix == 0 || !colors_dev || color_dev, "o3db_project: point colours need a colour image");
    cudaStream_t st = (cudaStream_t)stream;
    const Cam cam = make_cam(intrinsic_host, extrinsic_host, 1.0f);   // PointCloudCUDA.cu:46
    unsigned long long* keys = nullptr;
    O3DB_CUDA_CHECK(cudaMallocAsync(&keys, (size_t)std::max<int64_t>(npix, 1) * sizeof(unsigned long long), st));
    cudaError_t e = cudaMemsetAsync(keys, 0xff, (size_t)npix * sizeof(unsigned long long), st);
    if (e == cudaSuccess) {
        project_scatter_kernel<<<(unsigned)std::max<int64_t>(1, ceil_div(n, kPT)), kPT, 0, st>>>(
                points_dev, (int)n, cam, depth_scale, depth_max, rows, cols, keys);
        count_launch();
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        e = launch_pdl_ex(project_resolve_kernel, {(unsigned)std::max<int64_t>(1, ceil_div(npix, kPT)), kPT}, st,
                          keys, (long long)npix, colors_dev, depth_dev, color_dev);
        count_launch();
    }
    cudaFreeAsync(keys, st);
    if (e != cudaSuccess) {
        set_last_error("o3db_project: %s", cudaGetErrorString(e));
        return O3DB_ERR_CUDA;
    }
    return O3DB_OK;
}

}  // extern "C"
