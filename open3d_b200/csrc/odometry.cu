// odometry.cu — RGB-D odometry, PointToPlane method, for sm_90a (SURVEY.md 8f #2): what
// slam::Model::TrackFrameToModel runs between RayCast and Integrate in the dense-SLAM loop.
//
// Reference: t/pipelines/odometry/RGBDOdometry.cpp:56-206 (RGBDOdometryMultiScale / ...PointToPlane driver),
// :432-459 (ComputeOdometryResultPointToPlane), t/pipelines/kernel/RGBDOdometryCUDA.cu:37-125 + RGBDOdometryJacobianImpl.h
// (per-pixel Jacobian, Huber terms, 29-float BlockReduce + atomics, host DecodeAndSolve6x6), and the depth-pyramid
// kernels of t/geometry/kernel/ImageImpl.h:86-315 (ClipTransform, PyrDownDepth, CreateVertexMap, CreateNormalMap).
//
// Here the whole multi-scale loop is device resident, like the ICP loop of icp.cu: one kernel per iteration does the
// per-pixel projection + Jacobian, the 29-scalar reduction of reduce.cuh (f32 partials -> f64 tree, deterministic) and,
// in the last block, the f64 6x6 solve, T <- dT * T, the result bookkeeping and the reference's relative convergence
// test; a level that has converged turns its remaining launches into no-ops.  No host synchronisation until the end
// (upstream: one cuda::Synchronize + 29-float D2H + host LU per iteration).
//
// Image::FilterBilateral is NPP upstream (closed source): the kernel here evaluates NPP's documented
// definition of nppiFilterBilateralGaussBorder (see o3db_image_filter_bilateral in the header) — parity unpinned.
//
// All pixel-selecting arithmetic (projection, roundf, residual gate) is evaluated without FMA contraction in the
// reference's source order, as everywhere else in this library.
#include <atomic>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <vector>

#include <cooperative_groups.h>

#include "common.cuh"
#include "reduce.cuh"
#include "vbg.cuh"

namespace o3db {

static constexpr int kOT = 256;
#ifndef ODO_BLOCKS_PER_SM
#define ODO_BLOCKS_PER_SM 4   // blocks per SM of the iteration kernel; fewer = shorter serial tail in the last block (tunable)
#endif

// ------------------------------------------------------------ image kernels

template <typename src_t>
__global__ void clip_transform_kernel(const src_t* __restrict__ src, int64_t n, float scale, float min_value,
                                      float max_value, float clip_fill, float* __restrict__ dst) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float out = dvd((float)src[i], scale);   // ImageImpl.h:112-116
    out = out <= min_value ? clip_fill : out;
    out = out >= max_value ? clip_fill : out;
    dst[i] = out;
}

// ImageImpl.h:122-198
__global__ void pyr_down_depth_kernel(const float* __restrict__ src, int rows, int cols, float depth_diff,
                                      float invalid_fill, float* __restrict__ dst) {
    const int rows_down = rows / 2, cols_down = cols / 2;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows_down * cols_down) return;
    const int y = i / cols_down, x = i % cols_down;
    const int y_src = 2 * y, x_src = 2 * x;
    const float v_center = src[(size_t)y_src * cols + x_src];
    if (v_center == invalid_fill) {
        dst[i] = invalid_fill;
        return;
    }
    const float gweights[3] = {0.375f, 0.25f, 0.0625f};
    const int x_min = max(0, x_src - 2), y_min = max(0, y_src - 2);
    const int x_max = min(cols - 1, x_src + 2), y_max = min(rows - 1, y_src + 2);
    float v_sum = 0.f, w_sum = 0.f;
    for (int yk = y_min; yk <= y_max; ++yk)
        for (int xk = x_min; xk <= x_max; ++xk) {
            const float v = src[(size_t)yk * cols + xk];
            const int dy = abs(yk - y_src), dx = abs(xk - x_src);
            if (v != invalid_fill && fabsf(sub(v, v_center)) < depth_diff) {
                const float w = mul(gweights[dx], gweights[dy]);
                v_sum = add(v_sum, mul(w, v));
                w_sum = add(w_sum, w);
            }
        }
    dst[i] = w_sum == 0 ? invalid_fill : dvd(v_sum, w_sum);
}

__device__ __forceinline__ bool is_invalid(float v, float invalid_fill) {   // ImageImpl.h:227-231
    if (isinf(invalid_fill)) return isinf(v);
    if (isnan(invalid_fill)) return isnan(v);
    return v == invalid_fill;
}

// ImageImpl.h:200-248
__global__ void create_vertex_map_kernel(const float* __restrict__ depth, int rows, int cols, Cam ti, float invalid_fill,
                                         float* __restrict__ vertex) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * cols) return;
    const int y = i / cols, x = i % cols;
    const float d = depth[i];
    float vx = invalid_fill, vy = invalid_fill, vz = invalid_fill;
    if (!is_invalid(d, invalid_fill)) unproject(ti, (float)x, (float)y, d, vx, vy, vz);
    vertex[3 * (size_t)i] = vx;
    vertex[3 * (size_t)i + 1] = vy;
    vertex[3 * (size_t)i + 2] = vz;
}

// ImageImpl.h:249-315
__global__ void create_normal_map_kernel(const float* __restrict__ vertex, int rows, int cols, float invalid_fill,
                                         float* __restrict__ normal) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * cols) return;
    const int y = i / cols, x = i % cols;
    float n0 = invalid_fill, n1 = invalid_fill, n2 = invalid_fill;
    if (y < rows - 1 && x < cols - 1) {
        const float* v00 = vertex + 3 * (size_t)i;
        const float* v10 = v00 + 3;
        const float* v01 = v00 + 3 * (size_t)cols;
        const bool bad = (v00[0] == invalid_fill && v00[1] == invalid_fill && v00[2] == invalid_fill) ||
                         (v01[0] == invalid_fill && v01[1] == invalid_fill && v01[2] == invalid_fill) ||
                         (v10[0] == invalid_fill && v10[1] == invalid_fill && v10[2] == invalid_fill);
        if (!bad) {
            const float dx0 = sub(v01[0], v00[0]), dy0 = sub(v01[1], v00[1]), dz0 = sub(v01[2], v00[2]);
            const float dx1 = sub(v10[0], v00[0]), dy1 = sub(v10[1], v00[1]), dz1 = sub(v10[2], v00[2]);
            n0 = sub(mul(dy0, dz1), mul(dz0, dy1));
            n1 = sub(mul(dz0, dx1), mul(dx0, dz1));
            n2 = sub(mul(dx0, dy1), mul(dy0, dx1));
            float norm = __fsqrt_rn(add(add(mul(n0, n0), mul(n1, n1)), mul(n2, n2)));
            norm = fmaxf(norm, 1e-5f);
            n0 = dvd(n0, norm);
            n1 = dvd(n1, norm);
            n2 = dvd(n2, norm);
        }
    }
    normal[3 * (size_t)i] = n0;
    normal[3 * (size_t)i + 1] = n1;
    normal[3 * (size_t)i + 2] = n2;
}

// nppiFilterBilateralGaussBorder_32f_C1R (NPPImage.cpp:319-376) by its documented definition; replicated border.
__global__ void filter_bilateral_kernel(const float* __restrict__ src, int rows, int cols, int radius, float val2,
                                        float pos2, float* __restrict__ dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * cols) return;
    const int y = i / cols, x = i % cols;
    const float vc = src[i];
    float v_sum = 0.f, w_sum = 0.f;
    for (int dy = -radius; dy <= radius; ++dy)
        for (int dx = -radius; dx <= radius; ++dx) {
            const int yy = min(max(y + dy, 0), rows - 1), xx = min(max(x + dx, 0), cols - 1);
            const float v = src[(size_t)yy * cols + xx];
            const float dv = sub(v, vc);
            const float w = mul(expf(dvd(-((float)(dx * dx + dy * dy)), pos2)), expf(dvd(-mul(dv, dv), val2)));
            v_sum = add(v_sum, mul(w, v));
            w_sum = add(w_sum, w);
        }
    dst[i] = dvd(v_sum, w_sum);
}


// ------------------------------------------- fused pyramid level (the multi-scale driver's own path)

// Everything RGBDOdometryMultiScalePointToPlane needs from one pyramid level (RGBDOdometry.cpp:132-163) in ONE launch
// instead of seven: source and target vertex maps, the target normal map (bilateral filter -> vertex map of the
// smoothed depth -> normals) and, unless this is the coarsest level, both depth images of the next level.  A block
// owns a 32 x 8 pixel tile: the target depth tile with its 2-pixel filter apron (+1 for the normal stencil) is staged
// in shared memory once, the smoothed depths of the 33 x 9 stencil points and their vertices live in shared memory
// too, so the filter runs once per pixel and the normal map never reads a smoothed image back from HBM.  The
// per-pixel arithmetic is the stand-alone kernels' (same device functions, same order): bit-identical maps.
static constexpr int kMaxLevels = 8;

struct OdoState {
    double T[16];                 // source -> target, updated every iteration
    double sums[kSumStride];
    double res_rmse, res_fitness; // OdometryResult::inlier_rmse_ / fitness_ (RGBDOdometry.cpp:165, 190-191)
    int level_done[kMaxLevels];
    int status;                   // 0 ok, 1 singular 6x6, 2 inlier_count <= 0
    int executed;
    unsigned ticket;
};

static constexpr int kTW = 32, kTH = 8;
struct LevelArgs {
    const float* src_d;      // this level's depth images (metres, NaN = invalid)
    const float* tgt_d;
    int rows, cols;
    Cam ti;                  // this level's intrinsics
    float invalid_fill;      // NaN
    float val2, pos2;        // bilateral filter: 2 sigma_value^2, 2 sigma_position^2 (radius 2)
    float depth_diff;        // PyrDownDepth threshold
    float* sv;
    float* tv;
    float* tn;
    float* src_next;         // nullptr on the coarsest level
    float* tgt_next;
    OdoState* init_state;    // first launch of a track: the state the iterations start from (no copy / memset on the stream)
    double init_T[16];
};

__device__ __forceinline__ float pyr_down_pixel(const float* __restrict__ img, int rows, int cols, int yd, int xd,
                                                float depth_diff, float invalid_fill) {
    const int yc = 2 * yd, xc = 2 * xd;
    const float centre = img[(size_t)yc * cols + xc];
    if (centre == invalid_fill) return invalid_fill;      // (as upstream: never true for a NaN fill)
    const float gw[3] = {0.375f, 0.25f, 0.0625f};
    float num = 0.f, den = 0.f;
    for (int yk = max(0, yc - 2); yk <= min(rows - 1, yc + 2); ++yk)
        for (int xk = max(0, xc - 2); xk <= min(cols - 1, xc + 2); ++xk) {
            const float v = img[(size_t)yk * cols + xk];
            if (v != invalid_fill && fabsf(sub(v, centre)) < depth_diff) {
                const float w = mul(gw[abs(xk - xc)], gw[abs(yk - yc)]);
                num = add(num, mul(w, v));
                den = add(den, w);
            }
        }
    return den == 0 ? invalid_fill : dvd(num, den);
}

// kUnrollRows: the 5 x 5 tap loop fully unrolled (64 registers, 4 blocks per SM) or by rows (48 registers, 5 blocks).
template <bool kUnrollRows>
__global__ void __launch_bounds__(kTW* kTH) pyramid_level_kernel(LevelArgs a) {
    __shared__ float s_depth[kTH + 5][kTW + 5];       // target depth, rows y0-2 .. y0+kTH+2, cols x0-2 .. x0+kTW+2 (clamped)
    __shared__ float s_vert[kTH + 1][kTW + 1][3];     // vertices of the smoothed depth at the normal stencil points
    __shared__ float s_wpos[5][5];                    // the filter's spatial weights: one division + expf each, once per block
    pdl_grid_wait();
    pdl_grid_launch_dependents();
    if (a.init_state && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
        // RGBDOdometry.cpp:165 OdometryResult(trans, /*prev rmse*/ 0.0, /*prev fitness*/ 1.0); the iteration kernels read
        // it after their griddepcontrol.wait, i.e. after every pyramid launch has completed
        OdoState z{};
        for (int i = 0; i < 16; ++i) z.T[i] = a.init_T[i];
        z.res_fitness = 1.0;
        *a.init_state = z;
    }
    const int tx = threadIdx.x % kTW, ty = threadIdx.x / kTW;
    const int x0 = blockIdx.x * kTW, y0 = blockIdx.y * kTH;
    const int x = x0 + tx, y = y0 + ty;
    for (int k = threadIdx.x; k < (kTH + 5) * (kTW + 5); k += kTW * kTH) {
        const int ly = k / (kTW + 5), lx = k % (kTW + 5);
        const int gy = min(max(y0 + ly - 2, 0), a.rows - 1), gx = min(max(x0 + lx - 2, 0), a.cols - 1);   // replicated border
        s_depth[ly][lx] = a.tgt_d[(size_t)gy * a.cols + gx];
    }
    if (threadIdx.x < 25) {   // the very expression the per-tap code evaluated (and filter_bilateral_kernel evaluates): same bits
        const int dy = (int)threadIdx.x / 5 - 2, dx = (int)threadIdx.x % 5 - 2;
        s_wpos[dy + 2][dx + 2] = expf(dvd(-((float)(dx * dx + dy * dy)), a.pos2));
    }
    __syncthreads();
    // bilateral filter (radius 2) + vertex of the smoothed depth at every stencil point of the tile
    for (int k = threadIdx.x; k < (kTH + 1) * (kTW + 1); k += kTW * kTH) {
        const int ly = k / (kTW + 1), lx = k % (kTW + 1);
        const int gy = y0 + ly, gx = x0 + lx;
        float vx = a.invalid_fill, vy = a.invalid_fill, vz = a.invalid_fill;
        if (gy < a.rows && gx < a.cols) {
            const float vc = s_depth[ly + 2][lx + 2];
            float num = 0.f, den = 0.f;
            // the apron was loaded with clamped coordinates; inside the image clamping (gy + dy) equals indexing it
            int cy[5], cx[5];
#pragma unroll
            for (int d = 0; d < 5; ++d) {
                cy[d] = min(max(gy + d - 2, 0), a.rows - 1) - (y0 - 2);
                cx[d] = min(max(gx + d - 2, 0), a.cols - 1) - (x0 - 2);
            }
            auto taps_of_row = [&](int dy) {
#pragma unroll
                for (int dx = 0; dx < 5; ++dx) {
                    const float v = s_depth[cy[dy]][cx[dx]];
                    const float dv = sub(v, vc);
                    const float w = mul(s_wpos[dy][dx], expf(dvd(-mul(dv, dv), a.val2)));
                    num = add(num, mul(w, v));
                    den = add(den, w);
                }
            };
            if constexpr (kUnrollRows) {
#pragma unroll
                for (int dy = 0; dy < 5; ++dy) taps_of_row(dy);
            } else {
#pragma unroll 1
                for (int dy = 0; dy < 5; ++dy) taps_of_row(dy);
            }
            const float smooth = dvd(num, den);
            if (!is_invalid(smooth, a.invalid_fill)) unproject(a.ti, (float)gx, (float)gy, smooth, vx, vy, vz);
        }
        s_vert[ly][lx][0] = vx;
        s_vert[ly][lx][1] = vy;
        s_vert[ly][lx][2] = vz;
    }
    __syncthreads();
    if (y < a.rows && x < a.cols) {
        const size_t i = (size_t)y * a.cols + x;
        // source / target vertex maps (ImageImpl.h:200-248)
        const float ds = a.src_d[i], dt = s_depth[ty + 2][tx + 2];
        float v[3] = {a.invalid_fill, a.invalid_fill, a.invalid_fill};
        if (!is_invalid(ds, a.invalid_fill)) unproject(a.ti, (float)x, (float)y, ds, v[0], v[1], v[2]);
        a.sv[3 * i] = v[0];
        a.sv[3 * i + 1] = v[1];
        a.sv[3 * i + 2] = v[2];
        v[0] = v[1] = v[2] = a.invalid_fill;
        if (!is_invalid(dt, a.invalid_fill)) unproject(a.ti, (float)x, (float)y, dt, v[0], v[1], v[2]);
        a.tv[3 * i] = v[0];
        a.tv[3 * i + 1] = v[1];
        a.tv[3 * i + 2] = v[2];
        // target normal map from the smoothed vertices (ImageImpl.h:249-315)
        float n0 = a.invalid_fill, n1 = a.invalid_fill, n2 = a.invalid_fill;
        if (y < a.rows - 1 && x < a.cols - 1) {
            const float* v00 = s_vert[ty][tx];
            const float* v10 = s_vert[ty][tx + 1];
            const float* v01 = s_vert[ty + 1][tx];
            const float f = a.invalid_fill;
            const bool bad = (v00[0] == f && v00[1] == f && v00[2] == f) || (v01[0] == f && v01[1] == f && v01[2] == f) ||
                             (v10[0] == f && v10[1] == f && v10[2] == f);
            if (!bad) {
                const float ax = sub(v01[0], v00[0]), ay = sub(v01[1], v00[1]), az = sub(v01[2], v00[2]);
                const float bx = sub(v10[0], v00[0]), by = sub(v10[1], v00[1]), bz = sub(v10[2], v00[2]);
                n0 = sub(mul(ay, bz), mul(az, by));
                n1 = sub(mul(az, bx), mul(ax, bz));
                n2 = sub(mul(ax, by), mul(ay, bx));
                const float norm = fmaxf(__fsqrt_rn(add(add(mul(n0, n0), mul(n1, n1)), mul(n2, n2))), 1e-5f);
                n0 = dvd(n0, norm);
                n1 = dvd(n1, norm);
                n2 = dvd(n2, norm);
            }
        }
        a.tn[3 * i] = n0;
        a.tn[3 * i + 1] = n1;
        a.tn[3 * i + 2] = n2;
    }
    // next level's depth images (ImageImpl.h:122-198): the 16 x 4 half-resolution pixels under this tile, both images
    if (a.src_next && threadIdx.x < 2 * (kTW / 2) * (kTH / 2)) {
        const int which = threadIdx.x / ((kTW / 2) * (kTH / 2)), k = threadIdx.x % ((kTW / 2) * (kTH / 2));
        const int xd = x0 / 2 + k % (kTW / 2), yd = y0 / 2 + k / (kTW / 2);
        if (yd < a.rows / 2 && xd < a.cols / 2) {
            const float out = pyr_down_pixel(which ? a.tgt_d : a.src_d, a.rows, a.cols, yd, xd, a.depth_diff, a.invalid_fill);
            (which ? a.tgt_next : a.src_next)[(size_t)yd * (a.cols / 2) + xd] = out;
        }
    }
}

// ClipTransform of both frames in one launch (blockIdx.y selects the image).
template <typename s_t, typename t_t>
__global__ void clip_transform_pair_kernel(const s_t* __restrict__ src, const t_t* __restrict__ tgt, int64_t n, float scale,
                                           float min_value, float max_value, float clip_fill, float* __restrict__ src_out,
                                           float* __restrict__ tgt_out) {
    pdl_grid_wait();
    pdl_grid_launch_dependents();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float out = blockIdx.y == 0 ? dvd((float)src[i], scale) : dvd((float)tgt[i], scale);   // ImageImpl.h:112-116
    out = out <= min_value ? clip_fill : out;
    out = out >= max_value ? clip_fill : out;
    (blockIdx.y == 0 ? src_out : tgt_out)[i] = out;
}

// ------------------------------------------------------ per-pixel Jacobian

// RGBDOdometryJacobianImpl.h:29-37.  Sign() takes an int (GeometryMacros.h:92): the residual is truncated first.
__device__ __forceinline__ float huber_deriv(float r, float delta) {
    const float abs_r = fabsf(r);
    const int ir = (int)r;
    return abs_r < delta ? r : mul(delta, (float)((ir > 0) ? 1 : ((ir < 0) ? -1 : 0)));
}
__device__ __forceinline__ float huber_loss(float r, float delta) {
    const float abs_r = fabsf(r);
    // `0.5 * r * r` / `delta * abs_r - 0.5 * delta * delta`: double where the literal forces it, as written
    return abs_r < delta ? (float)__dmul_rn(__dmul_rn(0.5, (double)r), (double)r)
                         : (float)__dsub_rn((double)mul(delta, abs_r), __dmul_rn(__dmul_rn(0.5, (double)delta), (double)delta));
}

// RGBDOdometryJacobianImpl.h:106-160 in two phases, so that a thread can keep several pixels' loads in flight
// (odometry_level_kernel); jacobian_p2plane below is the two of them back to back.
// Phase 1: transformed source vertex and the target pixel it projects to; false = rejected.
__device__ __forceinline__ bool probe_source(float s0, float s1, float s2, int rows, int cols, const Cam& ti, float& p0,
                                             float& p1, float& p2, int& target_index) {
    if (isnan(s0)) return false;
    float u, v;
    rigid(ti, s0, s1, s2, p0, p1, p2);
    project(ti, p0, p1, p2, u, v);
    u = roundf(u);
    v = roundf(v);
    if (p2 < 0 || !in_boundary(u, v, rows, cols)) return false;
    target_index = (int)v * cols + (int)u;
    return true;
}
// Phase 2: residual gate and Jacobian from the target vertex t and normal n at that pixel.
__device__ __forceinline__ bool residual_jacobian(float p0, float p1, float p2, float t0, float t1, float t2, float n0,
                                                  float n1, float n2, float trunc, float (&J)[6], float& r) {
    if (isnan(t0) || isnan(n0)) return false;
    r = add(add(mul(sub(p0, t0), n0), mul(sub(p1, t1), n1)), mul(sub(p2, t2), n2));
    if (fabsf(r) > trunc) return false;
    J[0] = add(mul(-p2, n1), mul(p1, n2));
    J[1] = sub(mul(p2, n0), mul(p0, n2));
    J[2] = add(mul(-p1, n0), mul(p0, n1));
    J[3] = n0;
    J[4] = n1;
    J[5] = n2;
    return true;
}

__device__ __forceinline__ bool jacobian_p2plane(int x, int y, float trunc, const float* __restrict__ sv_map,
                                                 const float* __restrict__ tv_map, const float* __restrict__ tn_map,
                                                 int rows, int cols, const Cam& ti, float (&J)[6], float& r) {
    const float* sv = sv_map + 3 * ((size_t)y * cols + x);
    float p0, p1, p2;
    int ti_idx;
    if (!probe_source(sv[0], sv[1], sv[2], rows, cols, ti, p0, p1, p2, ti_idx)) return false;
    const float* tv = tv_map + 3 * (size_t)ti_idx;
    const float* tn = tn_map + 3 * (size_t)ti_idx;
    return residual_jacobian(p0, p1, p2, tv[0], tv[1], tv[2], tn[0], tn[1], tn[2], trunc, J, r);
}

template <int N>
__device__ __forceinline__ void accumulate_odometry(float (&acc)[N], const float (&J)[6], float r, float delta) {
    const float d_huber = huber_deriv(r, delta), r_huber = huber_loss(r, delta);
    int s = 0;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
#pragma unroll
        for (int k = 0; k <= j; ++k) acc[s++] += J[j] * J[k];   // NOT Huber-weighted, as upstream (:68-70)
        acc[21 + j] += J[j] * d_huber;
    }
    acc[27] += r_huber;
    acc[28] += 1.0f;
}

// ----------------------------------------------------------- fused loop

struct OdoArgs {
    const float* sv;
    const float* tv;
    const float* tn;
    int rows, cols, level;
    float fx, fy, cx, cy;         // this level's intrinsics (f32, TransformIndexer)
    float trunc, huber_delta;
    double rel_rmse, rel_fitness;
    double* partials;
    OdoState* st;
    double* per_iter;             // optional device log: (inlier_rmse, fitness) per executed iteration
    int standalone;               // 1: ComputeOdometryResultPointToPlane seam (T is not updated, delta -> st->sums[..])
    double* delta_out;            // standalone: 16 doubles (delta transformation)
    unsigned long long* host_out; // last launch of a track: pinned host block that receives the final state + token
    unsigned long long host_token;
};

static constexpr int kStateWords = (int)(sizeof(OdoState) / sizeof(unsigned long long));
static_assert(sizeof(OdoState) % sizeof(unsigned long long) == 0, "OdoState is copied as 8-byte words");
static constexpr int kHostTokenWord = 64;   // the token lands behind the state: the host that sees it has the state

// Final state -> pinned host memory, by the first kStateWords threads of one block (all of the block's threads must
// call it): every writer orders its stores system-wide, then one thread stores the token the host spins on — no
// device-to-host copy and no stream synchronisation at the end of a track.
__device__ __forceinline__ void publish_state(const OdoArgs& a, const OdoState* from) {
    if (!a.host_out) return;
    if (threadIdx.x < kStateWords) {
        reinterpret_cast<volatile unsigned long long*>(a.host_out)[threadIdx.x] =
            reinterpret_cast<const volatile unsigned long long*>(from)[threadIdx.x];
        __threadfence_system();
    }
    __syncthreads();
    if (threadIdx.x == 0) reinterpret_cast<volatile unsigned long long*>(a.host_out)[kHostTokenWord] = a.host_token;
}

// Host part of one Gauss-Newton step (RGBDOdometry.cpp:165-191, 441-462), run by ONE WARP (all 32 lanes must call
// it): the 6x6 solve is warp-parallel (reduce.cuh), the six sin / cos of the pose and the sixteen entries of
// T <- dT T are spread over lanes (as icp_finalize_iteration does), lane 0 keeps the books.  `st` is the state the
// step updates — the global one for the per-iteration kernel, a shared-memory copy for the level-resident kernel —
// `per_iter` the optional log.  `scratch`: >= 96 doubles of shared memory.
__device__ void odometry_finalize(const OdoArgs& a, OdoState* st, double* per_iter, const double* s_final, double* scratch) {
    const int lane = threadIdx.x & 31;
    double* s = scratch;            // [29] the sums as DecodeAndSolve6x6 receives them
    double* pose = scratch + 32;    // [6]
    double* trig = scratch + 40;    // [6] cos a, cos b, cos g, sin a, sin b, sin g (aliases the solve's matrix: dead by then)
    double* dT = scratch + 48;      // [16]
    // the 29 sums reach DecodeAndSolve6x6 as a Float32 tensor (RGBDOdometryCUDA.cu:112-124)
    if (lane < 29) s[lane] = (double)(float)s_final[lane];
    __syncwarp();
    const int count = (int)s[28];
    const bool solved = solve6x6_warp(s, scratch + 40, pose);   // TransformationConverter.cpp:215-225
    if (!solved || count <= 0) {    // singular system; RGBDOdometry.cpp:449-452 inlier_count <= 0
        if (lane == 0) st->status = !solved ? 1 : 2;
        return;
    }
    __syncwarp();
    if (lane < 3) trig[lane] = cos(pose[lane]);
    else if (lane < 6) trig[lane] = sin(pose[lane - 3]);
    __syncwarp();
    if (lane == 0) pose_to_T_trig(pose, trig[0], trig[3], trig[1], trig[4], trig[2], trig[5], dT);
    __syncwarp();
    const double d_rmse = (double)((float)s[27] / (float)count);   // float inlier_residual / int (:455)
    const double d_fit = (double)count / (double)((int64_t)a.rows * a.cols);
    if (a.standalone) {
        if (lane < 16) a.delta_out[lane] = dT[lane];
        if (lane == 0) {
            st->res_rmse = d_rmse;
            st->res_fitness = d_fit;
        }
        return;
    }
    if (lane < 16) {   // :175-176 result.transformation_ = delta.transformation_.Matmul(result.transformation_)
        const int i = lane >> 2, j = lane & 3;
        double v = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) v += dT[i * 4 + k] * st->T[k * 4 + j];
        __syncwarp(0xffffu);        // every lane has read the old T
        st->T[lane] = v;
    }
    if (lane != 0) return;
    if (per_iter) {
        per_iter[2 * st->executed] = d_rmse;
        per_iter[2 * st->executed + 1] = d_fit;
    }
    st->executed += 1;
    if (fabs(st->res_fitness - d_fit) / st->res_fitness < a.rel_fitness &&
        fabs(st->res_rmse - d_rmse) / st->res_rmse < a.rel_rmse) {   // :181-189 early exit
        st->level_done[a.level] = 1;
        return;
    }
    st->res_rmse = d_rmse;
    st->res_fitness = d_fit;
}

__global__ void __launch_bounds__(kThreads) odometry_iteration_kernel(OdoArgs a) {
    __shared__ double s_warp[kThreads / 32][kSumStride];
    __shared__ double s_final[kSumStride];
    __shared__ Cam s_cam;
    __shared__ int s_skip;
    pdl_grid_wait();                 // the previous iteration's T / flags, the pyramid kernels' maps
    pdl_grid_launch_dependents();
    if (threadIdx.x == 0) s_skip = (*(volatile int*)&a.st->level_done[a.level]) | (*(volatile int*)&a.st->status);
    if (threadIdx.x < 12) s_cam.e[threadIdx.x / 4][threadIdx.x % 4] = (float)a.st->T[threadIdx.x];   // TransformIndexer: f32
    if (threadIdx.x == 12) {
        s_cam.fx = a.fx;
        s_cam.fy = a.fy;
        s_cam.cx = a.cx;
        s_cam.cy = a.cy;
        s_cam.scale = 1.0f;
    }
    for (int k = threadIdx.x; k < (kThreads / 32) * kSumStride; k += kThreads) (&s_warp[0][0])[k] = 0.0;
    __syncthreads();
    if (s_skip) {
        if (blockIdx.x == 0) publish_state(a, a.st);   // (the state is final: the previous launch completed)
        return;
    }
    const Cam ti = s_cam;
    float acc[kNumSums];
#pragma unroll
    for (int k = 0; k < kNumSums; ++k) acc[k] = 0.f;
    const int n = a.rows * a.cols;
    int since = 0;
    for (int base = blockIdx.x * kThreads; base < n; base += gridDim.x * kThreads) {
        const int i = base + threadIdx.x;
        if (i < n) {
            float J[6], r;
            if (jacobian_p2plane(i % a.cols, i / a.cols, a.trunc, a.sv, a.tv, a.tn, a.rows, a.cols, ti, J, r))
                accumulate_odometry(acc, J, r, a.huber_delta);
        }
        if (++since == kFlushEvery) {
            flush_acc(acc, s_warp);
            since = 0;
        }
    }
    flush_acc(acc, s_warp);
    if (!block_reduce_to_global(s_warp, a.partials, &a.st->ticket, s_final)) return;
    if (threadIdx.x < 29) a.st->sums[threadIdx.x] = s_final[threadIdx.x];
    if (threadIdx.x < 32) odometry_finalize(a, a.st, a.per_iter, s_final, &s_warp[0][0]);   // (s_warp is dead: reused as scratch)
    if (a.host_out) {
        __threadfence();             // warp 0's updates of the state, before the block reads it back
        __syncthreads();
        publish_state(a, a.st);
    }
}

// ------------------------------------------------ level-resident iterations
//
// A coarse pyramid level is a few thousand pixels: its iteration is over in a couple of microseconds of work, and
// what the per-iteration kernel above spends is the fixed part — launch + drain of the predecessor, partial rows to
// global memory, the ticket, the last block's grand total.  For those levels ONE thread-block cluster runs ALL the
// iterations of the level in one launch: the pixels are strided over the cluster's CTAs, a CTA's 29 sums go through
// the transposed warp reduction (reduce.cuh) into one shared-memory row, the rows are exchanged through distributed
// shared memory behind one hardware cluster barrier per iteration, and EVERY CTA adds them in rank order and runs the
// same f64 solve / pose update on its own shared-memory copy of the state — bit-identical everywhere, so nothing is
// broadcast and the next iteration starts after a __syncthreads.  Rank 0 writes the state back at the end.
// The sums are those of the per-iteration kernel up to the association of the additions (f32 per thread and across
// the warp — at most kLevelFlush + kLevelBatch + 4 roundings deep — then f64), far inside the reference's own all-f32 reduction.
static constexpr int kLevelThreads = 512;
static constexpr int kMaxCluster = 16;
static constexpr int kLevelFlush = 16;       // f32 terms per thread between two warp reductions (at most kLevelFlush + kLevelBatch - 1)

// kLevelBatch: pixels a thread has in flight.
template <int kLevelBatch>
__global__ void __launch_bounds__(kLevelThreads, 1) odometry_level_kernel(OdoArgs a, int max_iteration) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    const unsigned crank = cluster.block_rank(), csize = cluster.num_blocks();
    __shared__ double s_warp[kLevelThreads / 32][kSumStride];
    __shared__ double s_part[2][kSumStride];     // this CTA's sums, double-buffered by iteration parity (see below)
    __shared__ double s_final[kSumStride];
    __shared__ double s_scratch[96];
    __shared__ OdoState s_st;
    __shared__ Cam s_cam;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    pdl_grid_wait();                 // the previous level's T / flags, the pyramid kernels' maps
    pdl_grid_launch_dependents();
    for (int k = threadIdx.x; k < kStateWords; k += kLevelThreads)
        reinterpret_cast<unsigned long long*>(&s_st)[k] = reinterpret_cast<const unsigned long long*>(a.st)[k];
    __syncthreads();
    // (every CTA of the cluster read the same state: the decision is uniform, no peer is left waiting)
    if (s_st.status | s_st.level_done[a.level]) {
        if (crank == 0) publish_state(a, &s_st);
        return;
    }
    double* per_iter = crank == 0 ? a.per_iter : nullptr;
    const int n = a.rows * a.cols;
    const int stride = (int)csize * kLevelThreads;
    for (int it = 0; it < max_iteration; ++it) {
        if (threadIdx.x < 12) s_cam.e[threadIdx.x / 4][threadIdx.x % 4] = (float)s_st.T[threadIdx.x];   // TransformIndexer: f32
        if (threadIdx.x == 12) {
            s_cam.fx = a.fx;
            s_cam.fy = a.fy;
            s_cam.cx = a.cx;
            s_cam.cy = a.cy;
            s_cam.scale = 1.0f;
        }
        __syncthreads();
        const Cam ti = s_cam;
        float acc[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) acc[k] = 0.f;
        double total = 0.0;          // lane l: sum l of this warp
        int since = 0;
        // kLevelBatch pixels per thread and round: all their source vertices are requested first, then all the target
        // vertices / normals — two dependent L2 round trips per round instead of two per pixel (the level is latency
        // bound: 2 - 10 pixels per thread).  The pixels are accumulated in index order, as a one-by-one loop would.
        for (int base = (int)crank * kLevelThreads; base < n; base += kLevelBatch * stride) {   // (block-uniform trip count)
            float p[kLevelBatch][3];
            int tix[kLevelBatch];
#pragma unroll
            for (int u = 0; u < kLevelBatch; ++u) {
                const int i = base + u * stride + (int)threadIdx.x;
                p[u][0] = __int_as_float(0x7fc00000);   // beyond the image: rejected like an invalid vertex
                p[u][1] = p[u][2] = 0.f;
                if (i < n) {
                    const float* sv = a.sv + 3 * (size_t)i;
                    p[u][0] = sv[0];
                    p[u][1] = sv[1];
                    p[u][2] = sv[2];
                }
            }
#pragma unroll
            for (int u = 0; u < kLevelBatch; ++u) {
                float q0, q1, q2;
                int t_index;
                if (probe_source(p[u][0], p[u][1], p[u][2], a.rows, a.cols, ti, q0, q1, q2, t_index)) {
                    p[u][0] = q0;
                    p[u][1] = q1;
                    p[u][2] = q2;
                    tix[u] = t_index;
                } else {
                    tix[u] = -1;
                }
            }
            float tv[kLevelBatch][3], tn[kLevelBatch][3];
#pragma unroll
            for (int u = 0; u < kLevelBatch; ++u) {
                const size_t o = 3 * (size_t)(tix[u] < 0 ? 0 : tix[u]);   // (a rejected pixel reads pixel 0 and ignores it)
                tv[u][0] = a.tv[o];
                tv[u][1] = a.tv[o + 1];
                tv[u][2] = a.tv[o + 2];
                tn[u][0] = a.tn[o];
                tn[u][1] = a.tn[o + 1];
                tn[u][2] = a.tn[o + 2];
            }
#pragma unroll
            for (int u = 0; u < kLevelBatch; ++u) {
                float J[6], r;
                if (tix[u] >= 0 && residual_jacobian(p[u][0], p[u][1], p[u][2], tv[u][0], tv[u][1], tv[u][2], tn[u][0],
                                                     tn[u][1], tn[u][2], a.trunc, J, r))
                    accumulate_odometry(acc, J, r, a.huber_delta);
            }
            since += kLevelBatch;
            if (since >= kLevelFlush) {
                total += (double)warp_transpose_sum32(acc);
#pragma unroll
                for (int k = 0; k < 32; ++k) acc[k] = 0.f;
                since = 0;
            }
        }
        total += (double)warp_transpose_sum32(acc);
        s_warp[w][lane] = total;
        __syncthreads();
        // Parity double buffer: a CTA refills s_part[p] two iterations later, which it can only reach after every
        // peer passed the barrier of the iteration in between — i.e. after every peer finished reading s_part[p].
        const int par = it & 1;
        if (threadIdx.x < 32) {
            double v = 0;
#pragma unroll
            for (int k = 0; k < kLevelThreads / 32; ++k) v += s_warp[k][lane];
            s_part[par][lane] = v;
        }
        cluster.sync();              // barrier.cluster arrive.release / wait.acquire: the rows are visible cluster-wide
        if (threadIdx.x < 32) {
            double t[kMaxCluster];   // all the peers' rows in flight, then added in rank order
#pragma unroll
            for (unsigned r = 0; r < kMaxCluster; ++r) {
                const double x = cluster.map_shared_rank(&s_part[par][0], r < csize ? r : crank)[lane];   // (always a valid rank)
                t[r] = r < csize ? x : 0.0;
            }
            double v = 0;
#pragma unroll
            for (unsigned r = 0; r < kMaxCluster; ++r) v += t[r];
            s_final[lane] = v;
            if (lane < 29) s_st.sums[lane] = v;
            __syncwarp();
            odometry_finalize(a, &s_st, per_iter, s_final, s_scratch);
        }
        __syncthreads();
        if (s_st.status | s_st.level_done[a.level]) break;   // identical in every CTA
    }
    cluster.sync();                  // nobody leaves while a peer may still read its shared memory
    if (crank == 0) {
        for (int k = threadIdx.x; k < kStateWords; k += kLevelThreads)
            reinterpret_cast<unsigned long long*>(a.st)[k] = reinterpret_cast<const unsigned long long*>(&s_st)[k];
        publish_state(a, &s_st);
    }
}

// ------------------------------------------------------------- host side

static int launch_image_1d(int64_t n) { return (int)ceil_div(n, kOT); }

static int check_image(const char* who, const void* src, const void* dst, int rows, int cols) {
    O3DB_REQUIRE(rows > 0 && cols > 0 && (int64_t)rows * cols < INT_MAX / 4, "%s: invalid shape (%d, %d)", who, rows, cols);
    O3DB_REQUIRE(src != nullptr && dst != nullptr, "%s: null image", who);
    return O3DB_OK;
}

static int clip_transform(const void* src, int dtype, int rows, int cols, float scale, float min_value, float max_value,
                          float clip_fill, float* dst, cudaStream_t st) {
    const int64_t n = (int64_t)rows * cols;
    if (dtype == O3DB_DEPTH_U16)
        clip_transform_kernel<uint16_t><<<launch_image_1d(n), kOT, 0, st>>>((const uint16_t*)src, n, scale, min_value,
                                                                          max_value, clip_fill, dst);
    else
        clip_transform_kernel<float><<<launch_image_1d(n), kOT, 0, st>>>((const float*)src, n, scale, min_value, max_value,
                                                                       clip_fill, dst);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

static Cam image_cam(const double* K) {
    const double eye[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    return make_cam(K, eye, 1.0f);
}

struct Level {
    int rows = 0, cols = 0;
    double K[9];
    float *sv = nullptr, *tv = nullptr, *tn = nullptr;
};

}  // namespace o3db

using namespace o3db;

extern "C" {

int o3db_image_clip_transform(const void* src_dev, int depth_dtype, int rows, int cols, float scale, float min_value,
                              float max_value, float clip_fill, float* dst_dev, void* stream) {
    int rc = check_image("ClipTransform", src_dev, dst_dev, rows, cols);
    if (rc) return rc;
    O3DB_REQUIRE(depth_dtype == O3DB_DEPTH_U16 || depth_dtype == O3DB_DEPTH_F32, "ClipTransform: dtype must be UInt16 or Float32");
    O3DB_REQUIRE(!(scale < 0 || min_value < 0 || max_value < 0),
                 "Expected positive scale, min_value, and max_value, but got %g, %g, and %g", scale, min_value, max_value);
    return clip_transform(src_dev, depth_dtype, rows, cols, scale, min_value, max_value, clip_fill, dst_dev, (cudaStream_t)stream);
}

int o3db_image_pyr_down_depth(const float* src_dev, int rows, int cols, float diff_threshold, float invalid_fill,
                              float* dst_dev, void* stream) {
    int rc = check_image("PyrDownDepth", src_dev, dst_dev, rows, cols);
    if (rc) return rc;
    if (rows / 2 == 0 || cols / 2 == 0) return O3DB_OK;
    pyr_down_depth_kernel<<<launch_image_1d((int64_t)(rows / 2) * (cols / 2)), kOT, 0, (cudaStream_t)stream>>>(
            src_dev, rows, cols, diff_threshold, invalid_fill, dst_dev);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

int o3db_image_create_vertex_map(const float* depth_dev, int rows, int cols, const double K[9], float invalid_fill,
                                 float* vertex_dev, void* stream) {
    int rc = check_image("CreateVertexMap", depth_dev, vertex_dev, rows, cols);
    if (rc) return rc;
    O3DB_REQUIRE(K != nullptr, "CreateVertexMap: null intrinsics");
    create_vertex_map_kernel<<<launch_image_1d((int64_t)rows * cols), kOT, 0, (cudaStream_t)stream>>>(
            depth_dev, rows, cols, image_cam(K), invalid_fill, vertex_dev);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

int o3db_image_create_normal_map(const float* vertex_dev, int rows, int cols, float invalid_fill, float* normal_dev,
                                 void* stream) {
    int rc = check_image("CreateNormalMap", vertex_dev, normal_dev, rows, cols);
    if (rc) return rc;
    create_normal_map_kernel<<<launch_image_1d((int64_t)rows * cols), kOT, 0, (cudaStream_t)stream>>>(
            vertex_dev, rows, cols, invalid_fill, normal_dev);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

int o3db_image_filter_bilateral(const float* src_dev, int rows, int cols, int kernel_size, float value_sigma,
                                float dist_sigma, float* dst_dev, void* stream) {
    int rc = check_image("FilterBilateral", src_dev, dst_dev, rows, cols);
    if (rc) return rc;
    O3DB_REQUIRE(kernel_size >= 3, "Kernel size must be >= 3, but got %d.", kernel_size);   // Image.cpp:251-253
    filter_bilateral_kernel<<<launch_image_1d((int64_t)rows * cols), kOT, 0, (cudaStream_t)stream>>>(
            src_dev, rows, cols, kernel_size / 2, 2.0f * (value_sigma * value_sigma), 2.0f * (dist_sigma * dist_sigma),
            dst_dev);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

}  // extern "C"

namespace o3db {

struct OdoScratch {
    OdoState* st = nullptr;
    OdoState* h_st = nullptr;
    double* partials = nullptr;
    double* per_iter = nullptr;
    double* delta = nullptr;
    int blocks = 1;
};

static void odo_scratch_free(OdoScratch* s, cudaStream_t st, bool pinned_idle = false) {
    // the pinned block may still feed / receive an async copy (not when the result arrived by publish_state: its
    // token is the last store the device makes to the block)
    if (s->h_st && !pinned_idle) cudaStreamSynchronize(st);
    if (s->st) cudaFreeAsync(s->st, st);
    if (s->partials) cudaFreeAsync(s->partials, st);
    if (s->per_iter) cudaFreeAsync(s->per_iter, st);
    if (s->delta) cudaFreeAsync(s->delta, st);
    if (s->h_st) pinned_release(s->h_st);
    *s = OdoScratch{};
}

// device_init: the first pyramid launch writes the initial state (LevelArgs::init_state) and every launch overwrites
// its own partial rows before reading them, so nothing has to be copied or cleared on the stream.
static int odo_scratch_alloc(OdoScratch* s, int64_t pixels, int log_entries, const double* T, cudaStream_t st,
                             bool device_init = false) {
    configure_memory_pool();
    s->blocks = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(pixels, kThreads), (int64_t)num_sms() * ODO_BLOCKS_PER_SM));
    static_assert(sizeof(OdoState) <= 4096 - 64, "OdoState and the token must fit a pinned block");
    static_assert(kStateWords <= kHostTokenWord && (kHostTokenWord + 1) * sizeof(unsigned long long) <= 4096, "token placement");
    O3DB_CUDA_CHECK(cudaMallocAsync(&s->st, sizeof(OdoState), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&s->partials, (size_t)s->blocks * kSumStride * sizeof(double), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&s->per_iter, (size_t)std::max(1, log_entries) * 2 * sizeof(double), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&s->delta, 16 * sizeof(double), st));
    s->h_st = (OdoState*)pinned_acquire(sizeof(OdoState));
    if (!s->h_st) {
        set_last_error("pinned host allocation failed");
        return O3DB_ERR_CUDA;
    }
    if (device_init) return O3DB_OK;
    OdoState h{};
    for (int i = 0; i < 16; ++i) h.T[i] = T[i];
    h.res_rmse = 0.0;       // RGBDOdometry.cpp:165 OdometryResult(trans, /*prev rmse*/ 0.0, /*prev fitness*/ 1.0)
    h.res_fitness = 1.0;
    memcpy(s->h_st, &h, sizeof(h));
    O3DB_CUDA_CHECK(cudaMemcpyAsync(s->st, s->h_st, sizeof(OdoState), cudaMemcpyHostToDevice, st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(s->partials, 0, (size_t)s->blocks * kSumStride * sizeof(double), st));
    return O3DB_OK;
}

static int odo_status_to_rc(int status) {
    if (status == 1) {
        set_last_error("Singular 6x6 linear system detected, tracking failed.");
        return O3DB_ERR_SINGULAR;
    }
    if (status == 2) {
        set_last_error("Invalid inlier_count value 0, must be > 0.");   // RGBDOdometry.cpp:449-452
        return O3DB_ERR_NO_INLIERS;
    }
    return O3DB_OK;
}

// Cluster size the level-resident kernel runs with on the current device: 16 CTAs (non-portable size, one GPC) when
// the device can co-schedule such a cluster, else 8, else 0 = the per-iteration kernel everywhere.  Decided once per
// device.  O3DB_ODO_LEVEL_CLUSTER = 0 | 8 | 16 caps it (measurements, fallback).
static int level_cluster_size() {
    static std::mutex mu;
    static int cached[64];
    static bool known[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 0;
    std::lock_guard<std::mutex> lk(mu);
    if (known[dev]) return cached[dev];
    int cap = 16;
    if (const char* e = getenv("O3DB_ODO_LEVEL_CLUSTER")) cap = atoi(e);
    int chosen = 0;
    for (int c : {16, 8}) {
        if (c > cap) continue;
        if (c > 8 && (cudaFuncSetAttribute(odometry_level_kernel<1>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
                      cudaFuncSetAttribute(odometry_level_kernel<3>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
                      cudaFuncSetAttribute(odometry_level_kernel<4>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess)) {
            cudaGetLastError();
            continue;
        }
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3((unsigned)c);
        cfg.blockDim = dim3(kLevelThreads);
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = (unsigned)c;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        int clusters = 0;
        if (cudaOccupancyMaxActiveClusters(&clusters, odometry_level_kernel<4>, &cfg) == cudaSuccess && clusters >= 1) {
            chosen = c;
            break;
        }
        cudaGetLastError();
    }
    cached[dev] = chosen;
    known[dev] = true;
    if (getenv("O3DB_ODO_VERBOSE")) fprintf(stderr, "[o3db] odometry level-resident kernel: cluster of %d CTAs on device %d\n", chosen, dev);
    return chosen;
}

// Pixels per thread up to which a level runs in the level-resident kernel: beyond that the cluster's 8 - 16 SMs are
// slower at the pixel loop than the whole GPU is at the per-iteration kernel's fixed cost.
static int level_pixels_per_thread() {
    static const int v = [] {
        const char* e = getenv("O3DB_ODO_LEVEL_PX_PER_THREAD");
        return e ? atoi(e) : 12;
    }();
    return v;
}

// O3DB_ODO_NO_ZERO_COPY=1: read the result back with a copy + stream synchronisation (measurements, fallback)
static bool zero_copy_result() {
    static const bool v = getenv("O3DB_ODO_NO_ZERO_COPY") == nullptr;
    return v;
}

static cudaError_t launch_level(const OdoArgs& a, int max_iteration, int cluster, cudaStream_t st) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)cluster);
    cfg.blockDim = dim3(kLevelThreads);
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = (unsigned)cluster;
    attr[1].val.clusterDim.y = 1;
    attr[1].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 2;
    static const int batch = [] {       // pixels in flight per thread (O3DB_ODO_LEVEL_BATCH = 1 | 3 | 4: measurements)
        const char* v = getenv("O3DB_ODO_LEVEL_BATCH");
        return v ? atoi(v) : 3;
    }();
    if (batch <= 1) return cudaLaunchKernelEx(&cfg, odometry_level_kernel<1>, a, max_iteration);
    if (batch >= 4) return cudaLaunchKernelEx(&cfg, odometry_level_kernel<4>, a, max_iteration);
    return cudaLaunchKernelEx(&cfg, odometry_level_kernel<3>, a, max_iteration);
}

}  // namespace o3db

extern "C" {

int o3db_compute_odometry_result_point_to_plane(const float* source_vertex_map_dev, const float* target_vertex_map_dev,
                                                const float* target_normal_map_dev, int rows, int cols,
                                                const double K[9], const double init_source_to_target[16],
                                                float depth_outlier_trunc, float depth_huber_delta,
                                                double delta_transformation_host[16], double* inlier_rmse_host,
                                                double* fitness_host, double* sums29_host, void* stream) {
    O3DB_REQUIRE(source_vertex_map_dev && target_vertex_map_dev && target_normal_map_dev,
                 "o3db_compute_odometry_result_point_to_plane: null map");
    O3DB_REQUIRE(rows > 0 && cols > 0 && K && init_source_to_target && delta_transformation_host,
                 "o3db_compute_odometry_result_point_to_plane: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    OdoScratch s;
    int rc = odo_scratch_alloc(&s, (int64_t)rows * cols, 1, init_source_to_target, st);
    if (rc) {
        odo_scratch_free(&s, st);
        return rc;
    }
    OdoArgs a{};
    a.sv = source_vertex_map_dev;
    a.tv = target_vertex_map_dev;
    a.tn = target_normal_map_dev;
    a.rows = rows;
    a.cols = cols;
    a.level = 0;
    a.fx = (float)K[0];
    a.fy = (float)K[4];
    a.cx = (float)K[2];
    a.cy = (float)K[5];
    a.trunc = depth_outlier_trunc;
    a.huber_delta = depth_huber_delta;
    a.partials = s.partials;
    a.st = s.st;
    a.standalone = 1;
    a.delta_out = s.delta;
    odometry_iteration_kernel<<<s.blocks, kThreads, 0, st>>>(a);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(s.h_st, s.st, sizeof(OdoState), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(delta_transformation_host, s.delta, 16 * sizeof(double), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
        set_last_error("o3db_compute_odometry_result_point_to_plane: %s", cudaGetErrorString(e));
        odo_scratch_free(&s, st);
        return O3DB_ERR_CUDA;
    }
    rc = odo_status_to_rc(s.h_st->status);
    if (inlier_rmse_host) *inlier_rmse_host = s.h_st->res_rmse;
    if (fitness_host) *fitness_host = s.h_st->res_fitness;
    if (sums29_host) memcpy(sums29_host, s.h_st->sums, 29 * sizeof(double));
    odo_scratch_free(&s, st);
    return rc;
}

int o3db_rgbd_odometry_multi_scale_point_to_plane(const void* source_depth_dev, int source_dtype,
                                                  const void* target_depth_dev, int target_dtype, int rows, int cols,
                                                  const double K[9], const double init_source_to_target[16],
                                                  float depth_scale, float depth_max,
                                                  const o3db_odometry_criteria* criteria, int num_levels,
                                                  float depth_outlier_trunc, float depth_huber_delta,
                                                  o3db_odometry_result* result_host, double* per_iteration_host,
                                                  void* stream) {
    O3DB_REQUIRE(result_host != nullptr, "o3db_rgbd_odometry_multi_scale_point_to_plane: null result");
    O3DB_REQUIRE(source_depth_dev && target_depth_dev && K && init_source_to_target && criteria,
                 "o3db_rgbd_odometry_multi_scale_point_to_plane: null argument");
    O3DB_REQUIRE(num_levels >= 1 && num_levels <= kMaxLevels, "o3db_rgbd_odometry_multi_scale_point_to_plane: 1..%d levels",
                 kMaxLevels);
    O3DB_REQUIRE(rows > 0 && cols > 0 && (rows >> (num_levels - 1)) > 1 && (cols >> (num_levels - 1)) > 1,
                 "o3db_rgbd_odometry_multi_scale_point_to_plane: image %dx%d too small for %d levels", cols, rows, num_levels);
    for (int d : {source_dtype, target_dtype})
        O3DB_REQUIRE(d == O3DB_DEPTH_U16 || d == O3DB_DEPTH_F32, "depth images must be UInt16 or Float32");
    cudaStream_t st = (cudaStream_t)stream;
    configure_memory_pool();
    const float nanf_ = nanf("");
    int total_iters = 0;
    for (int i = 0; i < num_levels; ++i) {
        O3DB_REQUIRE(criteria[i].max_iteration >= 0, "max_iteration must be non-negative");
        total_iters += criteria[i].max_iteration;
    }
    // one allocation for the whole pyramid
    std::vector<Level> lv(num_levels);
    size_t floats = 0;
    {
        int r = rows, c = cols;
        for (int i = 0; i < num_levels; ++i, r /= 2, c /= 2) floats += (size_t)r * c * 9;   // sv, tv, tn
    }
    const size_t full = (size_t)rows * cols;
    float* pool = nullptr;
    O3DB_CUDA_CHECK(cudaMallocAsync(&pool, (floats + full * 4 + full * 3) * sizeof(float), st));
    float* src_d = pool + floats;          // current source / target depth, ping-pong halves, smoothed target, its vertices
    float* tgt_d = src_d + full;
    float* tmp = tgt_d + full;
    float* smooth = tmp + full;
    OdoScratch s;
    int rc = O3DB_OK;
#define ODO_TRY(expr)                  \
    do {                               \
        if (rc == O3DB_OK) rc = (expr); \
    } while (0)
    ODO_TRY(odo_scratch_alloc(&s, full, total_iters, init_source_to_target, st, /*device_init=*/true));
    // RGBDOdometry.cpp:84-88 ClipTransform(depth_scale, 0, depth_max, NAN), both frames in one launch
    if (rc == O3DB_OK) {
        const int64_t npx = (int64_t)rows * cols;
        const dim3 grid((unsigned)launch_image_1d(npx), 2);
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = grid;
        cfg.blockDim = dim3(kOT);
        cfg.stream = st;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        cudaError_t e;
        const bool su = source_dtype == O3DB_DEPTH_U16, tu = target_dtype == O3DB_DEPTH_U16;
#define ODO_CLIP(S, T)                                                                                                   \
    e = cudaLaunchKernelEx(&cfg, clip_transform_pair_kernel<S, T>, (const S*)source_depth_dev, (const T*)target_depth_dev, npx, \
                           depth_scale, 0.0f, depth_max, nanf_, src_d, tgt_d)
        if (su && tu) ODO_CLIP(uint16_t, uint16_t);
        else if (su) ODO_CLIP(uint16_t, float);
        else if (tu) ODO_CLIP(float, uint16_t);
        else ODO_CLIP(float, float);
#undef ODO_CLIP
        count_launch();
        if (e != cudaSuccess) {
            set_last_error("clip_transform_pair_kernel launch failed: %s", cudaGetErrorString(e));
            rc = O3DB_ERR_CUDA;
        }
    }
    double Kp[9];
    memcpy(Kp, K, sizeof(Kp));
    {
        float* cursor = pool;
        int r = rows, c = cols;
        for (int i = 0; i < num_levels && rc == O3DB_OK; ++i) {   // :132-163, one fused launch per level
            Level& L = lv[num_levels - 1 - i];
            L.rows = r;
            L.cols = c;
            memcpy(L.K, Kp, sizeof(Kp));
            L.sv = cursor;
            L.tv = cursor + (size_t)r * c * 3;
            L.tn = cursor + (size_t)r * c * 6;
            cursor += (size_t)r * c * 9;
            const bool last = i == num_levels - 1;
            LevelArgs la{};
            la.src_d = src_d;
            la.tgt_d = tgt_d;
            la.rows = r;
            la.cols = c;
            const double eye[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
            la.ti = make_cam(Kp, eye, 1.0f);
            la.invalid_fill = nanf_;
            la.val2 = 2.0f * 5.0f * 5.0f;            // FilterBilateral(5, 5, 10): as o3db_image_filter_bilateral
            la.pos2 = 2.0f * 10.0f * 10.0f;
            la.depth_diff = depth_outlier_trunc * 2;
            la.sv = L.sv;
            la.tv = L.tv;
            la.tn = L.tn;
            // the next level's images go to the two spare buffers (tmp, smooth), then the roles swap
            la.src_next = last ? nullptr : tmp;
            la.tgt_next = last ? nullptr : smooth;
            la.init_state = i == 0 ? s.st : nullptr;
            for (int k = 0; k < 16; ++k) la.init_T[k] = init_source_to_target[k];
            cudaLaunchConfig_t cfg{};
            cfg.gridDim = dim3((unsigned)ceil_div(c, kTW), (unsigned)ceil_div(r, kTH));
            cfg.blockDim = dim3(kTW * kTH);
            cfg.stream = st;
            cudaLaunchAttribute attr[1];
            attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
            attr[0].val.programmaticStreamSerializationAllowed = 1;
            cfg.attrs = attr;
            cfg.numAttrs = 1;
            static const bool unroll_rows = [] {
                const char* v = getenv("O3DB_ODO_PYR_UNROLL");
                return v ? atoi(v) != 0 : false;
            }();
            const cudaError_t e = unroll_rows ? cudaLaunchKernelEx(&cfg, pyramid_level_kernel<true>, la)
                                              : cudaLaunchKernelEx(&cfg, pyramid_level_kernel<false>, la);
            count_launch();
            if (e != cudaSuccess) {
                set_last_error("pyramid_level_kernel launch failed: %s", cudaGetErrorString(e));
                rc = O3DB_ERR_CUDA;
            }
            if (!last) {
                std::swap(src_d, tmp);
                std::swap(tgt_d, smooth);
                r /= 2;
                c /= 2;
                for (int k = 0; k < 9; ++k) Kp[k] /= 2;   // :159-160
                Kp[8] = 1;
            }
        }
    }
    // which launch is the last one of the track (it publishes the result into pinned host memory)
    int final_level = -1;
    for (int i = 0; i < num_levels; ++i)
        if (criteria[i].max_iteration > 0) final_level = i;
    static std::atomic<unsigned long long> g_token{0};
    const unsigned long long token = ++g_token;
    volatile unsigned long long* h_words = reinterpret_cast<volatile unsigned long long*>(s.h_st);
    const bool zero_copy = zero_copy_result() && final_level >= 0 && rc == O3DB_OK;
    if (zero_copy) h_words[kHostTokenWord] = 0;
    for (int i = 0; i < num_levels && rc == O3DB_OK; ++i) {
        OdoArgs a{};
        a.sv = lv[i].sv;
        a.tv = lv[i].tv;
        a.tn = lv[i].tn;
        a.rows = lv[i].rows;
        a.cols = lv[i].cols;
        a.level = i;
        a.fx = (float)lv[i].K[0];
        a.fy = (float)lv[i].K[4];
        a.cx = (float)lv[i].K[2];
        a.cy = (float)lv[i].K[5];
        a.trunc = depth_outlier_trunc;
        a.huber_delta = depth_huber_delta;
        a.rel_rmse = criteria[i].relative_rmse;
        a.rel_fitness = criteria[i].relative_fitness;
        a.partials = s.partials;
        a.st = s.st;
        a.per_iter = s.per_iter;
        const int64_t pixels = (int64_t)a.rows * a.cols;
        const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(pixels, kThreads), s.blocks));
        const int cluster = level_cluster_size();
        cudaError_t e = cudaSuccess;
        if (cluster > 0 && criteria[i].max_iteration >= 2 &&
            pixels <= (int64_t)cluster * kLevelThreads * level_pixels_per_thread()) {
            // a coarse level: all its iterations in one launch of one thread-block cluster
            if (zero_copy && i == final_level) {
                a.host_out = const_cast<unsigned long long*>(h_words);
                a.host_token = token;
            }
            e = launch_level(a, criteria[i].max_iteration, cluster, st);
            count_launch();
        } else {
            for (int it = 0; it < criteria[i].max_iteration && e == cudaSuccess; ++it) {
                if (zero_copy && i == final_level && it == criteria[i].max_iteration - 1) {
                    a.host_out = const_cast<unsigned long long*>(h_words);
                    a.host_token = token;
                }
                e = launch_pdl_ex(odometry_iteration_kernel, (unsigned)blocks, (unsigned)kThreads, 0, st, a);
                count_launch();
            }
        }
        if (e != cudaSuccess) {
            set_last_error("odometry iteration kernel launch failed: %s", cudaGetErrorString(e));
            rc = O3DB_ERR_CUDA;
        }
    }
    bool published = false;
    if (rc == O3DB_OK) {
        cudaError_t e = cudaSuccess;
        if (zero_copy) {
            // the last launch stores the final state and then the token into the pinned block: spin on it instead of
            // a device-to-host copy + stream synchronisation; the stream is queried now and then so that a failed
            // launch (or a kernel that never published) ends the wait
            const auto t0 = std::chrono::steady_clock::now();
            for (unsigned spins = 1;; ++spins) {
                if (h_words[kHostTokenWord] == token) {
                    published = true;
                    break;
                }
                if ((spins & 0x3fffu) == 0) {
                    e = cudaStreamQuery(st);
                    if (e == cudaSuccess) {
                        published = h_words[kHostTokenWord] == token;
                        break;
                    }
                    if (e != cudaErrorNotReady) break;
                    e = cudaSuccess;
                    if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(30)) {
                        set_last_error("o3db_rgbd_odometry_multi_scale_point_to_plane: the device never published its result");
                        rc = O3DB_ERR_CUDA;
                        break;
                    }
                }
            }
            std::atomic_thread_fence(std::memory_order_acquire);
        }
        if (rc == O3DB_OK && e == cudaSuccess && !published) {
            e = cudaMemcpyAsync(s.h_st, s.st, sizeof(OdoState), cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        }
        if (rc == O3DB_OK && e == cudaSuccess && per_iteration_host && s.h_st->executed > 0) {
            e = cudaMemcpyAsync(per_iteration_host, s.per_iter, (size_t)s.h_st->executed * 2 * sizeof(double),
                                cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        }
        if (e != cudaSuccess) {
            set_last_error("o3db_rgbd_odometry_multi_scale_point_to_plane: %s", cudaGetErrorString(e));
            rc = O3DB_ERR_CUDA;
        } else if (rc == O3DB_OK) {
            memcpy(result_host->transformation, s.h_st->T, sizeof(s.h_st->T));
            result_host->inlier_rmse = s.h_st->res_rmse;
            result_host->fitness = s.h_st->res_fitness;
            result_host->iterations = s.h_st->executed;
            result_host->status = odo_status_to_rc(s.h_st->status);
            rc = result_host->status;
        }
    }
#undef ODO_TRY
    odo_scratch_free(&s, st, /*pinned_idle=*/published);
    cudaFreeAsync(pool, st);
    return rc;
}

}  // extern "C"
