// raycast.cu — VoxelBlockGrid::RayCast for sm_90a (SURVEY.md 8f #4): the step after Integrate in
// the dense-SLAM loop (slam::Model::SynthesizeModelFrame, slam/Model.cpp:38-66).
//
// Reference: VoxelBlockGrid.cpp:328-402 -> kernel::voxel_grid::EstimateRange (VoxelBlockGridImpl.h:310-555)
// + RayCast (VoxelBlockGridImpl.h:578-1120).
//
// EstimateRange.  Upstream runs three passes through a "fragment" buffer: every block's screen rectangle is
// cut into 16x16 fragments (pass 0, atomic append), the range map is initialised (pass 0.5), and every
// fragment pixel does an atomic min/max (pass 1).  The fragments only partition the rectangle, so here one
// warp takes one block: all lanes evaluate the 8 corners (a few dozen flops), then the lanes stride over the
// rectangle's pixels with integer atomics on the f32 bit patterns (all values are positive).  No fragment
// buffer, no host read-back of its fill level, and therefore no overflow mode (upstream: a warning and a
// partial map, :431-468).  Min/max are order-independent: the map is bit-identical to upstream's.
//
// RayCast.  One thread per pixel, 16x16-pixel tiles per CTA so that neighbouring rays walk the same voxel
// blocks (L1/L2 reuse of the 16 KB tsdf block); hash lookups go through the lock-free table of hash.cuh with
// the reference's 1-entry per-ray cache in registers.  Every f32 expression is evaluated in the reference's
// source order with explicit round-to-nearest intrinsics (no FMA contraction) because the march is a chain
// of floor()/truncation decisions: the CPU oracle (compiled with -ffp-contract=off) then agrees bit for bit.
#include <climits>
#include <cmath>

#include "common.cuh"
#include "hash.cuh"
#include "vbg.cuh"

namespace o3db {

static constexpr int kRT = 256;

// GeometryIndexer.h:81-97 Rotate
__device__ __forceinline__ void rotate(const Cam& c, float x, float y, float z, float& xo, float& yo, float& zo) {
    x = mul(x, c.scale);
    y = mul(y, c.scale);
    z = mul(z, c.scale);
    xo = add(add(mul(x, c.e[0][0]), mul(y, c.e[0][1])), mul(z, c.e[0][2]));
    yo = add(add(mul(x, c.e[1][0]), mul(y, c.e[1][1])), mul(z, c.e[1][2]));
    zo = add(add(mul(x, c.e[2][0]), mul(y, c.e[2][1])), mul(z, c.e[2][2]));
}

// ------------------------------------------------------------ EstimateRange

struct RangeArgs {
    const int* coords;       // [n,3] block keys, or null: keys[slots[b]]
    const int* keys;
    const int* slots;
    const int* n_dev;        // device count (frustum mode), or null
    int n;
    Cam w2c;
    int h_down, w_down;
    float down;              // down_factor as f32 (u /= down_factor)
    int resolution;
    float voxel_size, depth_min, depth_max;
    int* range;              // [h_down][w_down][2] f32 bit patterns
};

__global__ void range_init_kernel(float2* __restrict__ range, int n, float depth_max, float depth_min) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) range[i] = make_float2(depth_max, depth_min);   // VoxelBlockGridImpl.h:472-484
}

__global__ void __launch_bounds__(kRT) range_blocks_kernel(RangeArgs a) {
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int n = a.n_dev ? *a.n_dev : a.n;
    for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < n; b += warps) {
        const int* key = a.coords ? a.coords + 3 * (size_t)b : a.keys + 3 * (size_t)a.slots[b];
        const int kx = key[0], ky = key[1], kz = key[2];
        int u_min = a.w_down - 1, v_min = a.h_down - 1, u_max = 0, v_max = 0;
        float z_min = a.depth_max, z_max = a.depth_min;
#pragma unroll
        for (int i = 0; i < 8; ++i) {   // :389-412
            const float xw = mul((float)((long long)(kx + ((i & 1) > 0)) * a.resolution), a.voxel_size);
            const float yw = mul((float)((long long)(ky + ((i & 2) > 0)) * a.resolution), a.voxel_size);
            const float zw = mul((float)((long long)(kz + ((i & 4) > 0)) * a.resolution), a.voxel_size);
            float xc, yc, zc, u, v;
            rigid(a.w2c, xw, yw, zw, xc, yc, zc);
            if (zc <= 0) continue;
            project(a.w2c, xc, yc, zc, u, v);
            u = dvd(u, a.down);
            v = dvd(v, a.down);
            v_min = min((int)floorf(v), v_min);
            v_max = max((int)ceilf(v), v_max);
            u_min = min((int)floorf(u), u_min);
            u_max = max((int)ceilf(u), u_max);
            z_min = fminf(z_min, zc);
            z_max = fmaxf(z_max, zc);
        }
        v_min = max(0, v_min);
        v_max = min(a.h_down - 1, v_max);
        u_min = max(0, u_min);
        u_max = min(a.w_down - 1, u_max);
        if (v_min >= v_max || u_min >= u_max || z_min >= z_max) continue;   // :420
        const int rw = u_max - u_min + 1, cnt = rw * (v_max - v_min + 1);
        const int zlo = __float_as_int(z_min), zhi = __float_as_int(z_max);
        for (int p = lane; p < cnt; p += 32) {   // pass 1 (:497-541)
            const int v = v_min + p / rw, u = u_min + p % rw;
            int* r = a.range + 2 * ((size_t)v * a.w_down + u);
            atomicMin(r, zlo);
            atomicMax(r + 1, zhi);
        }
    }
}

// ------------------------------------------------------------------ RayCast

struct RayArgs {
    Table tab;
    const float* tsdf;
    const uint16_t* weight;
    const uint16_t* color;   // null: no colour rendering
    const float* range;
    Cam c2w, w2c;
    int h, w, h_down, w_down, down;
    int resolution;
    float voxel_size, block_size, depth_scale, weight_threshold, sdf_trunc;
    // outputs (any may be null)
    float* depth;
    float* vertex;
    float* color_out;
    float* normal;
    int64_t* index;
    uint8_t* mask;
    float* ratio;
    float* ratio_dx;
    float* ratio_dy;
    float* ratio_dz;
};

struct BlockCache {   // VoxelBlockGridImpl.h:557-576 MiniVecCache
    int x, y, z, slot;
};

__device__ __forceinline__ int find_block(const RayArgs& a, BlockCache& c, int x, int y, int z) {
    if (c.slot >= 0 && c.x == x && c.y == y && c.z == z) return c.slot;
    unsigned bucket;
    const int s = probe<false>(a.tab, nullptr, 0, x, y, z, &bucket);
    if (s < 0) return -1;
    c.x = x;
    c.y = y;
    c.z = z;
    c.slot = s;
    return s;
}

__device__ __forceinline__ int sign_of(int x) { return (x > 0) ? 1 : ((x < 0) ? -1 : 0); }

template <bool NEIGHBORS>
__global__ void __launch_bounds__(kRT) ray_cast_kernel(RayArgs a) {
    // 16 x 16 pixel tile per CTA
    const int tiles_x = (a.w + 15) >> 4;
    const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x;
    const int x = (tx << 4) + (threadIdx.x & 15), y = (ty << 4) + (threadIdx.x >> 4);
    if (x >= a.w || y >= a.h) return;
    const size_t pix = (size_t)y * a.w + x;

    // zero-initialise every requested output (:862-947)
    if (a.depth) a.depth[pix] = 0.f;
    if (a.vertex) a.vertex[3 * pix] = a.vertex[3 * pix + 1] = a.vertex[3 * pix + 2] = 0.f;
    if (a.normal) a.normal[3 * pix] = a.normal[3 * pix + 1] = a.normal[3 * pix + 2] = 0.f;
    if (a.color_out) a.color_out[3 * pix] = a.color_out[3 * pix + 1] = a.color_out[3 * pix + 2] = 0.f;
    if (NEIGHBORS) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (a.mask) a.mask[8 * pix + i] = 0;
            if (a.index) a.index[8 * pix + i] = 0;
            if (a.ratio) a.ratio[8 * pix + i] = 0.f;
            if (a.ratio_dx) a.ratio_dx[8 * pix + i] = 0.f;
            if (a.ratio_dy) a.ratio_dy[8 * pix + i] = 0.f;
            if (a.ratio_dz) a.ratio_dz[8 * pix + i] = 0.f;
        }
    }

    // (x / down, y / down) clamped to the map: with an image size that is not a multiple of the down factor
    // upstream indexes one cell past the last row / column (:851-852)
    const float* rng = a.range + 2 * ((size_t)min(y / a.down, a.h_down - 1) * a.w_down + min(x / a.down, a.w_down - 1));
    float t = rng[0];
    const float t_max = rng[1];
    if (t >= t_max) return;

    float x_c, y_c, z_c, x_g, y_g, z_g, x_o, y_o, z_o;
    float t_prev = t;
    float tsdf_prev = -1.0f, tsdf = 1.0f;
    rigid(a.c2w, 0.f, 0.f, 0.f, x_o, y_o, z_o);                       // camera origin
    unproject(a.c2w, (float)x, (float)y, 1.0f, x_c, y_c, z_c);        // direction
    rigid(a.c2w, x_c, y_c, z_c, x_g, y_g, z_g);
    const float x_d = sub(x_g, x_o), y_d = sub(y_g, y_o), z_d = sub(z_g, z_o);

    const int res = a.resolution, res2 = res * res;
    const int64_t res3 = (int64_t)res2 * res;
    BlockCache cache{0, 0, 0, -1};
    bool surface_found = false;
    while (t < t_max) {
        // GetLinearIdxAtT (:795-833)
        const float xg = add(x_o, mul(t, x_d)), yg = add(y_o, mul(t, y_d)), zg = add(z_o, mul(t, z_d));
        const int x_b = (int)floorf(dvd(xg, a.block_size));
        const int y_b = (int)floorf(dvd(yg, a.block_size));
        const int z_b = (int)floorf(dvd(zg, a.block_size));
        const int blk = find_block(a, cache, x_b, y_b, z_b);
        if (blk < 0) {
            t_prev = t;
            t = add(t, a.block_size);
        } else {
            // index_t((x_g - x_b * block_size) / voxel_size) (:826-828) can round up to `res` when x_g sits a
            // rounding error below a block face; upstream then reads the next row of the block (or past the
            // buffer).  Clamped to res-1 here — the one deliberate deviation (DESIGN.md).
            const int x_v = min((int)dvd(sub(xg, mul((float)x_b, a.block_size)), a.voxel_size), res - 1);
            const int y_v = min((int)dvd(sub(yg, mul((float)y_b, a.block_size)), a.voxel_size), res - 1);
            const int z_v = min((int)dvd(sub(zg, mul((float)z_b, a.block_size)), a.voxel_size), res - 1);
            const int64_t lin = blk * res3 + z_v * res2 + y_v * res + x_v;
            tsdf_prev = tsdf;
            tsdf = __ldg(&a.tsdf[lin]);
            const float w = (float)__ldg(&a.weight[lin]);
            if (tsdf_prev > 0 && w >= a.weight_threshold && tsdf <= 0) {
                surface_found = true;
                break;
            }
            t_prev = t;
            const float delta = mul(tsdf, a.sdf_trunc);
            t = add(t, delta < a.voxel_size ? a.voxel_size : delta);
        }
    }
    if (!surface_found) return;

    const float t_intersect = dvd(sub(mul(t, tsdf_prev), mul(t_prev, tsdf)), sub(tsdf_prev, tsdf));
    x_g = add(x_o, mul(t_intersect, x_d));
    y_g = add(y_o, mul(t_intersect, y_d));
    z_g = add(z_o, mul(t_intersect, z_d));
    if (a.depth) a.depth[pix] = mul(t_intersect, a.depth_scale);
    if (a.vertex) {
        float vx, vy, vz;
        rigid(a.w2c, x_g, y_g, z_g, vx, vy, vz);
        a.vertex[3 * pix] = vx;
        a.vertex[3 * pix + 1] = vy;
        a.vertex[3 * pix + 2] = vz;
    }
    if (!NEIGHBORS) return;

    // trilinear neighbourhood (:1002-1113)
    const int x_b = (int)floorf(dvd(x_g, a.block_size));
    const int y_b = (int)floorf(dvd(y_g, a.block_size));
    const int z_b = (int)floorf(dvd(z_g, a.block_size));
    const float x_v = dvd(sub(x_g, mul((float)x_b, a.block_size)), a.voxel_size);
    const float y_v = dvd(sub(y_g, mul((float)y_b, a.block_size)), a.voxel_size);
    const float z_v = dvd(sub(z_g, mul((float)z_b, a.block_size)), a.voxel_size);
    const int block_buf_idx = find_block(a, cache, x_b, y_b, z_b);
    if (block_buf_idx < 0) return;
    const int x_vf = (int)floorf(x_v), y_vf = (int)floorf(y_v), z_vf = (int)floorf(z_v);
    const float ratio_x = sub(x_v, (float)x_vf), ratio_y = sub(y_v, (float)y_vf), ratio_z = sub(z_v, (float)z_vf);

    float sum_r = 0.f;
    float nrm[3] = {0.f, 0.f, 0.f}, col[3] = {0.f, 0.f, 0.f};
#pragma unroll 1
    for (int k = 0; k < 8; ++k) {
        const int dx_v = (k & 1) > 0 ? 1 : 0, dy_v = (k & 2) > 0 ? 1 : 0, dz_v = (k & 4) > 0 ? 1 : 0;
        // GetLinearIdxAtP (:748-793)
        int64_t lin;
        {
            const int xv = x_vf + dx_v, yv = y_vf + dy_v, zv = z_vf + dz_v;
            const int x_vn = (xv + res) % res, y_vn = (yv + res) % res, z_vn = (zv + res) % res;
            const int dx_b = sign_of(xv - x_vn), dy_b = sign_of(yv - y_vn), dz_b = sign_of(zv - z_vn);
            if (dx_b == 0 && dy_b == 0 && dz_b == 0) {
                lin = block_buf_idx * res3 + zv * res2 + yv * res + xv;
            } else {
                const int nb = find_block(a, cache, x_b + dx_b, y_b + dy_b, z_b + dz_b);
                lin = nb < 0 ? -1 : nb * res3 + z_vn * res2 + y_vn * res + x_vn;
            }
        }
        if (lin >= 0 && __ldg(&a.weight[lin]) > 0) {
            const float rx = add(mul((float)dx_v, ratio_x), mul((float)(1 - dx_v), sub(1.0f, ratio_x)));
            const float ry = add(mul((float)dy_v, ratio_y), mul((float)(1 - dy_v), sub(1.0f, ratio_y)));
            const float rz = add(mul((float)dz_v, ratio_z), mul((float)(1 - dz_v), sub(1.0f, ratio_z)));
            const float r = mul(mul(rx, ry), rz);
            if (a.ratio) a.ratio[8 * pix + k] = r;
            if (a.mask) a.mask[8 * pix + k] = 1;
            if (a.index) a.index[8 * pix + k] = lin;
            const float tsdf_k = __ldg(&a.tsdf[lin]);
            const float r_dx = mul(mul(ry, rz), (float)(2 * dx_v - 1));
            const float r_dy = mul(mul(rx, rz), (float)(2 * dy_v - 1));
            const float r_dz = mul(mul(rx, ry), (float)(2 * dz_v - 1));
            if (a.ratio_dx) a.ratio_dx[8 * pix + k] = r_dx;
            if (a.ratio_dy) a.ratio_dy[8 * pix + k] = r_dy;
            if (a.ratio_dz) a.ratio_dz[8 * pix + k] = r_dz;
            nrm[0] = add(nrm[0], mul(r_dx, tsdf_k));
            nrm[1] = add(nrm[1], mul(r_dy, tsdf_k));
            nrm[2] = add(nrm[2], mul(r_dz, tsdf_k));
            if (a.color) {
                const uint16_t* c = a.color + 3 * lin;
                col[0] = add(col[0], mul(r, (float)__ldg(c)));
                col[1] = add(col[1], mul(r, (float)__ldg(c + 1)));
                col[2] = add(col[2], mul(r, (float)__ldg(c + 2)));
            }
            sum_r = add(sum_r, r);
        }
    }
    if (sum_r > 0) {
        sum_r = (float)((double)sum_r * 255.0);   // :1090 `sum_r *= 255.0` (double literal)
        if (a.color && a.color_out) {
            col[0] = dvd(col[0], sum_r);
            col[1] = dvd(col[1], sum_r);
            col[2] = dvd(col[2], sum_r);
        }
        if (a.normal) {
            float norm = __fsqrt_rn(add(add(mul(nrm[0], nrm[0]), mul(nrm[1], nrm[1])), mul(nrm[2], nrm[2])));
            norm = fmaxf(norm, 1e-5f);
            rotate(a.w2c, dvd(-nrm[0], norm), dvd(-nrm[1], norm), dvd(-nrm[2], norm), nrm[0], nrm[1], nrm[2]);
        }
    }
    if (a.color && a.color_out) {
        a.color_out[3 * pix] = col[0];
        a.color_out[3 * pix + 1] = col[1];
        a.color_out[3 * pix + 2] = col[2];
    }
    if (a.normal) {
        a.normal[3 * pix] = nrm[0];
        a.normal[3 * pix + 1] = nrm[1];
        a.normal[3 * pix + 2] = nrm[2];
    }
}

static int launch_estimate_range(o3db_vbg* v, const int32_t* coords, int64_t n, const double* K, const double* E,
                                 int height, int width, int down, float depth_min, float depth_max, float* range,
                                 cudaStream_t st) {
    const int h_down = height / down, w_down = width / down;
    const int cells = h_down * w_down;
    range_init_kernel<<<(unsigned)ceil_div(cells, kRT), kRT, 0, st>>>((float2*)range, cells, depth_max, depth_min);
    O3DB_LAUNCH_CHECK();
    RangeArgs a{};
    a.coords = coords;
    a.keys = v->map.keys.get();
    a.slots = v->frame_slots.get();
    a.n_dev = coords ? nullptr : &v->status->frame_count;    // block count of the last fused frame
    a.n = (int)n;
    a.w2c = make_cam(K, E, 1.0f);
    a.h_down = h_down;
    a.w_down = w_down;
    a.down = (float)down;
    a.resolution = v->resolution;
    a.voxel_size = v->voxel_size;
    a.depth_min = depth_min;
    a.depth_max = depth_max;
    a.range = (int*)range;
    const int64_t work = coords ? n : v->frustum_cap;
    if (work > 0) {
        const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(work * 32, kRT), (int64_t)num_sms() * 8));
        range_blocks_kernel<<<blocks, kRT, 0, st>>>(a);
        O3DB_LAUNCH_CHECK();
    }
    return O3DB_OK;
}

}  // namespace o3db

using namespace o3db;

extern "C" {

static int check_camera_args(const char* who, const o3db_vbg* v, const double* K, const double* E, int height,
                             int width, int down) {
    O3DB_REQUIRE(v != nullptr, "%s: null voxel grid", who);
    O3DB_REQUIRE(K != nullptr && E != nullptr, "%s: null intrinsic / extrinsic", who);
    O3DB_REQUIRE(height > 0 && width > 0, "%s: bad image size %dx%d", who, width, height);
    O3DB_REQUIRE(down >= 1 && height / down > 0 && width / down > 0, "%s: bad range_map_down_factor %d", who, down);
    return O3DB_OK;
}

int o3db_vbg_estimate_range(o3db_vbg* v, const int32_t* block_coords_dev, int64_t num_blocks, const double K[9],
                            const double E[16], int height, int width, int down_factor, float depth_min,
                            float depth_max, float* range_dev, void* stream) {
    int rc = check_camera_args("o3db_vbg_estimate_range", v, K, E, height, width, down_factor);
    if (rc) return rc;
    O3DB_REQUIRE(range_dev != nullptr, "o3db_vbg_estimate_range: null output");
    O3DB_REQUIRE(num_blocks >= 0 && num_blocks < INT_MAX, "o3db_vbg_estimate_range: bad block count");
    O3DB_REQUIRE(block_coords_dev != nullptr || v->frame_slots,
                 "o3db_vbg_estimate_range: no integrated frame to take the frustum from");
    return launch_estimate_range(v, block_coords_dev, num_blocks, K, E, height, width, down_factor, depth_min, depth_max,
                                 range_dev, (cudaStream_t)stream);
}

int o3db_vbg_ray_cast(o3db_vbg* v, const int32_t* block_coords_dev, int64_t num_blocks, const double K[9],
                      const double E[16], int width, int height, const o3db_raycast_outputs* out, float depth_scale,
                      float depth_min, float depth_max, float weight_threshold, float trunc_voxel_multiplier,
                      int range_map_down_factor, float* range_dev, void* stream) {
    int rc = check_camera_args("o3db_vbg_ray_cast", v, K, E, height, width, range_map_down_factor);
    if (rc) return rc;
    O3DB_REQUIRE(out != nullptr, "o3db_vbg_ray_cast: null outputs");
    O3DB_REQUIRE(num_blocks >= 0 && num_blocks < INT_MAX, "o3db_vbg_ray_cast: bad block count");
    O3DB_REQUIRE(block_coords_dev != nullptr || v->frame_slots,
                 "o3db_vbg_ray_cast: no integrated frame to take the frustum from");
    cudaStream_t st = (cudaStream_t)stream;
    const int h_down = height / range_map_down_factor, w_down = width / range_map_down_factor;
    DevPtr<float> own_range;   // when the caller passes no range map
    if (!range_dev) {
        rc = dev_alloc(own_range, (size_t)h_down * w_down * 2, st);
        if (rc) return rc;
    }
    float* range = range_dev ? range_dev : own_range.get();
    rc = launch_estimate_range(v, block_coords_dev, num_blocks, K, E, height, width, range_map_down_factor, depth_min,
                               depth_max, range, st);
    if (rc) return rc;
    RayArgs a{};
    a.tab = Table{v->map.table.get(), v->map.nbuckets - 1, v->map.keys.get()};
    a.tsdf = v->map.tsdf.get();
    a.weight = v->map.weight.get();
    a.color = (v->with_color && out->color) ? v->map.color.get() : nullptr;
    a.range = range;
    double Einv[16];
    inverse_transformation(E, Einv);   // VoxelBlockGridImpl.h:721-722
    a.c2w = make_cam(K, Einv, 1.0f);
    a.w2c = make_cam(K, E, 1.0f);
    a.h = height;
    a.w = width;
    a.h_down = h_down;
    a.w_down = w_down;
    a.down = range_map_down_factor;
    a.resolution = v->resolution;
    a.voxel_size = v->voxel_size;
    a.block_size = v->voxel_size * (float)v->resolution;
    a.depth_scale = depth_scale;
    a.weight_threshold = weight_threshold;
    a.sdf_trunc = v->voxel_size * trunc_voxel_multiplier;
    a.depth = out->depth;
    a.vertex = out->vertex;
    a.color_out = out->color;
    a.normal = out->normal;
    a.index = out->index;
    a.mask = out->mask;
    a.ratio = out->interp_ratio;
    a.ratio_dx = out->interp_ratio_dx;
    a.ratio_dy = out->interp_ratio_dy;
    a.ratio_dz = out->interp_ratio_dz;
    const bool neighbors = a.color || a.normal || a.mask || a.index || a.ratio || a.ratio_dx || a.ratio_dy ||
                           a.ratio_dz;   // :707-714 visit_neighbors
    const unsigned tiles = (unsigned)(((width + 15) / 16) * ((height + 15) / 16));
    if (neighbors) ray_cast_kernel<true><<<tiles, kRT, 0, st>>>(a);
    else ray_cast_kernel<false><<<tiles, kRT, 0, st>>>(a);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

}  // extern "C"
