// vbg.cuh — state of the voxel block grid handle and the f32 camera geometry shared by
// tsdf.cu (touch / integrate) and raycast.cu (EstimateRange / RayCast).
#pragma once

#include <vector>

#include "common.cuh"
#include "hash.cuh"

namespace o3db {

// --------------------------------------------------------- camera geometry

// t/geometry/kernel/GeometryIndexer.h:25-144 TransformIndexer: all f32.
struct Cam {
    float e[3][4];
    float fx, fy, cx, cy;
    float scale;
};

__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float dvd(float a, float b) { return __fdiv_rn(a, b); }

// GeometryIndexer.h:62-78 RigidTransform
__device__ __forceinline__ void rigid(const Cam& c, float x, float y, float z, float& xo, float& yo, float& zo) {
    x = mul(x, c.scale);
    y = mul(y, c.scale);
    z = mul(z, c.scale);
    xo = add(add(add(mul(x, c.e[0][0]), mul(y, c.e[0][1])), mul(z, c.e[0][2])), c.e[0][3]);
    yo = add(add(add(mul(x, c.e[1][0]), mul(y, c.e[1][1])), mul(z, c.e[1][2])), c.e[1][3]);
    zo = add(add(add(mul(x, c.e[2][0]), mul(y, c.e[2][1])), mul(z, c.e[2][2])), c.e[2][3]);
}
// :100-108 Project
__device__ __forceinline__ void project(const Cam& c, float x, float y, float z, float& u, float& v) {
    const float inv_z = __frcp_rn(z);   // == 1.0f / z correctly rounded (the same real number, the same rounding): fewer instructions than a general IEEE division
    u = add(mul(mul(c.fx, x), inv_z), c.cx);
    v = add(mul(mul(c.fy, y), inv_z), c.cy);
}
// :111-120 Unproject
__device__ __forceinline__ void unproject(const Cam& c, float u, float v, float d, float& x, float& y, float& z) {
    x = dvd(mul(sub(u, c.cx), d), c.fx);
    y = dvd(mul(sub(v, c.cy), d), c.fy);
    z = d;
}
// :294-297 InBoundary(x, y) with shape (rows, cols)
__device__ __forceinline__ bool in_boundary(float x, float y, int rows, int cols) {
    return y >= 0 && x >= 0 && y <= rows - 1.0f && x <= cols - 1.0f;
}

// t/geometry/Utility.h:77-115 InverseTransformation (f64, same operation order)
static void inverse_transformation(const double* T, double* Ti) {
    Ti[0] = T[0]; Ti[1] = T[4]; Ti[2] = T[8];
    Ti[4] = T[1]; Ti[5] = T[5]; Ti[6] = T[9];
    Ti[8] = T[2]; Ti[9] = T[6]; Ti[10] = T[10];
    Ti[3] = -(Ti[0] * T[3] + Ti[1] * T[7] + Ti[2] * T[11]);
    Ti[7] = -(Ti[4] * T[3] + Ti[5] * T[7] + Ti[6] * T[11]);
    Ti[11] = -(Ti[8] * T[3] + Ti[9] * T[7] + Ti[10] * T[11]);
    Ti[12] = 0; Ti[13] = 0; Ti[14] = 0; Ti[15] = 1;
}

static Cam make_cam(const double* K, const double* E, float scale) {
    Cam c;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 4; ++j) c.e[i][j] = (float)E[i * 4 + j];
    c.fx = (float)K[0];
    c.fy = (float)K[4];
    c.cx = (float)K[2];
    c.cy = (float)K[5];
    c.scale = scale;
    return c;
}

}  // namespace o3db

struct o3db_vbg {
    float voxel_size = 0;
    int resolution = 16;
    int64_t capacity = 0;
    bool with_color = false;
    // hash map
    int* table = nullptr;
    unsigned nbuckets = 0;
    int* keys = nullptr;
    int* stamp = nullptr;
    int* size_dev = nullptr;       // [0] size
    int* counters = nullptr;       // [0] n_exist [1] n_new [2] overflow [3] ticket
    // values
    float* tsdf = nullptr;
    uint16_t* weight = nullptr;
    uint16_t* color = nullptr;
    // per-frame scratch (sized for the frustum capacity (W/4)(H/4)*4)
    int64_t frustum_cap = 0;
    int* cand_keys = nullptr;
    int* exist_list = nullptr;
    int2* new_list = nullptr;
    int* frame_slots = nullptr;
    int* frame_count = nullptr;
    unsigned long long* exec_ns = nullptr;   // device-timer statistics of the fused integrate launches (o3db_vbg_exec_stats)
    const float* inv_w = nullptr;  // [65536] 1 / (w + 1) per u16 weight (integrate16_kernel); per-device table, not owned
    float checked_scale = 0.f;     // depth_scale the 3-FMA u16 division was last verified for ...
    bool checked_scale_ok = false; // ... and whether it reproduces d / scale for all 65536 u16 values
    bool sync_next_frame = false;  // the next fused frame sizes the map synchronously (after a reserve)
    // frustum-only table for the stand-alone GetUniqueBlockCoordinates
    int* ftable = nullptr;
    unsigned fbuckets = 0;
    // staging for the host-image entry point: two slots, uploads on a private copy stream so
    // that frame f+1's H2D overlaps frame f's kernels
    void* d_depth[2] = {nullptr, nullptr};
    void* d_color[2] = {nullptr, nullptr};
    size_t d_depth_bytes[2] = {0, 0}, d_color_bytes[2] = {0, 0};
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t copied[2] = {nullptr, nullptr}, consumed[2] = {nullptr, nullptr};
    int64_t host_frames = 0;
    // host mirrors: size_dev[0..15] is copied to pinned memory after every fused frame
    // (ring of 2) so that capacity can be managed without a per-frame host sync.
    int* h_pinned = nullptr;       // [0..15] synchronous read-back, then a ring of 8 x 16 ints the device writes into
                                   // directly (publish_status): per-frame status without a copy or an event in the stream
    cudaEvent_t ev[2] = {nullptr, nullptr};
    int frame_id = 0;
    int64_t frames = 0;            // fused frames launched
    int64_t known_size = 0;        // size as last read back (a lower bound)
    int64_t max_new_seen = 0;
    // optional per-kernel timing (o3db_vbg_profile)
    std::vector<cudaEvent_t> prof_ev;
    int64_t prof_frames = 0;
    bool prof_on = false;
    // o3db_vbg_extract_point_cloud (extract.cu): scratch for ext_blocks slots, outputs for ext_rows points
    int64_t ext_blocks = 0;
    int* ext_nb = nullptr;                    // [ext_blocks][27] neighbour slots, -1 = absent
    unsigned* ext_counts = nullptr;           // [ext_blocks + 1] points per block, then their exclusive scan
    unsigned* ext_scan = nullptr;             // scan tile sums
    unsigned* ext_masks = nullptr;            // [ext_blocks][ceil(res^3 / 32)][3] crossing bits per axis
    unsigned long long* ext_total = nullptr;  // 64-bit point count
    long long* h_ext_total = nullptr;         // pinned read-back of it
    int64_t ext_rows = 0;
    float* ext_points = nullptr;
    float* ext_normals = nullptr;
    float* ext_colors = nullptr;
};

namespace o3db {
// tsdf.cu: takes the status words size_dev[0..15] read back into h; O3DB_ERR_CAPACITY after a dropped frame
int absorb_status(o3db_vbg* v, const int* h);
// extract.cu: frees what o3db_vbg_extract_point_cloud allocated (o3db_vbg_destroy, after a device synchronise)
void extract_release(o3db_vbg* v);
}  // namespace o3db
