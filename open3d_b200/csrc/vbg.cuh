// vbg.cuh — state of the voxel block grid handle and the f32 camera geometry shared by
// tsdf.cu (touch / integrate) and raycast.cu (EstimateRange / RayCast).
#pragma once

#include <cstddef>
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

// Buffers an o3db_vbg keeps across calls.
template <typename T>
using GridPtr = DevPtr<T, DeviceFree>;

// Status of a volume.  The handle owns one record on the device; the touch kernel, the integrate kernels and the
// stand-alone hash ops update it.  The last CTA of fused frame f also publishes it into entry f % kStatusRing of a
// ring of pinned host records (publish_status), seq last, so that the host can follow the volume without a copy or
// an event in the stream.
struct VbgStatus {
    int size;                          // committed blocks: slots 0 .. size - 1
    int n_exist, n_new;                // this frame's touched committed blocks and keys first seen (touch_kernel)
    int overflow;                      // sticky: a list or the table overflowed, or a frame was dropped; cleared by a reserve
    int ticket;                        // CTAs of the integrate launch that have finished
    int frame_count;                   // blocks of the last fused frame (frame_slots), 0 if it was dropped
    int max_new;                       // most keys first seen in one frame
    int dropped_need, dropped_frame;   // blocks the first dropped frame needed, and its index + 1 (0 = none dropped)
    int work;                          // dynamic work-unit counter of integrate16_kernel
    int seq;                           // ring entries only: index + 1 of the frame that wrote the entry
    int pad[5];
};
static_assert(sizeof(VbgStatus) == 64, "VbgStatus is one 64-byte record");
static_assert(offsetof(VbgStatus, n_new) == offsetof(VbgStatus, n_exist) + sizeof(int), "touch counters are adjacent");
static constexpr int kStatusRing = 8;   // a power of two

// The hash map and its value buffers, sized together for `capacity` blocks.  A map that grows is built whole beside
// the old one and swapped in only once it is complete, so that a failed grow leaves the volume as it was.
struct VbgMap {
    int64_t capacity = 0;
    unsigned nbuckets = 0;
    GridPtr<int> table, keys, stamp;
    GridPtr<float> tsdf;
    GridPtr<uint16_t> weight, color;   // color only with_color
    void free_on(cudaStream_t st) {
        for (GridPtr<int>* p : {&table, &keys, &stamp}) o3db::free_on(*p, st);
        o3db::free_on(tsdf, st);
        o3db::free_on(weight, st);
        o3db::free_on(color, st);
    }
};

}  // namespace o3db

struct o3db_vbg {
    float voxel_size = 0;
    int resolution = 16;
    bool with_color = false;
    o3db::VbgMap map;
    o3db::GridPtr<o3db::VbgStatus> status;
    // per-frame scratch (sized for the frustum capacity (W/4)(H/4)*4)
    int64_t frustum_cap = 0;
    o3db::GridPtr<int> cand_keys;
    o3db::GridPtr<int> exist_list;
    o3db::GridPtr<int2> new_list;
    o3db::GridPtr<int> frame_slots;
    o3db::GridPtr<unsigned long long> exec_ns;   // device-timer statistics of the fused integrate launches (o3db_vbg_exec_stats)
    const float* inv_w = nullptr;  // [65536] 1 / (w + 1) per u16 weight (integrate16_kernel); per-device table, not owned
    bool sync_next_frame = false;  // the next fused frame sizes the map synchronously (after a reserve)
    // frustum-only table for the stand-alone GetUniqueBlockCoordinates
    o3db::GridPtr<int> ftable;
    unsigned fbuckets = 0;
    // staging for the host-image entry point: two slots, uploads on a private copy stream so
    // that frame f+1's H2D overlaps frame f's kernels
    o3db::GridPtr<char> d_depth[2];
    o3db::GridPtr<char> d_color[2];
    size_t d_depth_bytes[2] = {0, 0}, d_color_bytes[2] = {0, 0};
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t copied[2] = {nullptr, nullptr}, consumed[2] = {nullptr, nullptr};
    int64_t host_frames = 0;
    // [0] synchronous read-back of status (read_status), then the ring the fused frames publish into: capacity is
    // managed without a per-frame host synchronisation
    o3db::PinnedPtr<o3db::VbgStatus[]> h_status;
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
    o3db::GridPtr<int> ext_nb;                    // [ext_blocks][27] neighbour slots, -1 = absent
    o3db::GridPtr<unsigned> ext_counts;           // [ext_blocks + 1] points per block, then their exclusive scan
    o3db::GridPtr<unsigned> ext_scan;             // scan tile sums
    o3db::GridPtr<unsigned> ext_masks;            // [ext_blocks][ceil(res^3 / 32)][3] crossing bits per axis
    o3db::GridPtr<unsigned long long> ext_total;  // 64-bit point count
    o3db::PinnedPtr<long long> h_ext_total;       // pinned read-back of it
    int64_t ext_rows = 0;
    o3db::GridPtr<float> ext_points;
    o3db::GridPtr<float> ext_normals;
    o3db::GridPtr<float> ext_colors;
    // o3db_vbg_extract_triangle_mesh (extract.cu): its own scratch for mesh_blocks slots and outputs for mesh_vrows
    // vertices and mesh_trows triangles, so that neither extraction invalidates the other's results
    int64_t mesh_blocks = 0;
    o3db::GridPtr<int> mesh_nb;                     // [mesh_blocks][27] neighbour slots, -1 = absent
    o3db::GridPtr<unsigned char> mesh_cases;        // [mesh_blocks][res^3] cube case, 0 for a cube that does not contribute
    o3db::GridPtr<unsigned> mesh_vcounts;           // [mesh_blocks + 1] vertices per block, then their exclusive scan
    o3db::GridPtr<unsigned> mesh_tcounts;           // [mesh_blocks + 1] triangles per block, then their exclusive scan
    o3db::GridPtr<unsigned> mesh_scan;              // scan tile sums
    o3db::GridPtr<unsigned> mesh_masks;             // [mesh_blocks][ceil(res^3 / 32)][3] vertex bits per axis
    o3db::GridPtr<unsigned> mesh_wbase;             // [mesh_blocks][ceil(res^3 / 32)] block's vertices before each word
    o3db::GridPtr<unsigned long long> mesh_totals;  // 64-bit vertex and triangle counts
    o3db::PinnedPtr<long long[]> h_mesh_totals;     // pinned read-back of them
    int64_t mesh_vrows = 0, mesh_trows = 0;
    o3db::GridPtr<float> mesh_positions;
    o3db::GridPtr<float> mesh_normals;
    o3db::GridPtr<float> mesh_colors;
    o3db::GridPtr<int> mesh_triangles;
};

namespace o3db {
// tsdf.cu: reads the status back into h_status[0] (one stream synchronisation); O3DB_ERR_CAPACITY after a dropped frame
int read_status(o3db_vbg* v, cudaStream_t st);
}  // namespace o3db
