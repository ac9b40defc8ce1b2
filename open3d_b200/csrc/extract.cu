// extract.cu — VoxelBlockGrid::ExtractPointCloud for sm_90a: the TSDF surface as points with normals (and colours).
//
// Reference: VoxelBlockGrid.cpp:404-434 (driver), BufferRadiusNeighbors (:22-51) and
// kernel::voxel_grid::ExtractPointCloud (VoxelBlockGridImpl.h:1122-1381, DeviceGetLinearIdx / DeviceGetNormal :94-149).
// A point is emitted for voxel o and axis i when o and o + e_i both have weight > threshold and tsdf_i * tsdf_o < 0.
//
// Upstream appends points through an atomic counter, so its order changes from run to run.  Here the order is fixed:
// ascending block slot, then the linear voxel index (z*R + y)*R + x, then axis 0, 1, 2.  Four passes in six launches
// (the scan takes three) whatever the volume:
//   neighbours   27 hash probes per active block -> [slot][27] table (BufferRadiusNeighbors);
//   count        one CTA per block: each warp tests 32 consecutive voxels and keeps one ballot word per axis, the
//                CTA writes the block's point count and adds it to a 64-bit total;
//   scan         exclusive scan of the per-block counts (icp.cu's u32 scan, scan.cuh);
//   emit         one CTA per block: the voxels with crossing bits are compacted, in order, into a shared list with
//                their first row (from the ballot words), then one thread per listed voxel gathers what its points
//                need (the +-1 tsdf neighbours for the normals, two colours).
// The device holds the block count, so nothing waits for the host until the one read-back of the total and the map
// status.  The emit pass is queued before that read-back whenever the handle's output buffers are already large
// enough (every call but the ones that grow them): steady-state calls synchronise once, at the end.
//
// Every f32 expression is evaluated in the reference's source order with round-to-nearest intrinsics (no FMA
// contraction, no flush of subnormals), so the rows equal the CPU oracle's bit for bit.
#include <algorithm>
#include <climits>

#include "common.cuh"
#include "hash.cuh"
#include "scan.cuh"
#include "vbg.cuh"

namespace o3db {

static constexpr int kET = 256;   // threads per CTA of the extraction kernels

struct ExtractArgs {
    Table tab;
    const int* size;            // device: active blocks are slots 0..*size-1
    int capacity;               // slots the scratch covers
    int res, res3, words;       // block resolution, res^3, ceil(res^3 / 32)
    unsigned long long div_res, div_res2;   // fast_div multipliers for res and res^2
    float voxel_size, weight_threshold;
    const float* tsdf;
    const uint16_t* weight;
    const uint16_t* color;      // null: no colour attribute
    int* nb;
    unsigned* counts;
    unsigned* masks;
    unsigned long long* total;
    long long limit;            // rows to write
    float* points;
    float* normals;
    float* colors;
};

// floor(n / d) for n < 2^16 and d <= 1024 from m = ceil(2^32 / d): the error term n * (m*d - 2^32) / 2^32 stays
// below 1 / d, so the quotient is exact.
static unsigned long long fast_div_multiplier(unsigned d) { return ((1ull << 32) + d - 1) / d; }
__device__ __forceinline__ int fast_div(int n, unsigned long long m) {
    return (int)(((unsigned long long)(unsigned)n * m) >> 32);
}

__global__ void __launch_bounds__(kET) extract_neighbors_kernel(ExtractArgs a) {
    const long long n = (long long)*a.size * 27;
    for (long long i = blockIdx.x * (long long)kET + threadIdx.x; i < n; i += (long long)gridDim.x * kET) {
        const int b = (int)(i / 27), k = (int)(i % 27);
        const int* key = a.tab.keys + 3 * (size_t)b;
        unsigned bucket;
        const int s = probe<false>(a.tab, nullptr, 0, key[0] + k % 3 - 1, key[1] + (k % 9) / 3 - 1, key[2] + k / 9 - 1,
                                   &bucket);
        a.nb[i] = s >= 0 ? s : -1;
    }
}

__global__ void __launch_bounds__(kET) extract_count_kernel(ExtractArgs a) {
    __shared__ int s_face[3];   // slots of the +x, +y, +z neighbour blocks
    __shared__ unsigned s_warp[kET / 32];
    pdl_wait();
    const int n = *a.size;
    const int R = a.res, R3 = a.res3;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int stride[3] = {1, R, R * R};
    for (int b = blockIdx.x; b < a.capacity; b += gridDim.x) {
        if (b >= n) {   // the scan runs over every slot
            if (threadIdx.x == 0) a.counts[b] = 0;
            continue;
        }
        __syncthreads();
        if (threadIdx.x < 3) s_face[threadIdx.x] = a.nb[27 * (size_t)b + 13 + (threadIdx.x == 0 ? 1 : threadIdx.x == 1 ? 3 : 9)];
        __syncthreads();
        unsigned cnt = 0;
        for (int v0 = warp * 32; v0 < a.words * 32; v0 += kET) {
            const int v = v0 + lane;
            unsigned bits = 0;
            if (v < R3) {
                const size_t lin = (size_t)b * R3 + v;
                if ((float)a.weight[lin] > a.weight_threshold) {   // VoxelBlockGridImpl.h:1220-1222
                    const float tsdf_o = a.tsdf[lin];
                    const int q = fast_div(v, a.div_res), z = fast_div(v, a.div_res2);
                    const int c[3] = {v - q * R, q - z * R, z};
#pragma unroll
                    for (int i = 0; i < 3; ++i) {   // :1225-1237
                        size_t lin_i;
                        if (c[i] + 1 < R) {
                            lin_i = lin + stride[i];
                        } else {   // DeviceGetLinearIdx: voxel 0 of the next block along i
                            const int s = s_face[i];
                            if (s < 0) continue;
                            lin_i = (size_t)s * R3 + v - (size_t)(R - 1) * stride[i];
                        }
                        if ((float)a.weight[lin_i] > a.weight_threshold && mul(a.tsdf[lin_i], tsdf_o) < 0.f)
                            bits |= 1u << i;
                    }
                }
            }
            const unsigned m0 = __ballot_sync(0xffffffffu, bits & 1u);
            const unsigned m1 = __ballot_sync(0xffffffffu, bits & 2u);
            const unsigned m2 = __ballot_sync(0xffffffffu, bits & 4u);
            if (lane == 0) {
                unsigned* m = a.masks + ((size_t)b * a.words + (v0 >> 5)) * 3;
                m[0] = m0;
                m[1] = m1;
                m[2] = m2;
            }
            cnt += __popc(m0) + __popc(m1) + __popc(m2);
        }
        if (lane == 0) s_warp[warp] = cnt;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned t = 0;
#pragma unroll
            for (int w = 0; w < kET / 32; ++w) t += s_warp[w];
            a.counts[b] = t;
            if (t) atomicAdd(a.total, (unsigned long long)t);
        }
    }
}

__device__ __forceinline__ int isign(int x) { return (x > 0) ? 1 : ((x < 0) ? -1 : 0); }

// DeviceGetLinearIdx (VoxelBlockGridImpl.h:94-121) on the block's 27 neighbour slots; coordinates in [-1, R+1].
__device__ __forceinline__ long long linear_idx(const int* s_nb, int R, unsigned long long div_res, int xo, int yo,
                                               int zo) {
    const int xn = xo + R - fast_div(xo + R, div_res) * R;   // (xo + R) % R
    const int yn = yo + R - fast_div(yo + R, div_res) * R;
    const int zn = zo + R - fast_div(zo + R, div_res) * R;
    const int s = s_nb[(isign(xo - xn) + 1) + (isign(yo - yn) + 1) * 3 + (isign(zo - zn) + 1) * 9];
    if (s < 0) return -1;
    return (((long long)s * R + zn) * R + yn) * R + xn;
}

// DeviceGetNormal (:123-149): a component is written only when both of its neighbours exist.
__device__ __forceinline__ void tsdf_gradient(const float* __restrict__ tsdf, const int* s_nb, int R,
                                              unsigned long long dr, int x, int y, int z, float n[3]) {
    const long long vxp = linear_idx(s_nb, R, dr, x + 1, y, z), vxn = linear_idx(s_nb, R, dr, x - 1, y, z);
    const long long vyp = linear_idx(s_nb, R, dr, x, y + 1, z), vyn = linear_idx(s_nb, R, dr, x, y - 1, z);
    const long long vzp = linear_idx(s_nb, R, dr, x, y, z + 1), vzn = linear_idx(s_nb, R, dr, x, y, z - 1);
    if (vxp >= 0 && vxn >= 0) n[0] = sub(tsdf[vxp], tsdf[vxn]);
    if (vyp >= 0 && vyn >= 0) n[1] = sub(tsdf[vyp], tsdf[vyn]);
    if (vzp >= 0 && vzn >= 0) n[2] = sub(tsdf[vzp], tsdf[vzn]);
}

// The points of voxel v of block b (crossing bits `bits`, first row `idx`): :1279-1370.
__device__ void emit_voxel(const ExtractArgs& a, const int* s_nb, int b, int v, unsigned bits, long long idx) {
    const int R = a.res;
    const int q = fast_div(v, a.div_res), z = fast_div(v, a.div_res2);
    const int x = v - q * R, y = q - z * R;
    const long long lin = (long long)b * a.res3 + v;
    const float tsdf_o = a.tsdf[lin];
    float no[3] = {0.f, 0.f, 0.f}, ne[3] = {0.f, 0.f, 0.f};   // ne is not reset between the axes (:1283)
    tsdf_gradient(a.tsdf, s_nb, R, a.div_res, x, y, z, no);
    const int* key = a.tab.keys + 3 * (size_t)b;
    const int g[3] = {key[0] * R + x, key[1] * R + y, key[2] * R + z};
#pragma unroll 1
    for (int i = 0; i < 3; ++i) {
        if (!((bits >> i) & 1u)) continue;
        if (idx >= a.limit) return;
        const int xi = x + (i == 0), yi = y + (i == 1), zi = z + (i == 2);
        const long long lin_i = linear_idx(s_nb, R, a.div_res, xi, yi, zi);
        const float tsdf_i = a.tsdf[lin_i];
        const float ratio = dvd(sub(0.f, tsdf_o), sub(tsdf_i, tsdf_o));
        float* p = a.points + 3 * idx;
#pragma unroll
        for (int k = 0; k < 3; ++k) p[k] = mul(a.voxel_size, add((float)g[k], mul(ratio, k == i ? 1.f : 0.f)));
        tsdf_gradient(a.tsdf, s_nb, R, a.div_res, xi, yi, zi, ne);
        const float nx = add(mul(sub(1.f, ratio), no[0]), mul(ratio, ne[0]));
        const float ny = add(mul(sub(1.f, ratio), no[1]), mul(ratio, ne[1]));
        const float nz = add(mul(sub(1.f, ratio), no[2]), mul(ratio, ne[2]));
        // static_cast<float>(sqrt(nx*nx + ny*ny + nz*nz) + 1e-5) (:1341-1342): the reference's CPU build takes the
        // double sqrt of the f32 sum (DESIGN.md §4.12); + 1e-5 is a double add
        const float s = add(add(mul(nx, nx), mul(ny, ny)), mul(nz, nz));
        const float norm = __double2float_rn(__dadd_rn(__dsqrt_rn((double)s), 1e-5));
        float* q = a.normals + 3 * idx;
        q[0] = dvd(nx, norm);
        q[1] = dvd(ny, norm);
        q[2] = dvd(nz, norm);
        if (a.colors) {
            const uint16_t* co = a.color + 3 * lin;
            const uint16_t* ci = a.color + 3 * lin_i;
            float* c = a.colors + 3 * idx;
#pragma unroll
            for (int k = 0; k < 3; ++k)
                c[k] = dvd(add(mul(sub(1.f, ratio), (float)co[k]), mul(ratio, (float)ci[k])), 255.0f);
        }
        ++idx;
    }
}

// Exclusive scan of one value per thread over the CTA, and the CTA's total; every thread must call it.
__device__ __forceinline__ unsigned cta_exclusive_scan(unsigned v, unsigned* s_part, unsigned& total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    unsigned inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) s_part[w] = inc;
    __syncthreads();
    unsigned base = 0;
    total = 0;
#pragma unroll
    for (int k = 0; k < kET / 32; ++k) {
        base += k < w ? s_part[k] : 0u;
        total += s_part[k];
    }
    __syncthreads();
    return base + inc - v;
}

static constexpr int kRoundWords = 64;   // 32-voxel words compacted per round: at most 2048 voxels

// One CTA per block.  A surface crosses few voxels of a block (about 110 of 4096 in bench.py's volume), so the
// voxels with crossing bits are first compacted into a shared list, in order, kRoundWords words per round; then all
// threads of the CTA take one listed voxel each.
__global__ void __launch_bounds__(kET) extract_emit_kernel(ExtractArgs a) {
    __shared__ int s_nb[27];
    __shared__ unsigned s_part[kET / 32];
    __shared__ unsigned s_list[kRoundWords * 32];   // voxel | (its first row in the block << 15)
    pdl_wait();
    const int n = *a.size;
    for (int b = blockIdx.x; b < n; b += gridDim.x) {
        const long long base = a.counts[b];
        if (base >= a.limit) continue;
        __syncthreads();   // the previous block's readers of s_nb are done
        if (threadIdx.x < 27) s_nb[threadIdx.x] = a.nb[27 * (size_t)b + threadIdx.x];
        const unsigned* mb = a.masks + (size_t)b * a.words * 3;
        unsigned rows_before = 0;   // rows of the block before this round
        for (int w0 = 0; w0 < a.words; w0 += kRoundWords) {
            const int w = w0 + threadIdx.x;
            unsigned m0 = 0, m1 = 0, m2 = 0;
            if (threadIdx.x < kRoundWords && w < a.words) {
                m0 = mb[3 * w];
                m1 = mb[3 * w + 1];
                m2 = mb[3 * w + 2];
            }
            // voxels (low 16 bits, <= 2048) and rows (high 16 bits, <= 6144) of the round's words, scanned together
            unsigned any = m0 | m1 | m2, total;
            const unsigned ex = cta_exclusive_scan(__popc(any) | ((unsigned)(__popc(m0) + __popc(m1) + __popc(m2)) << 16),
                                                   s_part, total);
            unsigned pos = ex & 0xffffu, row = rows_before + (ex >> 16);
            while (any) {
                const int l = __ffs(any) - 1;
                any &= any - 1;
                s_list[pos++] = (unsigned)(32 * w + l) | (row << 15);   // voxel < 2^15, row < 3 * 2^15
                row += ((m0 >> l) & 1u) + ((m1 >> l) & 1u) + ((m2 >> l) & 1u);
            }
            __syncthreads();
            const int nv = (int)(total & 0xffffu);
            for (int k = threadIdx.x; k < nv; k += kET) {
                const unsigned e = s_list[k];
                const int v = (int)(e & 0x7fffu), l = v & 31;
                const long long idx = base + (e >> 15);
                const unsigned* m = mb + 3 * (v >> 5);
                const unsigned bits = ((m[0] >> l) & 1u) | (((m[1] >> l) & 1u) << 1) | (((m[2] >> l) & 1u) << 2);
                if (idx < a.limit) emit_voxel(a, s_nb, b, v, bits, idx);
            }
            rows_before += total >> 16;
            __syncthreads();   // s_list is refilled by the next round
        }
    }
}

static int ensure_scratch(o3db_vbg* v, cudaStream_t st) {
    if (v->ext_blocks >= v->map.capacity) return O3DB_OK;
    for (GridPtr<unsigned>* p : {&v->ext_counts, &v->ext_scan, &v->ext_masks}) free_on(*p, st);
    free_on(v->ext_nb, st);
    v->ext_blocks = 0;
    const int64_t cap = v->map.capacity;
    const int64_t words = ceil_div((int64_t)v->resolution * v->resolution * v->resolution, 32);
    if (int rc = dev_alloc(v->ext_nb, (size_t)cap * 27, st)) return rc;
    if (int rc = dev_alloc(v->ext_counts, (size_t)(cap + 1), st)) return rc;
    if (int rc = dev_alloc(v->ext_scan, (size_t)ceil_div(cap, kScanTile), st)) return rc;
    if (int rc = dev_alloc(v->ext_masks, (size_t)cap * words * 3, st)) return rc;
    if (!v->ext_total)
        if (int rc = dev_alloc(v->ext_total, 1, st)) return rc;
    if (!v->h_ext_total) {
        v->h_ext_total = pinned_block<long long>();
        O3DB_REQUIRE(v->h_ext_total != nullptr, "o3db_vbg_extract_point_cloud: out of pinned host memory");
    }
    v->ext_blocks = cap;
    return O3DB_OK;
}

static int ensure_rows(o3db_vbg* v, int64_t rows, cudaStream_t st) {
    if (rows <= v->ext_rows) return O3DB_OK;
    for (GridPtr<float>* p : {&v->ext_points, &v->ext_normals, &v->ext_colors}) free_on(*p, st);
    v->ext_rows = 0;
    rows = std::max<int64_t>(rows, std::min<int64_t>(INT_MAX, rows + rows / 4));   // headroom for a growing volume
    if (int rc = dev_alloc(v->ext_points, (size_t)rows * 3, st)) return rc;
    if (int rc = dev_alloc(v->ext_normals, (size_t)rows * 3, st)) return rc;
    if (v->with_color)
        if (int rc = dev_alloc(v->ext_colors, (size_t)rows * 3, st)) return rc;
    v->ext_rows = rows;
    return O3DB_OK;
}

static int launch_emit(const o3db_vbg* v, ExtractArgs a, long long limit, unsigned grid, cudaStream_t st) {
    a.limit = limit;
    a.points = v->ext_points.get();
    a.normals = v->ext_normals.get();
    a.colors = v->with_color ? v->ext_colors.get() : nullptr;
    O3DB_CUDA_CHECK(launch_pdl_ex(extract_emit_kernel, {grid, kET}, st, a));
    return O3DB_OK;
}

}  // namespace o3db

using namespace o3db;

extern "C" {

int o3db_vbg_extract_point_cloud(o3db_vbg* v, float weight_threshold, int64_t max_points, int64_t* num_points,
                                 float** points, float** normals, float** colors, void* stream) {
    O3DB_REQUIRE(v != nullptr, "o3db_vbg_extract_point_cloud: null voxel grid");
    O3DB_REQUIRE(num_points && points && normals && colors, "o3db_vbg_extract_point_cloud: null output");
    *num_points = 0;
    *points = *normals = *colors = nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = ensure_scratch(v, st);
    if (rc) return rc;
    ExtractArgs a{};
    a.tab = Table{v->map.table.get(), v->map.nbuckets - 1, v->map.keys.get()};
    a.size = &v->status->size;
    a.capacity = (int)v->map.capacity;
    a.res = v->resolution;
    a.res3 = v->resolution * v->resolution * v->resolution;
    a.words = (int)ceil_div(a.res3, 32);
    a.div_res = fast_div_multiplier((unsigned)a.res);
    a.div_res2 = fast_div_multiplier((unsigned)(a.res * a.res));
    a.voxel_size = v->voxel_size;
    a.weight_threshold = weight_threshold;
    a.tsdf = v->map.tsdf.get();
    a.weight = v->map.weight.get();
    a.color = v->with_color ? v->map.color.get() : nullptr;
    a.nb = v->ext_nb.get();
    a.counts = v->ext_counts.get();
    a.masks = v->ext_masks.get();
    a.total = v->ext_total.get();
    const unsigned grid = (unsigned)std::min<int64_t>(v->map.capacity, (int64_t)num_sms() * 8);
    O3DB_CUDA_CHECK(cudaMemsetAsync(v->ext_total.get(), 0, sizeof(unsigned long long), st));
    extract_neighbors_kernel<<<(unsigned)std::min<int64_t>(ceil_div(v->map.capacity * 27, kET), (int64_t)num_sms() * 8), kET,
                               0, st>>>(a);
    O3DB_LAUNCH_CHECK();
    O3DB_CUDA_CHECK(launch_pdl_ex(extract_count_kernel, {grid, kET}, st, a));
    rc = exclusive_scan_u32(v->ext_counts.get(), v->map.capacity, v->ext_scan.get(), st);
    if (rc) return rc;
    const long long cap_rows = max_points < 0 ? LLONG_MAX : (long long)max_points;
    const long long ahead = std::min<long long>(cap_rows, v->ext_rows);   // rows the current buffers can take
    if (ahead > 0) {
        rc = launch_emit(v, a, ahead, grid, st);
        if (rc) return rc;
    }
    // the one host synchronisation (read_status's): the point count and the map status (a frame dropped for capacity)
    O3DB_CUDA_CHECK(cudaMemcpyAsync(v->h_ext_total.get(), v->ext_total.get(), sizeof(long long), cudaMemcpyDeviceToHost, st));
    rc = read_status(v, st);
    if (rc) return rc;
    const long long total = *v->h_ext_total;
    if (total > INT_MAX) {
        set_last_error("o3db_vbg_extract_point_cloud: the surface has %lld points, more than the %d a point cloud "
                       "can hold; raise weight_threshold or extract a smaller volume", total, INT_MAX);
        return O3DB_ERR_INVALID;
    }
    const long long rows = std::min(total, cap_rows);
    if (rows > ahead) {
        rc = ensure_rows(v, rows, st);
        if (rc) return rc;
        rc = launch_emit(v, a, rows, grid, st);
        if (rc) return rc;
    }
    *num_points = rows;
    if (rows > 0) {
        *points = v->ext_points.get();
        *normals = v->ext_normals.get();
        *colors = v->with_color ? v->ext_colors.get() : nullptr;
    }
    return O3DB_OK;
}

}  // extern "C"
