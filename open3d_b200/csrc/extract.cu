// extract.cu — VoxelBlockGrid::ExtractPointCloud for sm_90a: the TSDF surface as points with normals (and colours);
// below it, VoxelBlockGrid::ExtractTriangleMesh, which reuses its neighbour table, vertex emission and scan.
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
#include "marching_cubes.cuh"
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

// ---------------------------------------------------------------------------------------------------------------
// VoxelBlockGrid::ExtractTriangleMesh (VoxelBlockGrid.cpp:436-472, kernel VoxelBlockGridImpl.h:1385-1780).  The cube
// at voxel o has corners o + {0,1}^3; it contributes when all 8 exist with weight > threshold, and its case is the
// 8-bit tsdf < 0 pattern (marching_cubes.cuh).  The edge (o, o + e_i) carries a vertex when one of the up to four
// cubes sharing it contributes and its corners differ in that bit (upstream's pass 0 marking).  Vertex rows are the
// point cloud's (extract_emit_kernel over the vertex bits, in its order); triangle rows come by block, then voxel,
// then the generated table's order, each written reversed as upstream writes it.  Nine passes in twelve launches:
//   neighbours   extract_neighbors_kernel;
//   classify     one CTA per block stages the tsdf < 0 / contributing bits of voxels [0, R]^3 in shared memory and
//                writes one case byte per cube;
//   count        one CTA per block stages the case bytes of cubes [-1, R-1]^3, derives each owned edge's vertex bit
//                into ballot words as extract_count_kernel does, keeps the block's vertices before each word, and
//                writes the block's vertex and triangle counts;
//   scan x 2     the per-block vertex and triangle counts;
//   vertices     extract_emit_kernel;
//   triangles    one CTA per block scans its cubes' triangle counts in voxel order; a corner's vertex is the owning
//                block's first row + the rank of its (voxel, axis) bit in that block's words.

static constexpr mc::Table kMcTable = mc::make_table();
__constant__ mc::Table c_mc = kMcTable;

struct MeshArgs {
    ExtractArgs e;              // as the point cloud's, with the mesh's nb / counts (vertices) / masks / total
    unsigned char* cases;
    unsigned* wbase;
    unsigned* tcounts;
    unsigned long long* ttotal;
    long long tlimit;           // triangle rows to write
    int* triangles;
};

// Loads s[((z*(R+1)) + y)*(R+1) + x] = f(linear index of voxel (x, y, z) + lo, or -1) for x, y, z in [0, R].
template <typename F>
__device__ __forceinline__ void stage_halo(const ExtractArgs& a, const int* s_nb, int lo, unsigned char* s, F f) {
    const int R = a.res, R1 = R + 1;
    for (int h = threadIdx.x; h < R1 * R1 * R1; h += kET) {
        const int x = h % R1, y = (h / R1) % R1, z = h / (R1 * R1);
        s[h] = f(linear_idx(s_nb, R, a.div_res, x + lo, y + lo, z + lo));
    }
}

__global__ void __launch_bounds__(kET) mesh_classify_kernel(MeshArgs m) {
    extern __shared__ unsigned char s_flag[];   // [(R+1)^3] voxels [0, R]^3: bit 0 exists with weight > threshold, bit 1 tsdf < 0
    __shared__ int s_nb[27];
    pdl_wait();
    const ExtractArgs& a = m.e;
    const int n = *a.size, R = a.res, R1 = R + 1;
    for (int b = blockIdx.x; b < n; b += gridDim.x) {
        __syncthreads();   // the previous block's readers of s_nb and s_flag are done
        if (threadIdx.x < 27) s_nb[threadIdx.x] = a.nb[27 * (size_t)b + threadIdx.x];
        __syncthreads();
        stage_halo(a, s_nb, 0, s_flag, [&](long long lin) -> unsigned char {
            // VoxelBlockGridImpl.h:1479-1484: a missing corner or weight <= threshold leaves the cube out
            if (lin < 0 || (float)a.weight[lin] <= a.weight_threshold) return 0;
            return a.tsdf[lin] < 0.f ? 3 : 1;
        });
        __syncthreads();
        for (int v = threadIdx.x; v < a.res3; v += kET) {
            const int q = fast_div(v, a.div_res), z = fast_div(v, a.div_res2);
            const int x = v - q * R, y = q - z * R;
            unsigned all = 1, c = 0;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const unsigned f = s_flag[((z + mc::corner_offset(k, 2)) * R1 + y + mc::corner_offset(k, 1)) * R1 +
                                                x + mc::corner_offset(k, 0)];
                all &= f;
                c |= (f >> 1) << k;
            }
            m.cases[(size_t)b * a.res3 + v] = (unsigned char)(all ? c : 0u);
        }
    }
}

__global__ void __launch_bounds__(kET) mesh_count_kernel(MeshArgs m) {
    extern __shared__ unsigned char s_case[];   // [(R+1)^3] cubes at voxels [-1, R-1]^3
    __shared__ int s_nb[27];
    __shared__ unsigned s_warp[kET / 32];
    pdl_wait();
    const ExtractArgs& a = m.e;
    const int n = *a.size, R = a.res, R1 = R + 1, R3 = a.res3;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int b = blockIdx.x; b < a.capacity; b += gridDim.x) {
        if (b >= n) {   // the scans run over every slot
            if (threadIdx.x == 0) a.counts[b] = m.tcounts[b] = 0;
            continue;
        }
        __syncthreads();
        if (threadIdx.x < 27) s_nb[threadIdx.x] = a.nb[27 * (size_t)b + threadIdx.x];
        __syncthreads();
        stage_halo(a, s_nb, -1, s_case,
                   [&](long long lin) -> unsigned char { return lin < 0 ? 0 : m.cases[lin]; });
        __syncthreads();
        unsigned rows = 0, tris = 0;
        for (int v0 = 0; v0 < a.words * 32; v0 += kET) {
            const int v = v0 + threadIdx.x;
            unsigned bits = 0;
            if (v < R3) {
                const int q = fast_div(v, a.div_res), z = fast_div(v, a.div_res2);
                const int x = v - q * R, y = q - z * R;
                const int h = ((z + 1) * R1 + y + 1) * R1 + x + 1;   // the cube at o
                tris += c_mc.ntri[s_case[h]];
                const int st[3] = {1, R1, R1 * R1};
#pragma unroll
                for (int i = 0; i < 3; ++i) {   // edge (o, o + e_i) as seen from the cubes at o - s
                    unsigned cross = 0;
#pragma unroll
                    for (int s = 0; s < 4; ++s) {
                        int off[3] = {0, 0, 0};
                        off[(i + 1) % 3] = s & 1;
                        off[(i + 2) % 3] = s >> 1;
                        const unsigned c = s_case[h - off[0] * st[0] - off[1] * st[1] - off[2] * st[2]];
                        const int lo = mc::corner_at(off[0], off[1], off[2]);
                        const int hi = mc::corner_at(off[0] + (i == 0), off[1] + (i == 1), off[2] + (i == 2));
                        cross |= (c >> lo) ^ (c >> hi);
                    }
                    bits |= (cross & 1u) << i;
                }
            }
            const unsigned m0 = __ballot_sync(0xffffffffu, bits & 1u);
            const unsigned m1 = __ballot_sync(0xffffffffu, bits & 2u);
            const unsigned m2 = __ballot_sync(0xffffffffu, bits & 4u);
            const int w = (v0 >> 5) + warp;
            if (lane == 0) s_warp[warp] = __popc(m0) + __popc(m1) + __popc(m2);
            __syncthreads();
            if (lane == 0 && w < a.words) {
                unsigned* mk = a.masks + ((size_t)b * a.words + w) * 3;
                mk[0] = m0;
                mk[1] = m1;
                mk[2] = m2;
                unsigned before = rows;
                for (int k = 0; k < warp; ++k) before += s_warp[k];
                m.wbase[(size_t)b * a.words + w] = before;
            }
#pragma unroll
            for (int k = 0; k < kET / 32; ++k) rows += s_warp[k];
            __syncthreads();   // s_warp is rewritten by the next round
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) tris += __shfl_xor_sync(0xffffffffu, tris, o);
        if (lane == 0) s_warp[warp] = tris;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned t = 0;
#pragma unroll
            for (int k = 0; k < kET / 32; ++k) t += s_warp[k];
            a.counts[b] = rows;
            m.tcounts[b] = t;
            if (rows) atomicAdd(a.total, (unsigned long long)rows);
            if (t) atomicAdd(m.ttotal, (unsigned long long)t);
        }
    }
}

// The triangles of the cube at voxel v of the current block (case c, nt triangles, first row `row`), :1704-1750.
__device__ void emit_cube(const MeshArgs& m, const int* s_nb, int v, unsigned c, unsigned nt, long long row) {
    const ExtractArgs& a = m.e;
    const int R = a.res;
    const int q = fast_div(v, a.div_res), z = fast_div(v, a.div_res2);
    const int x = v - q * R, y = q - z * R;
    for (unsigned t = 0; t < nt; ++t, ++row) {
        if (row >= m.tlimit) return;
        int* tri = m.triangles + 3 * row;
        for (int k = 0; k < 3; ++k) {
            const unsigned ow = c_mc.owner[c_mc.tri[c][3 * t + k]];
            const int o[3] = {x + (int)(ow & 1u), y + (int)((ow >> 1) & 1u), z + (int)((ow >> 2) & 1u)};
            const int axis = (int)(ow >> 3);
            const int bx = o[0] >= R, by = o[1] >= R, bz = o[2] >= R;   // owner in the +x / +y / +z neighbour
            const int slot = s_nb[13 + bx + 3 * by + 9 * bz];
            const int lv = ((o[2] - bz * R) * R + o[1] - by * R) * R + o[0] - bx * R, l = lv & 31;
            const size_t wi = (size_t)slot * a.words + (lv >> 5);
            const unsigned* mk = a.masks + 3 * wi;
            const unsigned below = (1u << l) - 1u;
            unsigned idx = a.counts[slot] + m.wbase[wi] + __popc(mk[0] & below) + __popc(mk[1] & below) +
                           __popc(mk[2] & below);
            if (axis > 0) idx += (mk[0] >> l) & 1u;
            if (axis > 1) idx += (mk[1] >> l) & 1u;
            tri[2 - k] = (int)idx;
        }
    }
}

__global__ void __launch_bounds__(kET) mesh_triangle_kernel(MeshArgs m) {
    __shared__ int s_nb[27];
    __shared__ unsigned s_part[kET / 32];
    pdl_wait();
    const ExtractArgs& a = m.e;
    const int n = *a.size;
    for (int b = blockIdx.x; b < n; b += gridDim.x) {
        long long row = m.tcounts[b];
        if (row >= m.tlimit) continue;
        __syncthreads();   // the previous block's readers of s_nb are done
        if (threadIdx.x < 27) s_nb[threadIdx.x] = a.nb[27 * (size_t)b + threadIdx.x];
        __syncthreads();
        for (int v0 = 0; v0 < a.res3; v0 += kET) {
            const int v = v0 + threadIdx.x;
            const unsigned c = v < a.res3 ? m.cases[(size_t)b * a.res3 + v] : 0u;
            const unsigned nt = c_mc.ntri[c];
            unsigned total;
            const unsigned ex = cta_exclusive_scan(nt, s_part, total);
            if (nt) emit_cube(m, s_nb, v, c, nt, row + ex);
            row += total;
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

static int ensure_mesh_scratch(o3db_vbg* v, cudaStream_t st) {
    if (v->mesh_blocks >= v->map.capacity) return O3DB_OK;
    for (GridPtr<unsigned>* p : {&v->mesh_vcounts, &v->mesh_tcounts, &v->mesh_scan, &v->mesh_masks, &v->mesh_wbase})
        free_on(*p, st);
    free_on(v->mesh_nb, st);
    free_on(v->mesh_cases, st);
    v->mesh_blocks = 0;
    const int64_t cap = v->map.capacity, r3 = (int64_t)v->resolution * v->resolution * v->resolution;
    const int64_t words = ceil_div(r3, 32);
    if (int rc = dev_alloc(v->mesh_nb, (size_t)cap * 27, st)) return rc;
    if (int rc = dev_alloc(v->mesh_cases, (size_t)(cap * r3), st)) return rc;
    if (int rc = dev_alloc(v->mesh_vcounts, (size_t)(cap + 1), st)) return rc;
    if (int rc = dev_alloc(v->mesh_tcounts, (size_t)(cap + 1), st)) return rc;
    if (int rc = dev_alloc(v->mesh_scan, (size_t)ceil_div(cap, kScanTile), st)) return rc;
    if (int rc = dev_alloc(v->mesh_masks, (size_t)cap * words * 3, st)) return rc;
    if (int rc = dev_alloc(v->mesh_wbase, (size_t)cap * words, st)) return rc;
    if (!v->mesh_totals)
        if (int rc = dev_alloc(v->mesh_totals, 2, st)) return rc;
    if (!v->h_mesh_totals) {
        v->h_mesh_totals = pinned_block<long long[]>(2);
        O3DB_REQUIRE(v->h_mesh_totals != nullptr, "o3db_vbg_extract_triangle_mesh: out of pinned host memory");
    }
    v->mesh_blocks = cap;
    return O3DB_OK;
}

// Grows the vertex and triangle buffers to at least `verts` and `tris` rows, with the point cloud's headroom.
static int ensure_mesh_rows(o3db_vbg* v, int64_t verts, int64_t tris, cudaStream_t st) {
    const auto grow = [](int64_t r) { return std::max<int64_t>(r, std::min<int64_t>(INT_MAX, r + r / 4)); };
    if (verts > v->mesh_vrows) {
        for (GridPtr<float>* p : {&v->mesh_positions, &v->mesh_normals, &v->mesh_colors}) free_on(*p, st);
        v->mesh_vrows = 0;
        verts = grow(verts);
        if (int rc = dev_alloc(v->mesh_positions, (size_t)verts * 3, st)) return rc;
        if (int rc = dev_alloc(v->mesh_normals, (size_t)verts * 3, st)) return rc;
        if (v->with_color)
            if (int rc = dev_alloc(v->mesh_colors, (size_t)verts * 3, st)) return rc;
        v->mesh_vrows = verts;
    }
    if (tris > v->mesh_trows) {
        free_on(v->mesh_triangles, st);
        v->mesh_trows = 0;
        tris = grow(tris);
        if (int rc = dev_alloc(v->mesh_triangles, (size_t)tris * 3, st)) return rc;
        v->mesh_trows = tris;
    }
    return O3DB_OK;
}

// The vertex and triangle emission into the handle's mesh buffers, limited to their first `verts` and `tris` rows.
static int launch_mesh_emit(const o3db_vbg* v, MeshArgs m, long long verts, long long tris, unsigned grid,
                            cudaStream_t st) {
    m.e.limit = verts;
    m.e.points = v->mesh_positions.get();
    m.e.normals = v->mesh_normals.get();
    m.e.colors = v->with_color ? v->mesh_colors.get() : nullptr;
    m.tlimit = tris;
    m.triangles = v->mesh_triangles.get();
    O3DB_CUDA_CHECK(launch_pdl_ex(extract_emit_kernel, {grid, kET}, st, m.e));
    O3DB_CUDA_CHECK(launch_pdl_ex(mesh_triangle_kernel, {grid, kET}, st, m));
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

int o3db_vbg_extract_triangle_mesh(o3db_vbg* v, float weight_threshold, int64_t estimated_vertex_number,
                                   int64_t* num_vertices, int64_t* num_triangles, float** vertices, float** normals,
                                   float** colors, int32_t** triangles, void* stream) {
    O3DB_REQUIRE(v != nullptr, "o3db_vbg_extract_triangle_mesh: null voxel grid");
    O3DB_REQUIRE(num_vertices && num_triangles && vertices && normals && colors && triangles,
                 "o3db_vbg_extract_triangle_mesh: null output");
    *num_vertices = *num_triangles = 0;
    *vertices = *normals = *colors = nullptr;
    *triangles = nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = ensure_mesh_scratch(v, st);
    if (rc) return rc;
    if (estimated_vertex_number > 0) {   // a sizing hint: room for that many vertices and twice as many triangles
        const int64_t hint = std::min<int64_t>(estimated_vertex_number, INT_MAX);
        rc = ensure_mesh_rows(v, hint, std::min<int64_t>(2 * hint, INT_MAX), st);
        if (rc) return rc;
    }
    MeshArgs m{};
    ExtractArgs& a = m.e;
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
    a.nb = v->mesh_nb.get();
    a.counts = v->mesh_vcounts.get();
    a.masks = v->mesh_masks.get();
    a.total = v->mesh_totals.get();
    m.cases = v->mesh_cases.get();
    m.wbase = v->mesh_wbase.get();
    m.tcounts = v->mesh_tcounts.get();
    m.ttotal = v->mesh_totals.get() + 1;
    const unsigned grid = (unsigned)std::min<int64_t>(v->map.capacity, (int64_t)num_sms() * 8);
    const size_t halo = (size_t)(a.res + 1) * (a.res + 1) * (a.res + 1);   // bytes of the staged voxels or cubes
    O3DB_CUDA_CHECK(cudaMemsetAsync(v->mesh_totals.get(), 0, 2 * sizeof(unsigned long long), st));
    extract_neighbors_kernel<<<(unsigned)std::min<int64_t>(ceil_div(v->map.capacity * 27, kET), (int64_t)num_sms() * 8), kET,
                               0, st>>>(a);
    O3DB_LAUNCH_CHECK();
    O3DB_CUDA_CHECK(launch_pdl_ex(mesh_classify_kernel, {grid, kET, halo}, st, m));
    O3DB_CUDA_CHECK(launch_pdl_ex(mesh_count_kernel, {grid, kET, halo}, st, m));
    rc = exclusive_scan_u32(v->mesh_vcounts.get(), v->map.capacity, v->mesh_scan.get(), st);
    if (rc) return rc;
    rc = exclusive_scan_u32(v->mesh_tcounts.get(), v->map.capacity, v->mesh_scan.get(), st);
    if (rc) return rc;
    // emitted before the read-back when the buffers already hold rows (every call but the ones that grow them)
    const bool ahead = v->mesh_vrows > 0 && v->mesh_trows > 0;
    const long long ahead_v = ahead ? v->mesh_vrows : 0, ahead_t = ahead ? v->mesh_trows : 0;
    if (ahead) {
        rc = launch_mesh_emit(v, m, ahead_v, ahead_t, grid, st);
        if (rc) return rc;
    }
    // the one host synchronisation (read_status's): the two counts and the map status (a frame dropped for capacity)
    O3DB_CUDA_CHECK(cudaMemcpyAsync(v->h_mesh_totals.get(), v->mesh_totals.get(), 2 * sizeof(long long),
                                    cudaMemcpyDeviceToHost, st));
    rc = read_status(v, st);
    if (rc) return rc;
    const long long verts = v->h_mesh_totals[0], tris = v->h_mesh_totals[1];
    if (verts > INT_MAX || tris > INT_MAX) {
        set_last_error("o3db_vbg_extract_triangle_mesh: the surface has %lld vertices and %lld triangles, more than "
                       "the %d that Int32 indices can address; raise weight_threshold or extract a smaller volume",
                       verts, tris, INT_MAX);
        return O3DB_ERR_INVALID;
    }
    if (verts > ahead_v || tris > ahead_t) {
        rc = ensure_mesh_rows(v, verts, tris, st);
        if (rc) return rc;
        rc = launch_mesh_emit(v, m, verts, tris, grid, st);
        if (rc) return rc;
    }
    *num_vertices = verts;
    *num_triangles = tris;
    if (verts > 0) {
        *vertices = v->mesh_positions.get();
        *normals = v->mesh_normals.get();
        *colors = v->with_color ? v->mesh_colors.get() : nullptr;
        *triangles = v->mesh_triangles.get();
    }
    return O3DB_OK;
}

}  // extern "C"
