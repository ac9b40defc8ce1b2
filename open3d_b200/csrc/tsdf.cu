// tsdf.cu — sparse voxel-block TSDF volume for sm_90a: lock-free open-addressing
// hash of int32x3 block keys, frustum block discovery ("touch") and the fused
// per-voxel depth-projection / weight-fusion kernel.  See include/open3d_b200.h
// for the reference interfaces replaced and DESIGN.md for layout + rooflines.
//
// Bit-exactness: everything that feeds a floor()/truncation (block keys, pixel
// selection) is evaluated with explicit round-to-nearest intrinsics in the
// reference's source order, so that nvcc cannot contract it into FMAs; the CPU
// oracle is compiled with -ffp-contract=off.  Keys and pixel choices therefore
// agree bit for bit; TSDF values then agree bit for bit as well.
//
// No CPU fallback: every entry point needs a CUDA device.
#include <cuda.h>   // CUtensorMap (types only: the encoder is resolved through cudaGetDriverEntryPoint)

#include <chrono>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <new>
#include <vector>

#include "common.cuh"
#include "hash.cuh"
#include "vbg.cuh"

namespace o3db {

static constexpr int kT = 256;
static constexpr int kStepSize = 3;                 // VoxelBlockGridCUDA.cu:125 step_size
static constexpr int kSamples = kStepSize + 1;      // est_multipler_factor
static constexpr int kStride = 4;                   // VoxelBlockGrid.cpp:221 down_factor
static constexpr int kPinnedInts = 16 + 8 * 16;     // o3db_vbg::h_pinned: [0..15] synchronous read-back, then a ring of 8 x 16

__device__ __forceinline__ void mbar_arrive(unsigned long long* b) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
// 2-D tiled TMA load (cp.async.bulk.tensor, SASS UTMALDG): box of the descriptor at element (x, y) of the image;
// out-of-image elements are zero-filled by the copy engine, completion is signalled on the mbarrier.
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int x, int y, unsigned long long* b) {
    asm volatile(
            "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                    smem_u32(dst)),
            "l"(map), "r"(smem_u32(b)), "r"(x), "r"(y)
            : "memory");
}

// ------------------------------------------------------------------ touch

struct TouchArgs {
    const void* depth;
    int rows, cols;
    Cam cam;                 // intrinsics + camera->world pose, scale 1 (VoxelBlockGridCUDA.cu:120)
    float block_size, sdf_trunc, depth_scale, depth_max;
    Table tab;
    int* cand_keys;          // [rows/4 * cols/4 * 4, 3] per-call candidate keys
    // fused mode (stamp != nullptr): touched committed slots + newly claimed buckets
    int* stamp;              // [capacity] last frame id that touched the slot
    int frame_id;
    int* exist_list;         // touched committed slots
    int2* new_list;          // (bucket, candidate) of keys first seen in this frame
    int* counters;           // [0] n_exist, [1] n_new, [2] overflow flag
    int max_list;
};

// VoxelBlockGridCUDA.cu:145-189 (DepthTouch lambda) fused with the hash insert
// (:200-204) so that candidate keys never make a round trip through a dense list.
template <typename depth_t>
__global__ void __launch_bounds__(kT) touch_kernel(TouchArgs a) {
    // One thread per (strided pixel, ray sample): 4x the threads of the reference's launch
    // (VoxelBlockGridCUDA.cu:145) and a 4x shorter dependent chain per thread — the kernel is
    // pure latency (a few table round trips), so parallelism is what buys time.
    pdl_wait();                 // the previous frame's integrate kernel: table, stamps, counters
    pdl_launch_dependents();
    const int cols_s = a.cols / kStride, rows_s = a.rows / kStride;
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    const int w = tid / kSamples, step = tid % kSamples;
    const int lane = threadIdx.x & 31;
    bool valid = w < cols_s * rows_s;
    float d = 0.f;
    int x = 0, y = 0;
    if (valid) {
        y = (w / cols_s) * kStride;
        x = (w % cols_s) * kStride;
        d = dvd((float)__ldg(&((const depth_t*)a.depth)[(size_t)y * a.cols + x]), a.depth_scale);
        valid = d > 0 && d < a.depth_max;
    }
    float xc, yc, zc, xg, yg, zg;
    unproject(a.cam, (float)x, (float)y, 1.0f, xc, yc, zc);
    rigid(a.cam, xc, yc, zc, xg, yg, zg);
    const float xo = a.cam.e[0][3], yo = a.cam.e[1][3], zo = a.cam.e[2][3];
    const float xd = sub(xg, xo), yd = sub(yg, yo), zd = sub(zg, zo);
    const float t_min = fmaxf(sub(d, a.sdf_trunc), 0.0f);
    const float t_max = fminf(add(d, a.sdf_trunc), a.depth_max);
    const float t_step = dvd(sub(t_max, t_min), (float)kStepSize);
    float t = t_min;                       // t += t_step, `step` times, exactly as the reference's loop
    for (int s = 0; s < step; ++s) t = add(t, t_step);
    const int kx = (int)floorf(dvd(add(xo, mul(t, xd)), a.block_size));
    const int ky = (int)floorf(dvd(add(yo, mul(t, yd)), a.block_size));
    const int kz = (int)floorf(dvd(add(zo, mul(t, zd)), a.block_size));
    // neighbouring rays / samples of a warp mostly hit the same few blocks: one lane per distinct
    // key does the table work (hash match first, then an exact key comparison with the leader)
    const uint64_t h = minivec_hash(kx, ky, kz);
    const unsigned tag = valid ? ((unsigned)h ^ (unsigned)(h >> 32)) | 1u : (unsigned)(lane << 1);
    const unsigned peers = __match_any_sync(0xffffffffu, tag);
    const int leader = __ffs(peers) - 1;
    const int lx = __shfl_sync(0xffffffffu, kx, leader), ly = __shfl_sync(0xffffffffu, ky, leader),
              lz = __shfl_sync(0xffffffffu, kz, leader);
    if (!valid || (lane != leader && lx == kx && ly == ky && lz == kz)) return;
    unsigned bucket = 0;
    const int cand = tid;                  // == w * kSamples + step
    int r = probe<false>(a.tab, a.cand_keys, 0, kx, ky, kz, &bucket);   // read-only fast path
    if (r == kResMiss) {
        int* ck = a.cand_keys + 3 * (size_t)cand;
        ck[0] = kx;
        ck[1] = ky;
        ck[2] = kz;
        __threadfence();   // the candidate key must be visible before its marker is
        r = probe<true>(a.tab, a.cand_keys, cand, kx, ky, kz, &bucket);
    }
    // (the exchange alone decides who is first in this frame: one round trip less than checking the stamp first;
    // only one lane per distinct key and warp gets here)
    const bool first_exist = r >= 0 && a.stamp && atomicExch(&a.stamp[r], a.frame_id) != a.frame_id;
    const bool first_new = r == kResInserted;
    if (r == kResFull) a.counters[2] = 1;
    // warp-aggregated list appends: one atomic per warp and list instead of one per block key
    const unsigned active = __activemask();
    const unsigned me = __ballot_sync(active, first_exist), mn = __ballot_sync(active, first_new);
    const unsigned lt = (1u << lane) - 1u;
    if (me) {
        const int lead = __ffs(me) - 1;
        int base = 0;
        if (lane == lead) base = atomicAdd(&a.counters[0], __popc(me));
        base = __shfl_sync(active, base, lead);
        if (first_exist) {
            const int p = base + __popc(me & lt);
            if (p < a.max_list) a.exist_list[p] = r;
            else a.counters[2] = 1;
        }
    }
    if (mn) {
        const int lead = __ffs(mn) - 1;
        int base = 0;
        if (lane == lead) base = atomicAdd(&a.counters[1], __popc(mn));
        base = __shfl_sync(active, base, lead);
        if (first_new) {
            const int p = base + __popc(mn & lt);
            if (p < a.max_list) a.new_list[p] = make_int2((int)bucket, cand);
            else a.counters[2] = 1;
        }
    }
}

// Stand-alone GetUniqueBlockCoordinates: the winners' keys are the unique set.
__global__ void emit_unique_keys_kernel(const int2* __restrict__ new_list, const int* __restrict__ counters,
                                        const int* __restrict__ cand_keys, int* __restrict__ out, int max_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = min(counters[1], max_out);
    if (i >= n) return;
    const int* k = cand_keys + 3 * (size_t)new_list[i].y;
    out[3 * i] = k[0];
    out[3 * i + 1] = k[1];
    out[3 * i + 2] = k[2];
}

// --------------------------------------------------- stand-alone hash ops

struct MapArgs {
    Table tab;
    int* keys_rw;        // committed key buffer (writable view of tab.keys)
    const int* in_keys;  // [n,3]
    int n;
    int* buf_indices;
    uint8_t* masks;
    int* bucket_of_input;  // scratch [n]
    int* size;             // device counter
    int capacity;
    int* overflow;
};

// HashMap::Activate pass 1: claim buckets with provisional markers (candidate id =
// input index; the candidate key array is the read-only input itself).
__global__ void activate_claim_kernel(MapArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    unsigned bucket = 0;
    const int r = probe<true>(a.tab, a.in_keys, i, a.in_keys[3 * i], a.in_keys[3 * i + 1], a.in_keys[3 * i + 2], &bucket);
    a.bucket_of_input[i] = r == kResInserted ? (int)bucket : -1;
    if (a.masks) a.masks[i] = r == kResInserted ? 1 : 0;
    if (r == kResFull) *a.overflow = 1;
}
// pass 2: winners pop a slot (CUDAHashBackendBufferAccessor.h:80-83 heap_top), publish key + slot.
__global__ void activate_commit_kernel(MapArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    const int b = a.bucket_of_input[i];
    if (b < 0) return;
    const int slot = atomicAdd(a.size, 1);
    if (slot >= a.capacity) {
        atomicSub(a.size, 1);
        a.tab.table[b] = kTomb;
        if (a.masks) a.masks[i] = 0;
        *a.overflow = 1;
        return;
    }
    a.keys_rw[3 * (size_t)slot] = a.in_keys[3 * i];
    a.keys_rw[3 * (size_t)slot + 1] = a.in_keys[3 * i + 1];
    a.keys_rw[3 * (size_t)slot + 2] = a.in_keys[3 * i + 2];
    a.tab.table[b] = slot;
}
// HashMap::Find (also pass 3 of Activate: every input learns its slot).
__global__ void find_kernel(MapArgs a, bool write_masks) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    unsigned bucket;
    const int r = probe<false>(a.tab, a.in_keys, 0, a.in_keys[3 * i], a.in_keys[3 * i + 1], a.in_keys[3 * i + 2], &bucket);
    if (a.buf_indices) a.buf_indices[i] = r >= 0 ? r : -1;
    if (write_masks && a.masks) a.masks[i] = r >= 0 ? 1 : 0;
}

__global__ void rehash_kernel(int* table, unsigned mask, const int* keys, int n) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    unsigned b = bucket_of(minivec_hash(keys[3 * s], keys[3 * s + 1], keys[3 * s + 2]), mask);
    for (;; b = (b + 1) & mask)
        if (atomicCAS(&table[b], kEmpty, s) == kEmpty) return;
}

__global__ void hash_keys_kernel(const int* __restrict__ keys, int64_t n, uint64_t* __restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) out[i] = minivec_hash(keys[3 * i], keys[3 * i + 1], keys[3 * i + 2]);
}

__global__ void iota_kernel(int* out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = i;
}

// --------------------------------------------------------------- integrate

struct IntegrateArgs {
    const void* depth;
    const void* color;       // may be null
    int rows, cols;
    Cam dcam;                // depth intrinsics + world->camera extrinsics, scale = voxel_size
    Cam ccam;                // colour intrinsics, identity extrinsics, scale 1
    float sdf_trunc, depth_scale, depth_max, color_multiplier;
    int resolution;          // 16 on the fast path
    const int* block_keys;   // [capacity,3]
    float* tsdf;
    uint16_t* weight;
    uint16_t* color_buf;     // may be null
    // list mode
    const int* buf_indices;
    int n_blocks;
    // fused mode (counters != nullptr): exist_list ++ new_list, commit on the fly
    const int* exist_list;
    const int2* new_list;
    const int* cand_keys;
    int* counters;           // [0] n_exist [1] n_new [2] overflow [3] ticket
    int* size;
    int* table;
    int* keys_rw;
    int* stamp;
    int* frame_slots;        // [max] slots of this frame's frustum blocks (Model::frustum_block_coords_)
    int* frame_count;
    int* max_new;            // running max of blocks first seen in one frame
    int* dropped;            // [0] capacity the first dropped frame needed, [1] its frame index + 1 (0 = none)
    int* host_status;        // pinned host memory, ring of 8 x 16 ints: the frame's status, written by the last CTA
    int* work;               // fused mode: dynamic work-unit counter (re-armed by the last CTA); null = static striding
    unsigned long long* exec_ns;   // fused mode: [0] earliest CTA start of this launch (re-armed by the last CTA), [1] sum over
                                   // launches of (last CTA end - earliest start), [2] launches — %globaltimer, unperturbed by events
    int frame_id;
    int frame_index;         // 0-based index of the fused frame (reported when a frame is dropped)
    int capacity;
    int max_list;            // size of exist_list / new_list
    // 16^3 fast path (integrate16_kernel)
    const float* inv_w;      // [65536] 1 / (w + 1), the reference's inv_wsum (VoxelBlockGridImpl.h:274) per u16 weight
    float inv_scale;         // RN(1 / depth_scale), used only when fast_scale
    int fast_scale;          // u16 depth: depth / depth_scale through a verified 3-FMA division (see depth_metres)
    int same_k;              // colour intrinsics == depth intrinsics: interior pixels map to themselves (see below)
    int use_tile;            // the depth image has a TMA descriptor: stage the projected tile in shared memory
};


// The last CTA of a fused frame publishes the frame's status straight into pinned HOST memory (a posted write over
// PCIe): slot frame_index & 7 of a ring, sequence tag last.  The host therefore learns sizes without a
// device-to-host copy or an event in the stream — the frame's two kernels stay adjacent, which programmatic
// dependent launch needs.
__device__ __forceinline__ void publish_status(const IntegrateArgs& a, int size_after, int n_new, int overflow,
                                               int frame_count, int max_new) {
    if (!a.host_status) return;
    volatile int* hs = a.host_status + 16 * (a.frame_index & 7);
    hs[0] = size_after;
    hs[5] = n_new;
    hs[6] = overflow;
    hs[8] = frame_count;
    hs[9] = max_new;
    hs[10] = a.dropped[0];
    hs[11] = a.dropped[1];
    __threadfence_system();
    hs[15] = a.frame_index + 1;
}

// VoxelBlockGridImpl.h:226-303 for one voxel.  Returns false if the voxel is not updated.
template <typename depth_t>
__device__ __forceinline__ bool voxel_sdf(const IntegrateArgs& a, int x, int y, int z, float& sdf, int& ui, int& vi) {
    float xc, yc, zc, u, v;
    rigid(a.dcam, (float)x, (float)y, (float)z, xc, yc, zc);
    project(a.dcam, xc, yc, zc, u, v);
    if (!in_boundary(u, v, a.rows, a.cols)) return false;
    ui = (int)u;
    vi = (int)v;
    const float depth = dvd((float)__ldg(&((const depth_t*)a.depth)[(size_t)vi * a.cols + ui]), a.depth_scale);
    sdf = sub(depth, zc);
    if (depth <= 0 || depth > a.depth_max || zc <= 0 || sdf < -a.sdf_trunc) return false;
    sdf = sdf < a.sdf_trunc ? sdf : a.sdf_trunc;
    sdf = dvd(sdf, a.sdf_trunc);
    return true;
}

// One 16^3 block per CTA iteration; each thread owns 4 consecutive x voxels per
// pass (128-bit tsdf, 64-bit weight, 3x64-bit colour accesses, fully coalesced).
// One quarter (4 z-slices = 1024 voxels) of a 16^3 block per CTA pass; each thread owns 4
// consecutive x voxels (128-bit tsdf, 64-bit weight, 3x64-bit colour accesses, fully coalesced).
template <typename depth_t, typename color_in_t, bool HAS_COLOR>
__device__ __forceinline__ void integrate_block16(const IntegrateArgs& a, int slot, int unit, int xb, int yb, int zb) {
    float* tsdf = a.tsdf + (size_t)slot * 4096;
    uint16_t* wt = a.weight + (size_t)slot * 4096;
    uint16_t* cb = HAS_COLOR ? a.color_buf + (size_t)slot * 4096 * 3 : nullptr;
    {
        const int quad = unit * kT + threadIdx.x;
        const int xq = (quad & 3) * 4, yv = (quad >> 2) & 15, zv = quad >> 6;
        const int lin = quad * 4;
        float sdf[4];
        int ui[4], vi[4];
        bool up[4];
        bool any = false;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            up[k] = voxel_sdf<depth_t>(a, xb * 16 + xq + k, yb * 16 + yv, zb * 16 + zv, sdf[k], ui[k], vi[k]);
            any |= up[k];
        }
        if (!any) return;
        float4 t4 = *reinterpret_cast<float4*>(tsdf + lin);
        ushort4 w4 = *reinterpret_cast<ushort4*>(wt + lin);
        float tv[4] = {t4.x, t4.y, t4.z, t4.w};
        unsigned short wv[4] = {w4.x, w4.y, w4.z, w4.w};
        unsigned short cv[12];
        if (HAS_COLOR) {
            const uint2* cp = reinterpret_cast<const uint2*>(cb + (size_t)lin * 3);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const uint2 c2 = cp[k];
                cv[4 * k + 0] = (unsigned short)(c2.x & 0xffffu);
                cv[4 * k + 1] = (unsigned short)(c2.x >> 16);
                cv[4 * k + 2] = (unsigned short)(c2.y & 0xffffu);
                cv[4 * k + 3] = (unsigned short)(c2.y >> 16);
            }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (!up[k]) continue;
            const float inv_wsum = dvd(1.0f, (float)((int)wv[k] + 1));   // :274
            const float weight = (float)wv[k];
            tv[k] = mul(add(mul(weight, tv[k]), sdf[k]), inv_wsum);     // :276
            if (HAS_COLOR) {
                float px, py, pz, uf, vf;
                unproject(a.dcam, (float)ui[k], (float)vi[k], 1.0f, px, py, pz);   // :283
                project(a.ccam, px, py, pz, uf, vf);                                 // :286
                if (in_boundary(uf, vf, a.rows, a.cols)) {
                    const int cu = (int)roundf(uf), cw = (int)roundf(vf);
                    const color_in_t* in = (const color_in_t*)a.color + ((size_t)cw * a.cols + cu) * 3;
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float v = mul(add(mul(weight, (float)cv[3 * k + c]),
                                                mul((float)__ldg(&in[c]), a.color_multiplier)),
                                            inv_wsum);                              // :295-298
                        cv[3 * k + c] = (unsigned short)v;
                    }
                }
            }
            wv[k] = (unsigned short)add(weight, 1.0f);                  // :302
        }
        *reinterpret_cast<float4*>(tsdf + lin) = make_float4(tv[0], tv[1], tv[2], tv[3]);
        *reinterpret_cast<ushort4*>(wt + lin) = make_ushort4(wv[0], wv[1], wv[2], wv[3]);
        if (HAS_COLOR) {
            uint2* cp = reinterpret_cast<uint2*>(cb + (size_t)lin * 3);
#pragma unroll
            for (int k = 0; k < 3; ++k)
                cp[k] = make_uint2((unsigned)cv[4 * k] | ((unsigned)cv[4 * k + 1] << 16),
                                   (unsigned)cv[4 * k + 2] | ((unsigned)cv[4 * k + 3] << 16));
        }
    }
}

// Generic resolution (any res, scalar accesses) and generic value layout — the parity path for res != 16 and for
// the reference's Float32 weight / Float32 colour instantiations (VoxelBlockGridCUDA.cu:238-244).
template <typename depth_t, typename color_in_t, bool HAS_COLOR, typename weight_t, typename color_t>
__device__ __forceinline__ void integrate_block_generic(const IntegrateArgs& a, int slot, int xb, int yb, int zb) {
    const int res = a.resolution, res3 = res * res * res;
    weight_t* wbuf = reinterpret_cast<weight_t*>(a.weight);
    color_t* cbuf = reinterpret_cast<color_t*>(a.color_buf);
    for (int vox = threadIdx.x; vox < res3; vox += kT) {
        const int xv = vox % res, yv = (vox / res) % res, zv = vox / (res * res);
        float sdf;
        int ui, vi;
        if (!voxel_sdf<depth_t>(a, xb * res + xv, yb * res + yv, zb * res + zv, sdf, ui, vi)) continue;
        const size_t lin = (size_t)slot * res3 + vox;
        const weight_t w = wbuf[lin];
        // :274  1.0f / (*weight_ptr + 1): an int sum for UInt16 weights, a float sum for Float32 weights
        const float inv_wsum = sizeof(weight_t) == 2 ? dvd(1.0f, (float)((int)w + 1)) : dvd(1.0f, add((float)w, 1.0f));
        const float weight = (float)w;
        a.tsdf[lin] = mul(add(mul(weight, a.tsdf[lin]), sdf), inv_wsum);
        if (HAS_COLOR) {
            float px, py, pz, uf, vf;
            unproject(a.dcam, (float)ui, (float)vi, 1.0f, px, py, pz);
            project(a.ccam, px, py, pz, uf, vf);
            if (in_boundary(uf, vf, a.rows, a.cols)) {
                const int cu = (int)roundf(uf), cw = (int)roundf(vf);
                const color_in_t* in = (const color_in_t*)a.color + ((size_t)cw * a.cols + cu) * 3;
                for (int c = 0; c < 3; ++c)
                    cbuf[3 * lin + c] = (color_t)mul(
                            add(mul(weight, (float)cbuf[3 * lin + c]), mul((float)in[c], a.color_multiplier)), inv_wsum);
            }
        }
        wbuf[lin] = (weight_t)add(weight, 1.0f);
    }
}

template <typename depth_t, typename color_in_t, bool HAS_COLOR, typename weight_t = uint16_t, typename color_t = uint16_t>
__global__ void __launch_bounds__(kT) integrate_kernel(IntegrateArgs a) {
    __shared__ int s_slot, s_key[3];
    const bool fused = a.counters != nullptr;
    int n_exist = 0, n_new = 0, n_total = a.n_blocks, size0 = 0;
    bool drop = false;
    pdl_wait();
    pdl_launch_dependents();
    if (fused) {   // same whole-frame drop rule as integrate16_kernel
        n_exist = a.counters[0];
        n_new = a.counters[1];
        size0 = *a.size;
        drop = a.counters[2] != 0 || size0 + n_new > a.capacity;
        n_total = drop ? 0 : n_exist + n_new;
        if (drop) {
            const int n_roll = min(n_new, a.max_list);
            for (int i = blockIdx.x * kT + threadIdx.x; i < n_roll; i += gridDim.x * kT) a.table[a.new_list[i].x] = kEmpty;
        }
    }
    // work unit = one quarter of a 16^3 block (whole block for other resolutions)
    constexpr bool kVec = sizeof(weight_t) == 2;     // the vectorised quarter-block path is the u16 / u16 layout's
    const int upb = (kVec && a.resolution == 16) ? 4 : 1;
    for (int wu = blockIdx.x; wu < n_total * upb; wu += gridDim.x) {
        const int b = wu / upb, unit = wu % upb;
        if (threadIdx.x == 0) {
            int slot;
            const int* k;
            if (!fused) {
                slot = a.buf_indices[b];
                k = a.block_keys + 3 * (size_t)slot;
            } else if (b < n_exist) {
                slot = a.exist_list[b];
                k = a.block_keys + 3 * (size_t)slot;
            } else {
                // a block first seen in this frame: slot = old size + rank; unit 0 commits it
                const int2 nl = a.new_list[b - n_exist];
                slot = size0 + (b - n_exist);
                k = a.cand_keys + 3 * (size_t)nl.y;
                if (unit == 0) {
                    a.keys_rw[3 * (size_t)slot] = k[0];
                    a.keys_rw[3 * (size_t)slot + 1] = k[1];
                    a.keys_rw[3 * (size_t)slot + 2] = k[2];
                    a.stamp[slot] = a.frame_id;
                    a.table[nl.x] = slot;
                }
            }
            s_slot = slot;
            if (slot >= 0) {
                s_key[0] = k[0];
                s_key[1] = k[1];
                s_key[2] = k[2];
                if (fused && unit == 0) a.frame_slots[b] = slot;
            }
        }
        __syncthreads();
        const int slot = s_slot;
        if (slot >= 0) {
            if (kVec && a.resolution == 16) integrate_block16<depth_t, color_in_t, HAS_COLOR>(a, slot, unit, s_key[0], s_key[1], s_key[2]);
            else integrate_block_generic<depth_t, color_in_t, HAS_COLOR, weight_t, color_t>(a, slot, s_key[0], s_key[1], s_key[2]);
        }
        __syncthreads();
    }
    if (fused) {
        // last CTA publishes the new size and re-arms the per-frame counters
        __shared__ bool s_last;
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) s_last = atomicAdd(&a.counters[3], 1) == (int)gridDim.x - 1;
        __syncthreads();
        if (s_last && threadIdx.x == 0) {
            if (drop) {
                *a.frame_count = 0;
                if (a.dropped[1] == 0) {
                    a.dropped[0] = size0 + n_new;
                    a.dropped[1] = a.frame_index + 1;
                }
                a.counters[2] = 1;
            } else {
                *a.frame_count = n_total;
                *a.size = size0 + n_new;
            }
            if (n_new > *a.max_new) *a.max_new = n_new;
            a.counters[0] = 0;
            a.counters[1] = 0;
            a.counters[3] = 0;
            publish_status(a, drop ? size0 : size0 + n_new, n_new, drop ? 1 : 0, drop ? 0 : n_total, *a.max_new);
            // counters[2] (overflow) is sticky until the host reads it
        }
    }
}


// ------------------------------------------ integrate, 16^3 blocks: TMA-staged depth tile

static constexpr int kTileRows = 96;        // rows of the staged depth tile
static constexpr int kTileRowBytes = 256;   // 128 u16 / 64 f32 pixels per row
static constexpr unsigned kTileBytes = kTileRows * kTileRowBytes;

// depth / depth_scale (VoxelBlockGridImpl.h:253).  For u16 images the quotient has only 65536 possible
// numerators: the host checks ONCE per scale, over all of them, that the division-free sequence
// q = d y, r = fma(-q, s, d), q' = fma(r, y, q) with y = RN(1/s) returns exactly RN(d / s) (Markstein's
// correction step; same IEEE operations on host and device), and only then sets fast_scale.
template <typename depth_t>
__device__ __forceinline__ float depth_metres(const IntegrateArgs& a, depth_t raw) {
    const float d = (float)raw;
    if (sizeof(depth_t) == 2 && a.fast_scale) {
        const float q = __fmul_rn(d, a.inv_scale);
        const float r = __fmaf_rn(-q, a.depth_scale, d);
        return __fmaf_rn(r, a.inv_scale, q);
    }
    return dvd(d, a.depth_scale);
}

// One launch integrates a frame into 16^3 blocks.  Work unit = a quarter block (4 z-slices, 1024 voxels, 4
// consecutive x voxels per thread).  Per unit and CTA:
//   * thread 32 fetches the NEXT unit's slot / block key (and commits the block if this frame created it)
//     while the current unit is computed: the list -> key dependent loads are off the critical path;
//   * warp 0 projects the unit's 8 corners, and lane 0 issues ONE 2-D TMA load of the bounding pixel rectangle of
//     the depth image into shared memory (out-of-image parts zero-filled), completion on an mbarrier;
//   * every thread first issues its tsdf / weight (/ colour) loads, then does the voxel -> pixel geometry
//     (the IEEE divisions that make the result bit-exact) while the tile and the voxel values are in flight,
//     then waits on the mbarrier and reads its 4 depths from shared memory;
//   * one __syncthreads per unit (tile / metadata hand-over).
// Rectangles that do not fit the tile (very close blocks), units with a corner behind the camera and images
// without a descriptor read the depth image directly; every tile read is bounds-checked against the staged
// rectangle, so the staging can never change a result.
template <typename depth_t, typename color_in_t, bool HAS_COLOR>
__global__ void __launch_bounds__(kT) integrate16_kernel(const __grid_constant__ IntegrateArgs a,
                                                         const __grid_constant__ CUtensorMap dmap) {
    __shared__ __align__(128) unsigned char s_tile[kTileBytes];
    __shared__ __align__(8) unsigned long long s_mbar;
    __shared__ int s_meta[2][4];   // slot, block key
    __shared__ int s_rect[4];      // x0, y0 of the staged rectangle, staged?
    __shared__ int s_wu[2];        // work unit of this / the next trip (-1 = none left)
    __shared__ bool s_last;
    constexpr int kTileCols = kTileRowBytes / (int)sizeof(depth_t);
    const int tid = threadIdx.x;
    if (tid == 0) {
        mbar_init(&s_mbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    pdl_wait();                 // the touch kernel's lists / counters, the previous frame's size
    pdl_launch_dependents();
    if (a.exec_ns && tid == 0) atomicMin(&a.exec_ns[0], (unsigned long long)global_ns());
    const bool fused = a.counters != nullptr;
    int n_exist = 0, n_new = 0, n_total = a.n_blocks, size0 = 0;
    bool drop = false;
    if (fused) {
        n_exist = a.counters[0];
        n_new = a.counters[1];
        size0 = *a.size;
        // ONE decision for every CTA (all four values are final once the touch kernel has finished): a frame
        // whose new blocks do not fit, whose lists overflowed, or that follows a dropped frame, is dropped as
        // a whole — nothing integrated, its provisional table entries released — and reported by the host.
        drop = a.counters[2] != 0 || size0 + n_new > a.capacity;
        n_total = drop ? 0 : n_exist + n_new;
        if (drop) {
            // no committed key's probe chain passes over a bucket that was empty when the frame began, so
            // emptying every bucket this frame claimed restores the table exactly
            const int n_roll = min(n_new, a.max_list);
            for (int i = blockIdx.x * kT + tid; i < n_roll; i += gridDim.x * kT) a.table[a.new_list[i].x] = kEmpty;
        }
    }
    const int n_units = n_total * 4;

    auto fetch = [&](int wu, int buf) {    // one thread: metadata of work unit wu
        const int b = wu >> 2, unit = wu & 3;
        int slot;
        const int* k;
        if (!fused) {
            slot = a.buf_indices[b];
            k = a.block_keys + 3 * (size_t)slot;
        } else if (b < n_exist) {
            slot = a.exist_list[b];
            k = a.block_keys + 3 * (size_t)slot;
        } else {
            // a block first seen in this frame: slot = old size + rank; its unit 0 commits it
            const int2 nl = a.new_list[b - n_exist];
            slot = size0 + (b - n_exist);
            k = a.cand_keys + 3 * (size_t)nl.y;
            if (unit == 0) {
                a.keys_rw[3 * (size_t)slot] = k[0];
                a.keys_rw[3 * (size_t)slot + 1] = k[1];
                a.keys_rw[3 * (size_t)slot + 2] = k[2];
                a.stamp[slot] = a.frame_id;
                a.table[nl.x] = slot;
            }
        }
        if (fused && unit == 0) a.frame_slots[b] = slot;
        s_meta[buf][0] = slot;
        s_meta[buf][1] = k[0];
        s_meta[buf][2] = k[1];
        s_meta[buf][3] = k[2];
    };
    // Work units are handed out dynamically after the first one per CTA (units differ a lot in cost: a quarter block
    // behind the surface leaves at the truncation test), so the grid drains evenly instead of waiting for the CTAs
    // that drew one unit more.
    if (tid == 32) {
        const int first = (int)blockIdx.x < n_units ? (int)blockIdx.x : -1;
        s_wu[0] = first;
        if (first >= 0) fetch(first, 0);
    }

    for (int it = 0;; ++it) {
        __syncthreads();   // unit + metadata published; every thread is done with the previous tile / rect
        const int wu = s_wu[it & 1];
        if (wu < 0) break;
        const int slot = s_meta[it & 1][0];
        const int xb = s_meta[it & 1][1], yb = s_meta[it & 1][2], zb = s_meta[it & 1][3];
        const int unit = wu & 3;
        const int quad = unit * kT + tid;
        const int xq = (quad & 3) * 4, yv = (quad >> 2) & 15, zv = quad >> 6;
        const int lin = quad * 4;
        float* tsdf = a.tsdf + (size_t)slot * 4096 + lin;
        uint16_t* wt = a.weight + (size_t)slot * 4096 + lin;
        uint16_t* cb = HAS_COLOR ? a.color_buf + ((size_t)slot * 4096 + lin) * 3 : nullptr;
        // voxel values first: their DRAM latency overlaps the geometry below
        const float4 t4 = *reinterpret_cast<const float4*>(tsdf);
        const ushort4 w4 = *reinterpret_cast<const ushort4*>(wt);
        uint2 c2[3];
        if (HAS_COLOR) {
#pragma unroll
            for (int k = 0; k < 3; ++k) c2[k] = reinterpret_cast<const uint2*>(cb)[k];
        }
        if (tid < 32) {
            // bounding pixel rectangle of the unit's voxels: perspective projection maps the convex hull of
            // the 8 extreme voxels (all in front of the camera) into the hull of their projections
            const int c = tid & 7;
            float xc, yc, zc, u = 0.f, v = 0.f;
            rigid(a.dcam, (float)(xb * 16 + ((c & 1) ? 15 : 0)), (float)(yb * 16 + ((c & 2) ? 15 : 0)),
                  (float)(zb * 16 + unit * 4 + ((c & 4) ? 3 : 0)), xc, yc, zc);
            bool ok = zc > 1e-3f;
            if (ok) project(a.dcam, xc, yc, zc, u, v);
            ok = ok && fabsf(u) < 1e6f && fabsf(v) < 1e6f;
            float umin = u, umax = u, vmin = v, vmax = v;
#pragma unroll
            for (int o = 1; o < 8; o <<= 1) {
                umin = fminf(umin, __shfl_xor_sync(0xffffffffu, umin, o));
                umax = fmaxf(umax, __shfl_xor_sync(0xffffffffu, umax, o));
                vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, o));
                vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
            }
            ok = __all_sync(0xffffffffu, ok);
            if (tid == 0) {
                // the box must start on a 16-byte boundary of the image row (TMA requirement): round x0 down
                const int x0 = ((int)floorf(umin) - 1) & ~(16 / (int)sizeof(depth_t) - 1), x1 = (int)floorf(umax) + 1;
                const int y0 = (int)floorf(vmin) - 1, y1 = (int)floorf(vmax) + 1;
                const bool stage = a.use_tile && ok && x1 - x0 < kTileCols && y1 - y0 < kTileRows && x1 >= 0 && y1 >= 0 &&
                                   x0 < a.cols && y0 < a.rows;
                s_rect[0] = x0;
                s_rect[1] = y0;
                s_rect[2] = stage ? 1 : 0;
                if (stage) {
                    mbar_arrive_expect_tx(&s_mbar, kTileBytes);
                    tma_load_2d(s_tile, &dmap, x0, y0, &s_mbar);
                } else {
                    mbar_arrive(&s_mbar);   // (release: s_rect is visible to every waiter)
                }
            }
        } else if (tid == 32) {
            int next = a.work ? (int)gridDim.x + atomicAdd(a.work, 1) : wu + (int)gridDim.x;
            if (next >= n_units) next = -1;
            s_wu[(it + 1) & 1] = next;
            if (next >= 0) fetch(next, (it + 1) & 1);
        }
        // VoxelBlockGridImpl.h:226-247: voxel -> camera -> pixel, uncontracted, reference order; the y / z
        // products are shared by the thread's 4 voxels
        const float ys = mul((float)(yb * 16 + yv), a.dcam.scale), zs = mul((float)(zb * 16 + zv), a.dcam.scale);
        float py[3], pz[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            py[r] = mul(ys, a.dcam.e[r][1]);
            pz[r] = mul(zs, a.dcam.e[r][2]);
        }
        float zc[4];
        int pix[4];       // ui | vi << 16, -1 = outside the image
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float xs = mul((float)(xb * 16 + xq + k), a.dcam.scale);
            const float xc = add(add(add(mul(xs, a.dcam.e[0][0]), py[0]), pz[0]), a.dcam.e[0][3]);
            const float yc = add(add(add(mul(xs, a.dcam.e[1][0]), py[1]), pz[1]), a.dcam.e[1][3]);
            zc[k] = add(add(add(mul(xs, a.dcam.e[2][0]), py[2]), pz[2]), a.dcam.e[2][3]);
            float u, v;
            project(a.dcam, xc, yc, zc[k], u, v);
            pix[k] = in_boundary(u, v, a.rows, a.cols) ? ((int)u | ((int)v << 16)) : -1;
        }
        mbar_wait(&s_mbar, (unsigned)it & 1u);
        const int rx0 = s_rect[0], ry0 = s_rect[1];
        const bool staged = s_rect[2] != 0;
        const depth_t* tile = reinterpret_cast<const depth_t*>(s_tile);
        float tv[4] = {t4.x, t4.y, t4.z, t4.w};
        unsigned short wv[4] = {w4.x, w4.y, w4.z, w4.w};
        unsigned short cv[12];
        if (HAS_COLOR) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                cv[4 * k + 0] = (unsigned short)(c2[k].x & 0xffffu);
                cv[4 * k + 1] = (unsigned short)(c2[k].x >> 16);
                cv[4 * k + 2] = (unsigned short)(c2[k].y & 0xffffu);
                cv[4 * k + 3] = (unsigned short)(c2[k].y >> 16);
            }
        }
        bool any = false;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (pix[k] < 0) continue;
            const int ui = pix[k] & 0xffff, vi = pix[k] >> 16;
            const int tx = ui - rx0, ty = vi - ry0;
            const depth_t raw = (staged && (unsigned)tx < (unsigned)kTileCols && (unsigned)ty < (unsigned)kTileRows)
                                        ? tile[ty * kTileCols + tx]
                                        : __ldg(&((const depth_t*)a.depth)[(size_t)vi * a.cols + ui]);
            const float depth = depth_metres<depth_t>(a, raw);                      // :253
            float sdf = sub(depth, zc[k]);
            if (depth <= 0 || depth > a.depth_max || zc[k] <= 0 || sdf < -a.sdf_trunc) continue;   // :256-258
            sdf = sdf < a.sdf_trunc ? sdf : a.sdf_trunc;
            sdf = dvd(sdf, a.sdf_trunc);
            any = true;
            const float inv_wsum = __ldg(&a.inv_w[wv[k]]);                           // :274, 1 / (w + 1) per u16 weight
            const float weight = (float)wv[k];
            tv[k] = mul(add(mul(weight, tv[k]), sdf), inv_wsum);                    // :276
            if (HAS_COLOR) {
                int cu, cw;
                bool inb;
                if (a.same_k && ui >= 1 && vi >= 1 && ui <= a.cols - 2 && vi <= a.rows - 2) {
                    // :283-290 with identical intrinsics: uf = (fx ((ui - cx) / fx)) + cx differs from ui by
                    // a few ulps of the image width (<< 0.5), so round(uf) == ui and an INTERIOR pixel is
                    // always inside the boundary; border pixels take the general path below
                    cu = ui;
                    cw = vi;
                    inb = true;
                } else {
                    float px, pyy, pzz, uf, vf;
                    unproject(a.dcam, (float)ui, (float)vi, 1.0f, px, pyy, pzz);   // :283
                    project(a.ccam, px, pyy, pzz, uf, vf);                           // :286
                    inb = in_boundary(uf, vf, a.rows, a.cols);
                    cu = (int)roundf(uf);
                    cw = (int)roundf(vf);
                }
                if (inb) {
                    const color_in_t* in = (const color_in_t*)a.color + ((size_t)cw * a.cols + cu) * 3;
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float v = mul(add(mul(weight, (float)cv[3 * k + c]),
                                                mul((float)__ldg(&in[c]), a.color_multiplier)),
                                            inv_wsum);                              // :295-298
                        cv[3 * k + c] = (unsigned short)v;
                    }
                }
            }
            wv[k] = (unsigned short)add(weight, 1.0f);                              // :302
        }
        if (any) {
            *reinterpret_cast<float4*>(tsdf) = make_float4(tv[0], tv[1], tv[2], tv[3]);
            *reinterpret_cast<ushort4*>(wt) = make_ushort4(wv[0], wv[1], wv[2], wv[3]);
            if (HAS_COLOR) {
#pragma unroll
                for (int k = 0; k < 3; ++k)
                    reinterpret_cast<uint2*>(cb)[k] = make_uint2((unsigned)cv[4 * k] | ((unsigned)cv[4 * k + 1] << 16),
                                                                 (unsigned)cv[4 * k + 2] | ((unsigned)cv[4 * k + 3] << 16));
            }
        }
    }
    if (fused) {
        // last CTA publishes the new size and re-arms the per-frame counters
        __threadfence();
        __syncthreads();
        if (tid == 0) s_last = atomicAdd(&a.counters[3], 1) == (int)gridDim.x - 1;
        __syncthreads();
        if (s_last && tid == 0) {
            if (drop) {
                *a.frame_count = 0;
                if (a.dropped[1] == 0) {          // first dropped frame: what it needed, and which one it was
                    a.dropped[0] = size0 + n_new;
                    a.dropped[1] = a.frame_index + 1;
                }
                a.counters[2] = 1;                // sticky: later frames are dropped too until the host reserves
            } else {
                *a.frame_count = n_total;
                *a.size = size0 + n_new;
            }
            if (n_new > *a.max_new) *a.max_new = n_new;
            a.counters[0] = 0;
            a.counters[1] = 0;
            a.counters[3] = 0;
            if (a.work) *a.work = 0;
            if (a.exec_ns) {
                const unsigned long long now = global_ns();
                a.exec_ns[1] += now - a.exec_ns[0];
                a.exec_ns[2] += 1;
                a.exec_ns[0] = ~0ull;
            }
            publish_status(a, drop ? size0 : size0 + n_new, n_new, drop ? 1 : 0, drop ? 0 : n_total, *a.max_new);
        }
    }
}

__global__ void inv_weight_table_kernel(float* __restrict__ out) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w < 65536) out[w] = dvd(1.0f, (float)(w + 1));   // VoxelBlockGridImpl.h:274 inv_wsum for weight w
}

__global__ void gather_keys_kernel(const int* __restrict__ keys, const int* __restrict__ slots, int n,
                                   int* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = slots[i];
    out[3 * i] = keys[3 * (size_t)s];
    out[3 * i + 1] = keys[3 * (size_t)s + 1];
    out[3 * i + 2] = keys[3 * (size_t)s + 2];
}

}  // namespace o3db

using namespace o3db;


namespace o3db {


// cuTensorMapEncodeTiled, resolved at run time through the runtime API (no link against libcuda).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            p = nullptr;
        (void)cudaGetLastError();
        return (EncodeTiledFn)p;
    }();
    return fn;
}

// TMA descriptor of a row-major [rows][cols] depth image for kTileRowBytes x kTileRows boxes.  Returns false when
// the image cannot be described (unaligned base / pitch, tiny image, no driver entry point): the kernel then
// reads the image directly.
static bool make_depth_tensor_map(CUtensorMap* map, const void* depth, int depth_dtype, int rows, int cols) {
    memset(map, 0, sizeof(*map));
    const size_t es = depth_dtype == O3DB_DEPTH_U16 ? 2 : 4;
    const int box_cols = (int)(kTileRowBytes / es);
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc || ((uintptr_t)depth & 15) || ((size_t)cols * es) % 16 || cols < box_cols || rows < kTileRows) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)cols * es};
    const cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)kTileRows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = enc(map, depth_dtype == O3DB_DEPTH_U16 ? CU_TENSOR_MAP_DATA_TYPE_UINT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32,
                           2, const_cast<void*>(depth), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// Is q' = fma(fma(-d y, s, d), y, d y), y = RN(1 / s), equal to RN(d / s) for EVERY u16 d?  (See depth_metres.)
static bool verify_fast_scale(float s) {
    if (!(s > 0.f) || !std::isfinite(s)) return false;
    const float y = 1.0f / s;
    for (int i = 0; i < 65536; ++i) {
        const float d = (float)i;
        const float q = d * y;
        const float r = fmaf(-q, s, d);
        if (fmaf(r, y, q) != d / s) return false;
    }
    return true;
}

// 1 / (w + 1) for every u16 weight: one table per device, built once (and synchronised once), shared by all
// handles and by the stateless entry points.
static const float* inv_weight_table() {
    static float* tab[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    if (!tab[dev]) {
        float* p = nullptr;
        if (cudaMalloc(&p, 65536 * sizeof(float)) != cudaSuccess) return nullptr;
        inv_weight_table_kernel<<<65536 / kT, kT>>>(p);
        count_launch();
        if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) {
            cudaFree(p);
            return nullptr;
        }
        tab[dev] = p;
    }
    return tab[dev];
}

static unsigned pow2_at_least(int64_t v) {
    unsigned p = 16;
    while ((int64_t)p < v) p <<= 1;
    return p;
}

static size_t res3(const o3db_vbg* v) { return (size_t)v->resolution * v->resolution * v->resolution; }

static int alloc_map(o3db_vbg* v, int64_t capacity, cudaStream_t st) {
    v->capacity = capacity;
    v->nbuckets = pow2_at_least(2 * capacity);
    const size_t r3 = res3(v);
    O3DB_CUDA_CHECK(cudaMallocAsync(&v->table, (size_t)v->nbuckets * sizeof(int), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&v->keys, (size_t)capacity * 3 * sizeof(int), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&v->stamp, (size_t)capacity * sizeof(int), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&v->tsdf, (size_t)capacity * r3 * sizeof(float), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&v->weight, (size_t)capacity * r3 * sizeof(uint16_t), st));
    if (v->with_color) O3DB_CUDA_CHECK(cudaMallocAsync(&v->color, (size_t)capacity * r3 * 3 * sizeof(uint16_t), st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(v->table, 0xff, (size_t)v->nbuckets * sizeof(int), st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(v->keys, 0, (size_t)capacity * 3 * sizeof(int), st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(v->stamp, 0xff, (size_t)capacity * sizeof(int), st));
    // value buffers are zero-initialised at allocation (CUDAHashBackendBufferAccessor.h:56-57)
    O3DB_CUDA_CHECK(cudaMemsetAsync(v->tsdf, 0, (size_t)capacity * r3 * sizeof(float), st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(v->weight, 0, (size_t)capacity * r3 * sizeof(uint16_t), st));
    if (v->with_color) O3DB_CUDA_CHECK(cudaMemsetAsync(v->color, 0, (size_t)capacity * r3 * 3 * sizeof(uint16_t), st));
    return O3DB_OK;
}

static int ensure_frame_scratch(o3db_vbg* v, int rows, int cols, cudaStream_t st) {
    const int64_t need = (int64_t)(rows / kStride) * (cols / kStride) * kSamples;   // VoxelBlockGrid.cpp:225-227
    if (need <= v->frustum_cap) return O3DB_OK;
    if (v->cand_keys) {
        cudaFreeAsync(v->cand_keys, st);
        cudaFreeAsync(v->exist_list, st);
        cudaFreeAsync(v->new_list, st);
        cudaFreeAsync(v->frame_slots, st);
        cudaFreeAsync(v->ftable, st);
    }
    v->frustum_cap = need;
    v->fbuckets = pow2_at_least(2 * need);
    O3DB_CUDA_CHECK(cudaMallocAsync(&v->cand_keys, (size_t)need * 3 * sizeof(int), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&v->exist_list, (size_t)need * sizeof(int), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&v->new_list, (size_t)need * sizeof(int2), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&v->frame_slots, (size_t)need * sizeof(int), st));
    O3DB_CUDA_CHECK(cudaMallocAsync(&v->ftable, (size_t)v->fbuckets * sizeof(int), st));
    return O3DB_OK;
}

static int grow(o3db_vbg* v, int64_t new_capacity, cudaStream_t st) {
    // HashMap::Reserve (HashMap.cpp:47-77): upstream re-inserts active entries into
    // new buffers; here slots keep their indices, only the table is rebuilt.
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    int size = 0;
    O3DB_CUDA_CHECK(cudaMemcpy(&size, v->size_dev, sizeof(int), cudaMemcpyDeviceToHost));
    o3db_vbg old = *v;
    int rc = alloc_map(v, new_capacity, st);
    if (rc) return rc;
    const size_t r3 = res3(v);
    if (size > 0) {
        O3DB_CUDA_CHECK(cudaMemcpyAsync(v->keys, old.keys, (size_t)size * 3 * sizeof(int), cudaMemcpyDeviceToDevice, st));
        O3DB_CUDA_CHECK(cudaMemcpyAsync(v->stamp, old.stamp, (size_t)size * sizeof(int), cudaMemcpyDeviceToDevice, st));
        O3DB_CUDA_CHECK(cudaMemcpyAsync(v->tsdf, old.tsdf, (size_t)size * r3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
        O3DB_CUDA_CHECK(cudaMemcpyAsync(v->weight, old.weight, (size_t)size * r3 * sizeof(uint16_t), cudaMemcpyDeviceToDevice, st));
        if (v->with_color)
            O3DB_CUDA_CHECK(cudaMemcpyAsync(v->color, old.color, (size_t)size * r3 * 3 * sizeof(uint16_t), cudaMemcpyDeviceToDevice, st));
        rehash_kernel<<<(unsigned)ceil_div(size, kT), kT, 0, st>>>(v->table, v->nbuckets - 1, v->keys, size);
        O3DB_LAUNCH_CHECK();
    }
    cudaFreeAsync(old.table, st);
    cudaFreeAsync(old.keys, st);
    cudaFreeAsync(old.stamp, st);
    cudaFreeAsync(old.tsdf, st);
    cudaFreeAsync(old.weight, st);
    if (old.color) cudaFreeAsync(old.color, st);
    return O3DB_OK;
}

static int absorb_status(o3db_vbg* v, const int* h) {
    v->known_size = h[0];
    v->max_new_seen = std::max<int64_t>(v->max_new_seen, h[9]);
    if (h[6]) {
        // Frames are atomic and ordered on the device: a frame whose new blocks did not fit (HashMap::Activate would
        // have grown the map, HashMap.cpp:166-181) and every frame after it were dropped whole — nothing integrated,
        // the table restored — so the volume is exactly the state before that frame.
        set_last_error("voxel block hash map capacity (%lld blocks) exceeded: fused frame #%d needed %d blocks; that frame "
                       "and all later ones were dropped (volume unchanged).  Call o3db_vbg_reserve with a larger capacity "
                       "and resubmit from that frame.",
                       (long long)v->capacity, h[11] - 1, h[10]);
        return O3DB_ERR_CAPACITY;
    }
    return O3DB_OK;
}

// size_dev layout: [0] size, [4] n_exist [5] n_new [6] overflow [7] ticket, [8] frame_count, [9] max_new,
// [10] blocks the first dropped frame needed, [11] its frame id (0 = no frame dropped)
static int read_status(o3db_vbg* v, cudaStream_t st) {
    O3DB_CUDA_CHECK(cudaMemcpyAsync(v->h_pinned, v->size_dev, 16 * sizeof(int), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    return absorb_status(v, v->h_pinned);
}

// Launches the integrate kernel for the input dtypes (VoxelBlockGridCUDA.cu:238-244, value layout u16 weight /
// u16 colour): the 16^3 fast path with its TMA-staged depth tile, or the generic-resolution kernel.
template <typename depth_t, typename color_in_t, bool HAS_COLOR>
static int launch_integrate_typed(o3db_vbg* v, IntegrateArgs& a, int depth_dtype, unsigned grid, cudaStream_t st) {
    cudaError_t e;
    if (v->resolution == 16 && a.rows <= 32767 && a.cols <= 65535) {
        CUtensorMap map;
        a.use_tile = make_depth_tensor_map(&map, a.depth, depth_dtype, a.rows, a.cols) ? 1 : 0;
        if (!a.use_tile) memset(&map, 0, sizeof(map));
        e = launch_pdl_ex(integrate16_kernel<depth_t, color_in_t, HAS_COLOR>, {grid, kT}, st, a, map);
    } else {
        e = launch_pdl_ex(integrate_kernel<depth_t, color_in_t, HAS_COLOR>, {grid, kT}, st, a);
    }
    count_launch();
    if (e != cudaSuccess) {
        set_last_error("integrate kernel launch failed: %s", cudaGetErrorString(e));
        return O3DB_ERR_CUDA;
    }
    return O3DB_OK;
}

static int launch_integrate(o3db_vbg* v, IntegrateArgs& a, int depth_dtype, int color_dtype, bool has_color, unsigned grid,
                            cudaStream_t st) {
    if (depth_dtype == O3DB_DEPTH_U16) {
        if (!has_color) return launch_integrate_typed<uint16_t, uint8_t, false>(v, a, depth_dtype, grid, st);
        if (color_dtype == O3DB_COLOR_U8) return launch_integrate_typed<uint16_t, uint8_t, true>(v, a, depth_dtype, grid, st);
        set_last_error("u16 depth requires u8 color (kernel/VoxelBlockGrid.cpp:107-146)");
        return O3DB_ERR_INVALID;
    }
    if (depth_dtype == O3DB_DEPTH_F32) {
        if (!has_color) return launch_integrate_typed<float, float, false>(v, a, depth_dtype, grid, st);
        if (color_dtype == O3DB_COLOR_F32) return launch_integrate_typed<float, float, true>(v, a, depth_dtype, grid, st);
        set_last_error("f32 depth requires f32 color (kernel/VoxelBlockGrid.cpp:107-146)");
        return O3DB_ERR_INVALID;
    }
    set_last_error("Unsupported depth dtype");
    return O3DB_ERR_INVALID;
}

// Resident CTAs per SM of the integrate kernels (the persistent grids are sized from it).
static unsigned integrate_grid() {
    static int per_sm = 0;
    if (per_sm == 0) {
        int n = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, integrate16_kernel<uint16_t, uint8_t, true>, kT, 0) != cudaSuccess || n <= 0)
            n = 4;
        per_sm = n;
    }
    return (unsigned)(num_sms() * per_sm);
}

static IntegrateArgs base_integrate_args(o3db_vbg* v, const void* depth, const void* color, int color_dtype, int rows,
                                         int cols, const double* dK, const double* cK, const double* E,
                                         float depth_scale, float depth_max, float trunc_mult) {
    IntegrateArgs a{};
    a.depth = depth;
    a.color = color;
    a.rows = rows;
    a.cols = cols;
    a.dcam = make_cam(dK, E, v->voxel_size);                       // VoxelBlockGridImpl.h:184
    const double eye[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    a.ccam = make_cam(cK ? cK : dK, eye, 1.0f);                     // :185-187
    a.sdf_trunc = v->voxel_size * trunc_mult;                       // VoxelBlockGrid.cpp:325
    a.depth_scale = depth_scale;
    a.depth_max = depth_max;
    a.color_multiplier = color_dtype == O3DB_COLOR_F32 ? 255.0f : 1.0f;   // VoxelBlockGridImpl.h:216-218
    a.resolution = v->resolution;
    a.block_keys = v->keys;
    a.tsdf = v->tsdf;
    a.weight = v->weight;
    a.color_buf = v->color;
    a.capacity = (int)v->capacity;
    a.max_list = (int)v->frustum_cap;
    a.dropped = v->size_dev + 10;
    a.inv_w = v->inv_w;
    if (v->checked_scale != depth_scale) {     // one 65536-value host check per scale (see depth_metres)
        v->checked_scale = depth_scale;
        v->checked_scale_ok = verify_fast_scale(depth_scale);
    }
    a.fast_scale = v->checked_scale_ok ? 1 : 0;
    a.inv_scale = 1.0f / depth_scale;
    // colour intrinsics identical to the depth intrinsics (what slam::Model passes) and sane: interior pixels map to
    // themselves (integrate16_kernel); anything else takes the reference's unproject / project per voxel
    a.same_k = (a.ccam.fx == a.dcam.fx && a.ccam.fy == a.dcam.fy && a.ccam.cx == a.dcam.cx && a.ccam.cy == a.dcam.cy &&
                a.dcam.fx > 1e-3f && a.dcam.fy > 1e-3f && std::isfinite(a.dcam.fx) && std::isfinite(a.dcam.fy) &&
                fabsf(a.dcam.cx) < 1e5f && fabsf(a.dcam.cy) < 1e5f && rows <= 16384 && cols <= 16384)
                       ? 1 : 0;
    return a;
}

static int check_images(const void* depth, int depth_dtype, const void* color, int color_dtype, int rows, int cols) {
    O3DB_REQUIRE(depth != nullptr && rows > 0 && cols > 0, "depth image is empty");
    O3DB_REQUIRE(depth_dtype == O3DB_DEPTH_U16 || depth_dtype == O3DB_DEPTH_F32, "Unsupported depth image dtype");
    O3DB_REQUIRE(color == nullptr || color_dtype == O3DB_COLOR_U8 || color_dtype == O3DB_COLOR_F32,
                 "Unsupported color image dtype");
    return O3DB_OK;
}

static TouchArgs make_touch_args(o3db_vbg* v, const void* depth, int rows, int cols, const double* K, const double* E,
                                 float depth_scale, float depth_max, float trunc_mult) {
    TouchArgs t{};
    double pose[16];
    inverse_transformation(E, pose);               // VoxelBlockGridCUDA.cu:119
    t.depth = depth;
    t.rows = rows;
    t.cols = cols;
    t.cam = make_cam(K, pose, 1.0f);               // :120
    t.block_size = v->voxel_size * v->resolution;  // :143
    t.sdf_trunc = v->voxel_size * trunc_mult;      // VoxelBlockGrid.cpp:241
    t.depth_scale = depth_scale;
    t.depth_max = depth_max;
    t.cand_keys = v->cand_keys;
    t.new_list = v->new_list;
    t.exist_list = v->exist_list;
    t.counters = v->counters;
    t.max_list = (int)v->frustum_cap;
    return t;
}

}  // namespace o3db

extern "C" {

int o3db_vbg_create(float voxel_size, int block_resolution, int64_t block_count, int with_color, void* stream,
                    o3db_vbg** out) {
    O3DB_REQUIRE(out != nullptr, "o3db_vbg_create: out is null");
    *out = nullptr;
    O3DB_REQUIRE(voxel_size > 0, "voxel_size must be positive");
    O3DB_REQUIRE(block_resolution >= 1 && block_resolution <= 32, "block_resolution must be in 1..32");
    O3DB_REQUIRE(block_count >= 1 && block_count < (int64_t(1) << 29), "block_count out of range");
    configure_memory_pool();
    cudaStream_t st = (cudaStream_t)stream;
    o3db_vbg* v = new (std::nothrow) o3db_vbg();
    O3DB_REQUIRE(v != nullptr, "out of host memory");
    v->voxel_size = voxel_size;
    v->resolution = block_resolution;
    v->with_color = with_color != 0;
    int rc = alloc_map(v, block_count, st);
    cudaError_t e = cudaSuccess;
    if (rc == O3DB_OK) e = cudaMallocAsync(&v->size_dev, 16 * sizeof(int), st);
    if (rc == O3DB_OK && e == cudaSuccess) e = cudaMemsetAsync(v->size_dev, 0, 16 * sizeof(int), st);
    if (rc == O3DB_OK && e == cudaSuccess) {
        v->h_pinned = (int*)pinned_acquire(kPinnedInts * sizeof(int));
        if (!v->h_pinned) e = cudaErrorMemoryAllocation;
    }
    if (rc == O3DB_OK && e == cudaSuccess) e = cudaEventCreateWithFlags(&v->ev[0], cudaEventDisableTiming);
    if (rc == O3DB_OK && e == cudaSuccess) e = cudaEventCreateWithFlags(&v->ev[1], cudaEventDisableTiming);
    if (rc != O3DB_OK || e != cudaSuccess) {
        if (e != cudaSuccess) {
            set_last_error("o3db_vbg_create: %s", cudaGetErrorString(e));
            rc = O3DB_ERR_CUDA;
        }
        o3db_vbg_destroy(v);
        return rc;
    }
    v->counters = v->size_dev + 4;
    v->frame_count = v->size_dev + 8;
    memset(v->h_pinned, 0, kPinnedInts * sizeof(int));
    if (cudaMalloc(&v->exec_ns, 3 * sizeof(unsigned long long)) == cudaSuccess) {
        const unsigned long long init[3] = {~0ull, 0ull, 0ull};
        cudaMemcpy(v->exec_ns, init, sizeof(init), cudaMemcpyHostToDevice);
    } else {
        v->exec_ns = nullptr;
        (void)cudaGetLastError();
    }
    v->inv_w = inv_weight_table();
    if (!v->inv_w) {
        set_last_error("o3db_vbg_create: could not build the weight table: %s", cudaGetErrorString(cudaGetLastError()));
        o3db_vbg_destroy(v);
        return O3DB_ERR_CUDA;
    }
    *out = v;
    return O3DB_OK;
}

void o3db_vbg_destroy(o3db_vbg* v) {
    if (!v) return;
    cudaDeviceSynchronize();
    void* ptrs[] = {v->table, v->keys, v->stamp, v->size_dev, v->tsdf, v->weight, v->color, v->cand_keys,
                    v->exist_list, v->new_list, v->frame_slots, v->ftable, v->exec_ns, v->d_depth[0], v->d_depth[1],
                    v->d_color[0], v->d_color[1]};
    for (void* p : ptrs)
        if (p) cudaFree(p);
    if (v->h_pinned) pinned_release(v->h_pinned);
    for (auto& e : v->ev)
        if (e) cudaEventDestroy(e);
    for (auto& e : v->prof_ev)
        if (e) cudaEventDestroy(e);
    for (int i = 0; i < 2; ++i) {
        if (v->copied[i]) cudaEventDestroy(v->copied[i]);
        if (v->consumed[i]) cudaEventDestroy(v->consumed[i]);
    }
    if (v->copy_stream) cudaStreamDestroy(v->copy_stream);
    delete v;
}

int64_t o3db_vbg_size(o3db_vbg* v, void* stream) {
    if (!v) return O3DB_ERR_INVALID;
    int rc = read_status(v, (cudaStream_t)stream);
    if (rc) return rc;
    return v->known_size;
}

int64_t o3db_vbg_capacity(const o3db_vbg* v) { return v ? v->capacity : 0; }

int o3db_vbg_reserve(o3db_vbg* v, int64_t capacity, void* stream) {
    O3DB_REQUIRE(v != nullptr, "o3db_vbg_reserve: null handle");
    cudaStream_t st = (cudaStream_t)stream;
    int rc = O3DB_OK;
    if (capacity > v->capacity) rc = grow(v, capacity, st);
    if (rc) return rc;
    // a reserve acknowledges dropped frames (absorb_status): re-arm the device flag and forget the stale
    // read-backs, so that the caller can resubmit from the first dropped frame
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(v->counters + 2, 0, sizeof(int), st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(v->size_dev + 10, 0, 2 * sizeof(int), st));
    for (int i = 0; i < kPinnedInts; ++i)
        if (i % 16 == 6 || i % 16 == 10 || i % 16 == 11) v->h_pinned[i] = 0;
    v->sync_next_frame = true;
    return O3DB_OK;
}

int32_t* o3db_vbg_key_buffer(o3db_vbg* v) { return v ? v->keys : nullptr; }
float* o3db_vbg_tsdf_buffer(o3db_vbg* v) { return v ? v->tsdf : nullptr; }
uint16_t* o3db_vbg_weight_buffer(o3db_vbg* v) { return v ? v->weight : nullptr; }
uint16_t* o3db_vbg_color_buffer(o3db_vbg* v) { return v ? v->color : nullptr; }

int o3db_hash_keys(const int32_t* keys_dev, int64_t n, uint64_t* hashes_dev, void* stream) {
    O3DB_REQUIRE(n >= 0 && (n == 0 || (keys_dev && hashes_dev)), "o3db_hash_keys: bad arguments");
    if (n == 0) return O3DB_OK;
    hash_keys_kernel<<<(unsigned)ceil_div(n, kT), kT, 0, (cudaStream_t)stream>>>(keys_dev, n, hashes_dev);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

int o3db_vbg_activate(o3db_vbg* v, const int32_t* keys_dev, int64_t n, int32_t* buf_indices_dev, uint8_t* masks_dev,
                      void* stream) {
    O3DB_REQUIRE(v != nullptr && n >= 0 && n < INT_MAX && (n == 0 || keys_dev), "o3db_vbg_activate: bad arguments");
    if (n == 0) return O3DB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    // HashMap.cpp:166-181: grow when Size() + len(keys) > capacity, to max(new_size, 2*capacity)
    int rc = read_status(v, st);
    if (rc) return rc;
    const int64_t new_size = v->known_size + n;
    if (new_size > v->capacity) {
        rc = grow(v, std::max(new_size, 2 * v->capacity), st);
        if (rc) return rc;
    }
    int* scratch = nullptr;
    O3DB_CUDA_CHECK(cudaMallocAsync(&scratch, (size_t)n * sizeof(int), st));
    MapArgs a{};
    a.tab = Table{v->table, v->nbuckets - 1, v->keys};
    a.keys_rw = v->keys;
    a.in_keys = keys_dev;
    a.n = (int)n;
    a.buf_indices = buf_indices_dev;
    a.masks = masks_dev;
    a.bucket_of_input = scratch;
    a.size = v->size_dev;
    a.capacity = (int)v->capacity;
    a.overflow = v->counters + 2;
    const unsigned nb = (unsigned)ceil_div(n, kT);
    activate_claim_kernel<<<nb, kT, 0, st>>>(a);
    O3DB_LAUNCH_CHECK();
    activate_commit_kernel<<<nb, kT, 0, st>>>(a);
    O3DB_LAUNCH_CHECK();
    if (buf_indices_dev) {
        find_kernel<<<nb, kT, 0, st>>>(a, false);
        O3DB_LAUNCH_CHECK();
    }
    O3DB_CUDA_CHECK(cudaFreeAsync(scratch, st));
    return O3DB_OK;
}

int o3db_vbg_find(o3db_vbg* v, const int32_t* keys_dev, int64_t n, int32_t* buf_indices_dev, uint8_t* masks_dev,
                  void* stream) {
    O3DB_REQUIRE(v != nullptr && n >= 0 && n < INT_MAX && (n == 0 || keys_dev), "o3db_vbg_find: bad arguments");
    if (n == 0) return O3DB_OK;
    MapArgs a{};
    a.tab = Table{v->table, v->nbuckets - 1, v->keys};
    a.in_keys = keys_dev;
    a.n = (int)n;
    a.buf_indices = buf_indices_dev;
    a.masks = masks_dev;
    find_kernel<<<(unsigned)ceil_div(n, kT), kT, 0, (cudaStream_t)stream>>>(a, true);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

int64_t o3db_vbg_active_indices(o3db_vbg* v, int32_t* buf_indices_dev, int64_t max_count, void* stream) {
    if (!v) return O3DB_ERR_INVALID;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = read_status(v, st);
    if (rc) return rc;
    const int64_t n = std::min<int64_t>(v->known_size, max_count);
    if (n > 0 && buf_indices_dev) {
        iota_kernel<<<(unsigned)ceil_div(n, kT), kT, 0, st>>>(buf_indices_dev, (int)n);
        O3DB_LAUNCH_CHECK();
    }
    return v->known_size;
}

int o3db_vbg_unique_block_coordinates(o3db_vbg* v, const void* depth_dev, int depth_dtype, int rows, int cols,
                                      const double K[9], const double E[16], float depth_scale, float depth_max,
                                      float trunc_mult, int32_t* block_coords_dev, int64_t max_blocks,
                                      int64_t* num_blocks_host, void* stream) {
    O3DB_REQUIRE(v != nullptr && K && E, "o3db_vbg_unique_block_coordinates: null argument");
    int rc = check_images(depth_dev, depth_dtype, nullptr, 0, rows, cols);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    rc = ensure_frame_scratch(v, rows, cols, st);
    if (rc) return rc;
    // frustum_hashmap_->Clear() (VoxelBlockGrid.cpp:234)
    O3DB_CUDA_CHECK(cudaMemsetAsync(v->ftable, 0xff, (size_t)v->fbuckets * sizeof(int), st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(v->counters, 0, 2 * sizeof(int), st));
    TouchArgs t = make_touch_args(v, depth_dev, rows, cols, K, E, depth_scale, depth_max, trunc_mult);
    t.tab = Table{v->ftable, v->fbuckets - 1, v->keys};
    t.stamp = nullptr;
    const int nthreads = (rows / kStride) * (cols / kStride) * kSamples;
    const unsigned nb = (unsigned)std::max<int64_t>(1, ceil_div(nthreads, kT));
    if (depth_dtype == O3DB_DEPTH_U16) touch_kernel<uint16_t><<<nb, kT, 0, st>>>(t);
    else touch_kernel<float><<<nb, kT, 0, st>>>(t);
    O3DB_LAUNCH_CHECK();
    int h[2] = {0, 0};
    O3DB_CUDA_CHECK(cudaMemcpyAsync(h, v->counters, sizeof(h), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    const int64_t n = h[1];
    if (num_blocks_host) *num_blocks_host = n;
    if (n == 0) {  // VoxelBlockGridCUDA.cu:193-198
        set_last_error("No block is touched in TSDF volume, abort integration. Please check specified parameters, "
                       "especially depth_scale and voxel_size");
        return O3DB_ERR_NO_BLOCKS;
    }
    if (block_coords_dev) {
        O3DB_REQUIRE(max_blocks >= n, "block_coords buffer too small: %lld < %lld", (long long)max_blocks, (long long)n);
        emit_unique_keys_kernel<<<(unsigned)ceil_div(n, kT), kT, 0, st>>>(v->new_list, v->counters, v->cand_keys,
                                                                          block_coords_dev, (int)max_blocks);
        O3DB_LAUNCH_CHECK();
    }
    O3DB_CUDA_CHECK(cudaMemsetAsync(v->counters, 0, 2 * sizeof(int), st));
    return O3DB_OK;
}

int o3db_vbg_integrate(o3db_vbg* v, const int32_t* block_coords_dev, int64_t num_blocks, const void* depth_dev,
                       int depth_dtype, const void* color_dev, int color_dtype, int rows, int cols,
                       const double dK[9], const double cK[9], const double E[16], float depth_scale,
                       float depth_max, float trunc_mult, void* stream) {
    O3DB_REQUIRE(v != nullptr && dK && E && block_coords_dev && num_blocks > 0 && num_blocks < INT_MAX,
                 "o3db_vbg_integrate: bad arguments");
    int rc = check_images(depth_dev, depth_dtype, color_dev, color_dtype, rows, cols);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const bool has_color = color_dev != nullptr && v->with_color;   // VoxelBlockGridImpl.h:206-207
    int* buf = nullptr;
    O3DB_CUDA_CHECK(cudaMallocAsync(&buf, (size_t)num_blocks * sizeof(int), st));
    // VoxelBlockGrid.cpp:313-315: Activate, then Find
    rc = o3db_vbg_activate(v, block_coords_dev, num_blocks, buf, nullptr, st);
    if (rc) {
        cudaFreeAsync(buf, st);
        return rc;
    }
    IntegrateArgs a = base_integrate_args(v, depth_dev, has_color ? color_dev : nullptr, color_dtype, rows, cols, dK, cK,
                                          E, depth_scale, depth_max, trunc_mult);
    a.buf_indices = buf;
    a.n_blocks = (int)num_blocks;
    const unsigned grid = (unsigned)std::min<int64_t>(num_blocks * 4, (int64_t)integrate_grid());
    rc = launch_integrate(v, a, depth_dtype, color_dtype, has_color, grid, st);
    cudaFreeAsync(buf, st);
    return rc;
}

/* Stateless twins of DepthTouchCUDA / IntegrateCUDA for the case where the hash map and its buffers stay the
 * reference's own (integration/o3d_forwarders.cpp). */
int o3db_depth_touch(const void* depth_dev, int depth_dtype, int rows, int cols, const double K[9], const double E[16],
                     int block_resolution, float voxel_size, float sdf_trunc, float depth_scale, float depth_max,
                     int stride, int32_t* block_coords_dev, int64_t max_blocks, int64_t* num_blocks_host, void* stream) {
    O3DB_REQUIRE(K && E && voxel_size > 0 && block_resolution >= 1, "o3db_depth_touch: bad arguments");
    O3DB_REQUIRE(stride == kStride, "o3db_depth_touch: stride must be 4 (VoxelBlockGrid.cpp:221 down_factor)");
    int rc = check_images(depth_dev, depth_dtype, nullptr, 0, rows, cols);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    // scratch of one call: candidate keys, winners, a frustum-sized table (VoxelBlockGrid.cpp:225-234)
    const int64_t need = (int64_t)(rows / kStride) * (cols / kStride) * kSamples;
    const unsigned fbuckets = pow2_at_least(2 * need);
    int *cand = nullptr, *ftable = nullptr, *counters = nullptr;
    int2* winners = nullptr;
    cudaError_t e = cudaMallocAsync(&cand, (size_t)need * 3 * sizeof(int), st);
    if (e == cudaSuccess) e = cudaMallocAsync(&winners, (size_t)need * sizeof(int2), st);
    if (e == cudaSuccess) e = cudaMallocAsync(&ftable, (size_t)fbuckets * sizeof(int), st);
    if (e == cudaSuccess) e = cudaMallocAsync(&counters, 4 * sizeof(int), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(ftable, 0xff, (size_t)fbuckets * sizeof(int), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(counters, 0, 4 * sizeof(int), st);
    int h[2] = {0, 0};
    if (e == cudaSuccess) {
        TouchArgs t{};
        double pose[16];
        inverse_transformation(E, pose);
        t.depth = depth_dev;
        t.rows = rows;
        t.cols = cols;
        t.cam = make_cam(K, pose, 1.0f);
        t.block_size = voxel_size * block_resolution;
        t.sdf_trunc = sdf_trunc;
        t.depth_scale = depth_scale;
        t.depth_max = depth_max;
        t.cand_keys = cand;
        t.new_list = winners;
        t.counters = counters;
        t.max_list = (int)need;
        t.tab = Table{ftable, fbuckets - 1, nullptr};
        const unsigned nb = (unsigned)std::max<int64_t>(1, ceil_div(need, kT));
        if (depth_dtype == O3DB_DEPTH_U16) touch_kernel<uint16_t><<<nb, kT, 0, st>>>(t);
        else touch_kernel<float><<<nb, kT, 0, st>>>(t);
        count_launch();
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(h, counters, sizeof(h), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    }
    rc = O3DB_OK;
    const int64_t n = h[1];
    if (e == cudaSuccess) {
        if (num_blocks_host) *num_blocks_host = n;
        if (n == 0) {
            set_last_error("No block is touched in TSDF volume, abort integration. Please check specified parameters, "
                           "especially depth_scale and voxel_size");
            rc = O3DB_ERR_NO_BLOCKS;
        } else if (block_coords_dev) {
            if (max_blocks < n) {
                set_last_error("block_coords buffer too small: %lld < %lld", (long long)max_blocks, (long long)n);
                rc = O3DB_ERR_INVALID;
            } else {
                emit_unique_keys_kernel<<<(unsigned)ceil_div(n, kT), kT, 0, st>>>(winners, counters, cand, block_coords_dev,
                                                                                  (int)max_blocks);
                count_launch();
                e = cudaGetLastError();
            }
        }
    }
    for (void* p : {(void*)cand, (void*)winners, (void*)ftable, (void*)counters})
        if (p) cudaFreeAsync(p, st);
    if (e != cudaSuccess) {
        set_last_error("o3db_depth_touch: %s", cudaGetErrorString(e));
        return O3DB_ERR_CUDA;
    }
    return rc;
}

int o3db_integrate_blocks(const void* depth_dev, int depth_dtype, const void* color_dev, int color_dtype, int rows,
                          int cols, const int32_t* block_indices_dev, int64_t num_blocks,
                          const int32_t* block_keys_dev, float* tsdf_dev, void* weight_dev, void* color_buf_dev,
                          int value_layout, const double dK[9], const double cK[9], const double E[16],
                          int block_resolution, float voxel_size, float sdf_trunc, float depth_scale, float depth_max,
                          void* stream) {
    O3DB_REQUIRE(dK && E && block_indices_dev && block_keys_dev && tsdf_dev && weight_dev && num_blocks > 0 &&
                         num_blocks < INT_MAX && voxel_size > 0 && block_resolution >= 1,
                 "o3db_integrate_blocks: bad arguments");
    O3DB_REQUIRE(value_layout == O3DB_VALUES_U16 || value_layout == O3DB_VALUES_F32,
                 "Unsupported value data type combination. Expected (float, float) or (uint16, uint16)");
    int rc = check_images(depth_dev, depth_dtype, color_dev, color_dtype, rows, cols);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const bool has_color = color_dev != nullptr && color_buf_dev != nullptr;     // VoxelBlockGridImpl.h:202-203
    o3db_vbg tmp;                 // only a carrier for base_integrate_args: nothing is owned
    tmp.voxel_size = voxel_size;
    tmp.resolution = block_resolution;
    tmp.keys = const_cast<int*>(block_keys_dev);
    tmp.tsdf = tsdf_dev;
    tmp.weight = (uint16_t*)weight_dev;
    tmp.color = (uint16_t*)color_buf_dev;
    tmp.inv_w = inv_weight_table();
    O3DB_REQUIRE(tmp.inv_w != nullptr, "o3db_integrate_blocks: could not build the weight table");
    static float s_scale = 0.f;   // (benign race: both values are recomputed from depth_scale alone)
    static bool s_ok = false;
    tmp.checked_scale = s_scale;
    tmp.checked_scale_ok = s_ok;
    IntegrateArgs a = base_integrate_args(&tmp, depth_dev, has_color ? color_dev : nullptr, color_dtype, rows, cols, dK, cK, E,
                                          depth_scale, depth_max, 1.0f);
    s_scale = tmp.checked_scale;
    s_ok = tmp.checked_scale_ok;
    a.sdf_trunc = sdf_trunc;      // the reference passes the truncation itself (VoxelBlockGrid.h:369-381)
    a.capacity = INT_MAX;
    a.buf_indices = block_indices_dev;
    a.n_blocks = (int)num_blocks;
    if (value_layout == O3DB_VALUES_U16) {
        const unsigned grid = (unsigned)std::min<int64_t>(num_blocks * 4, (int64_t)integrate_grid());
        return launch_integrate(&tmp, a, depth_dtype, color_dtype, has_color, grid, st);
    }
    // Float32 weight / Float32 colour (VoxelBlockGridCUDA.cu:238-244, second and fourth instantiation)
    const unsigned grid = (unsigned)std::min<int64_t>(num_blocks, (int64_t)num_sms() * 8);
    cudaError_t e = cudaErrorInvalidValue;
    if (depth_dtype == O3DB_DEPTH_U16 && (!has_color || color_dtype == O3DB_COLOR_U8)) {
        e = has_color ? launch_pdl_ex(integrate_kernel<uint16_t, uint8_t, true, float, float>, {grid, kT}, st, a)
                      : launch_pdl_ex(integrate_kernel<uint16_t, uint8_t, false, float, float>, {grid, kT}, st, a);
    } else if (depth_dtype == O3DB_DEPTH_F32 && (!has_color || color_dtype == O3DB_COLOR_F32)) {
        e = has_color ? launch_pdl_ex(integrate_kernel<float, float, true, float, float>, {grid, kT}, st, a)
                      : launch_pdl_ex(integrate_kernel<float, float, false, float, float>, {grid, kT}, st, a);
    } else {
        set_last_error("Unsupported input data type combination. Expected (float, float) or (uint16, uint8)");
        return O3DB_ERR_INVALID;
    }
    count_launch();
    if (e != cudaSuccess) {
        set_last_error("integrate kernel launch failed: %s", cudaGetErrorString(e));
        return O3DB_ERR_CUDA;
    }
    return O3DB_OK;
}

int o3db_vbg_integrate_frame(o3db_vbg* v, const void* depth_dev, int depth_dtype, const void* color_dev,
                             int color_dtype, int rows, int cols, const double K[9], const double E[16],
                             float depth_scale, float depth_max, float trunc_mult, void* stream) {
    O3DB_REQUIRE(v != nullptr && K && E, "o3db_vbg_integrate_frame: null argument");
    int rc = check_images(depth_dev, depth_dtype, color_dev, color_dtype, rows, cols);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    rc = ensure_frame_scratch(v, rows, cols, st);
    if (rc) return rc;
    // Capacity management without a per-frame host sync: wait for the frame launched two
    // calls ago (normally long finished), read the size it published, and grow ahead of
    // need (HashMap.cpp:166-181 grows when size + n > capacity).  Three frames (two in
    // flight + this one) may add blocks the host has not seen yet.
    if (v->frames >= 2) {
        // the status frame (frames - 2) published into pinned memory; normally long there — the wait only bounds how
        // far the host may run ahead of the device (two frames)
        const int64_t f = v->frames - 2;
        volatile int* hs = v->h_pinned + 16 + 16 * (int)(f & 7);
        if (hs[15] != (int)(f + 1)) {
            const auto t0 = std::chrono::steady_clock::now();
            while (hs[15] != (int)(f + 1)) {
                if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(20)) {
                    const cudaError_t e = cudaStreamQuery(st);
                    set_last_error("fused frame #%lld never reported its status (%s)", (long long)f,
                                   e == cudaSuccess || e == cudaErrorNotReady ? "timeout" : cudaGetErrorString(e));
                    return O3DB_ERR_CUDA;
                }
            }
        }
        int h[16];
        for (int i = 0; i < 16; ++i) h[i] = hs[i];
        rc = absorb_status(v, h);
        if (rc) return rc;
    }
    const int64_t per_frame = std::max<int64_t>(2 * v->max_new_seen, 2048);
    if (v->known_size + 3 * per_frame > v->capacity) {
        rc = read_status(v, st);
        if (rc) return rc;
        if (v->known_size + 3 * per_frame > v->capacity) {
            rc = grow(v, std::max<int64_t>(2 * v->capacity, v->known_size + 6 * per_frame), st);
            if (rc) return rc;
        }
    }
    const bool has_color = color_dev != nullptr && v->with_color;
    const int nthreads = (rows / kStride) * (cols / kStride) * kSamples;
    const unsigned nb = (unsigned)std::max<int64_t>(1, ceil_div(nthreads, kT));
    const bool prof = v->prof_on && (size_t)(3 * v->prof_frames + 2) < v->prof_ev.size();
    if (prof) cudaEventRecord(v->prof_ev[3 * v->prof_frames], st);
    auto touch = [&]() -> int {
        v->frame_id += 1;
        TouchArgs t = make_touch_args(v, depth_dev, rows, cols, K, E, depth_scale, depth_max, trunc_mult);
        t.tab = Table{v->table, v->nbuckets - 1, v->keys};
        t.stamp = v->stamp;
        t.frame_id = v->frame_id;
        const cudaError_t e = depth_dtype == O3DB_DEPTH_U16 ? launch_pdl_ex(touch_kernel<uint16_t>, {nb, kT}, st, t)
                                                            : launch_pdl_ex(touch_kernel<float>, {nb, kT}, st, t);
        count_launch();
        if (e != cudaSuccess) {
            set_last_error("touch kernel launch failed: %s", cudaGetErrorString(e));
            return O3DB_ERR_CUDA;
        }
        return O3DB_OK;
    };
    rc = touch();
    if (rc) return rc;
    if (v->frames == 0 || v->sync_next_frame) {
        // Nothing is known yet about how many blocks a frame of this sequence adds (first frame, or the first one
        // after a reserve that followed a dropped frame): size the map from the touch kernel's own count before
        // integrating, as HashMap::Activate does (HashMap.cpp:166-181).  One host synchronisation, once.
        v->sync_next_frame = false;
        O3DB_CUDA_CHECK(cudaMemcpyAsync(v->h_pinned, v->size_dev, 16 * sizeof(int), cudaMemcpyDeviceToHost, st));
        O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
        const int64_t need = (int64_t)v->h_pinned[0] + v->h_pinned[5];
        if (need > v->capacity && !v->h_pinned[6]) {
            rc = grow(v, std::max<int64_t>(2 * v->capacity, need + std::max<int64_t>(need / 2, 2048)), st);
            if (rc) return rc;
            // the provisional entries lived in the old table: discover the frame again in the new one
            O3DB_CUDA_CHECK(cudaMemsetAsync(v->counters, 0, 2 * sizeof(int), st));
            rc = touch();
            if (rc) return rc;
        }
    }
    if (prof) cudaEventRecord(v->prof_ev[3 * v->prof_frames + 1], st);
    IntegrateArgs a = base_integrate_args(v, depth_dev, has_color ? color_dev : nullptr, color_dtype, rows, cols, K, K, E,
                                          depth_scale, depth_max, trunc_mult);
    a.exist_list = v->exist_list;
    a.new_list = v->new_list;
    a.cand_keys = v->cand_keys;
    a.counters = v->counters;
    a.size = v->size_dev;
    a.table = v->table;
    a.keys_rw = v->keys;
    a.stamp = v->stamp;
    a.frame_slots = v->frame_slots;
    a.frame_count = v->frame_count;
    a.max_new = v->size_dev + 9;
    a.frame_id = v->frame_id;
    a.frame_index = (int)v->frames;
    a.host_status = v->h_pinned + 16;
    a.work = v->size_dev + 12;
    a.exec_ns = v->exec_ns;
    rc = launch_integrate(v, a, depth_dtype, color_dtype, has_color, integrate_grid(), st);
    if (rc) return rc;
    if (prof) {
        cudaEventRecord(v->prof_ev[3 * v->prof_frames + 2], st);
        v->prof_frames += 1;
    }
    v->frames += 1;
    return O3DB_OK;
}

int o3db_vbg_integrate_frame_host(o3db_vbg* v, const void* depth_host, int depth_dtype, const void* color_host,
                                  int color_dtype, int rows, int cols, const double K[9], const double E[16],
                                  float depth_scale, float depth_max, float trunc_mult, void* stream) {
    O3DB_REQUIRE(v != nullptr, "o3db_vbg_integrate_frame_host: null handle");
    int rc = check_images(depth_host, depth_dtype, color_host, color_dtype, rows, cols);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t dbytes = (size_t)rows * cols * (depth_dtype == O3DB_DEPTH_U16 ? 2 : 4);
    const size_t cbytes = color_host ? (size_t)rows * cols * 3 * (color_dtype == O3DB_COLOR_U8 ? 1 : 4) : 0;
    if (!v->copy_stream) {
        O3DB_CUDA_CHECK(cudaStreamCreateWithFlags(&v->copy_stream, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            O3DB_CUDA_CHECK(cudaEventCreateWithFlags(&v->copied[i], cudaEventDisableTiming));
            O3DB_CUDA_CHECK(cudaEventCreateWithFlags(&v->consumed[i], cudaEventDisableTiming));
        }
    }
    const int slot = (int)(v->host_frames & 1);
    // the slot is free once the kernels of the frame that used it two calls ago are done
    O3DB_CUDA_CHECK(cudaStreamWaitEvent(v->copy_stream, v->consumed[slot], 0));
    if (dbytes > v->d_depth_bytes[slot]) {
        O3DB_CUDA_CHECK(cudaStreamSynchronize(v->copy_stream));
        if (v->d_depth[slot]) O3DB_CUDA_CHECK(cudaFree(v->d_depth[slot]));
        O3DB_CUDA_CHECK(cudaMalloc(&v->d_depth[slot], dbytes));
        v->d_depth_bytes[slot] = dbytes;
    }
    if (cbytes > v->d_color_bytes[slot]) {
        O3DB_CUDA_CHECK(cudaStreamSynchronize(v->copy_stream));
        if (v->d_color[slot]) O3DB_CUDA_CHECK(cudaFree(v->d_color[slot]));
        O3DB_CUDA_CHECK(cudaMalloc(&v->d_color[slot], cbytes));
        v->d_color_bytes[slot] = cbytes;
    }
    O3DB_CUDA_CHECK(cudaMemcpyAsync(v->d_depth[slot], depth_host, dbytes, cudaMemcpyHostToDevice, v->copy_stream));
    if (cbytes) O3DB_CUDA_CHECK(cudaMemcpyAsync(v->d_color[slot], color_host, cbytes, cudaMemcpyHostToDevice, v->copy_stream));
    O3DB_CUDA_CHECK(cudaEventRecord(v->copied[slot], v->copy_stream));
    O3DB_CUDA_CHECK(cudaStreamWaitEvent(st, v->copied[slot], 0));
    const int rc2 = o3db_vbg_integrate_frame(v, v->d_depth[slot], depth_dtype, cbytes ? v->d_color[slot] : nullptr, color_dtype,
                                             rows, cols, K, E, depth_scale, depth_max, trunc_mult, st);
    O3DB_CUDA_CHECK(cudaEventRecord(v->consumed[slot], st));
    v->host_frames += 1;
    return rc2;
}

int o3db_vbg_integrate_sequence(o3db_vbg* v, int64_t n_frames, const void* const* depth_ptrs, int depth_dtype,
                                const void* const* color_ptrs, int color_dtype, int rows, int cols,
                                const double K[9], const double* extrinsics, float depth_scale, float depth_max,
                                float trunc_mult, int host_images, void* stream) {
    O3DB_REQUIRE(v != nullptr && n_frames >= 0 && (n_frames == 0 || (depth_ptrs && extrinsics && K)),
                 "o3db_vbg_integrate_sequence: bad arguments");
    for (int64_t f = 0; f < n_frames; ++f) {
        const void* c = color_ptrs ? color_ptrs[f] : nullptr;
        const int rc = host_images ? o3db_vbg_integrate_frame_host(v, depth_ptrs[f], depth_dtype, c, color_dtype, rows,
                                                                   cols, K, extrinsics + 16 * f, depth_scale,
                                                                   depth_max, trunc_mult, stream)
                                   : o3db_vbg_integrate_frame(v, depth_ptrs[f], depth_dtype, c, color_dtype, rows, cols, K,
                                                              extrinsics + 16 * f, depth_scale, depth_max, trunc_mult,
                                                              stream);
        if (rc != O3DB_OK) return rc;
    }
    return O3DB_OK;
}

int o3db_vbg_exec_stats(o3db_vbg* v, double* integrate_exec_ms, int64_t* launches, int reset, void* stream) {
    O3DB_REQUIRE(v != nullptr, "o3db_vbg_exec_stats: null handle");
    unsigned long long h[3] = {0, 0, 0};
    if (v->exec_ns) {
        O3DB_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
        O3DB_CUDA_CHECK(cudaMemcpy(h, v->exec_ns, sizeof(h), cudaMemcpyDeviceToHost));
        if (reset) {
            const unsigned long long init[3] = {~0ull, 0ull, 0ull};
            O3DB_CUDA_CHECK(cudaMemcpy(v->exec_ns, init, sizeof(init), cudaMemcpyHostToDevice));
        }
    }
    if (integrate_exec_ms) *integrate_exec_ms = 1e-6 * (double)h[1];
    if (launches) *launches = (int64_t)h[2];
    return O3DB_OK;
}

int o3db_vbg_profile(o3db_vbg* v, int enable) {
    O3DB_REQUIRE(v != nullptr, "o3db_vbg_profile: null handle");
    if (enable && v->prof_ev.empty()) {
        v->prof_ev.resize(3 * 4096);
        for (auto& e : v->prof_ev) O3DB_CUDA_CHECK(cudaEventCreate(&e));
    }
    v->prof_on = enable != 0;
    v->prof_frames = 0;
    return O3DB_OK;
}

int o3db_vbg_profile_read(o3db_vbg* v, double* touch_ms, double* integrate_ms, int64_t* frames) {
    O3DB_REQUIRE(v != nullptr, "o3db_vbg_profile_read: null handle");
    double t = 0, g = 0;
    for (int64_t f = 0; f < v->prof_frames; ++f) {
        float a = 0, b = 0;
        O3DB_CUDA_CHECK(cudaEventSynchronize(v->prof_ev[3 * f + 2]));
        O3DB_CUDA_CHECK(cudaEventElapsedTime(&a, v->prof_ev[3 * f], v->prof_ev[3 * f + 1]));
        O3DB_CUDA_CHECK(cudaEventElapsedTime(&b, v->prof_ev[3 * f + 1], v->prof_ev[3 * f + 2]));
        t += a;
        g += b;
    }
    if (touch_ms) *touch_ms = t;
    if (integrate_ms) *integrate_ms = g;
    if (frames) *frames = v->prof_frames;
    v->prof_frames = 0;
    return O3DB_OK;
}

int64_t o3db_vbg_last_frustum_blocks(o3db_vbg* v, int32_t* block_coords_dev, int64_t max_blocks, void* stream) {
    if (!v) return O3DB_ERR_INVALID;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = read_status(v, st);
    if (rc) return rc;
    const int64_t n = v->h_pinned[8];
    const int64_t m = std::min(n, max_blocks);
    if (m > 0 && block_coords_dev) {
        gather_keys_kernel<<<(unsigned)ceil_div(m, kT), kT, 0, st>>>(v->keys, v->frame_slots, (int)m, block_coords_dev);
        O3DB_LAUNCH_CHECK();
    }
    return n;
}

}  // extern "C"
