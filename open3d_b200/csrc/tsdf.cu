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
    VbgStatus* status;       // n_exist, n_new, overflow
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
    if (r == kResFull) a.status->overflow = 1;
    // warp-aggregated list appends: one atomic per warp and list instead of one per block key
    const unsigned active = __activemask();
    const unsigned me = __ballot_sync(active, first_exist), mn = __ballot_sync(active, first_new);
    const unsigned lt = (1u << lane) - 1u;
    if (me) {
        const int lead = __ffs(me) - 1;
        int base = 0;
        if (lane == lead) base = atomicAdd(&a.status->n_exist, __popc(me));
        base = __shfl_sync(active, base, lead);
        if (first_exist) {
            const int p = base + __popc(me & lt);
            if (p < a.max_list) a.exist_list[p] = r;
            else a.status->overflow = 1;
        }
    }
    if (mn) {
        const int lead = __ffs(mn) - 1;
        int base = 0;
        if (lane == lead) base = atomicAdd(&a.status->n_new, __popc(mn));
        base = __shfl_sync(active, base, lead);
        if (first_new) {
            const int p = base + __popc(mn & lt);
            if (p < a.max_list) a.new_list[p] = make_int2((int)bucket, cand);
            else a.status->overflow = 1;
        }
    }
}

// Stand-alone GetUniqueBlockCoordinates: the winners' keys are the unique set.
__global__ void emit_unique_keys_kernel(const int2* __restrict__ new_list, const VbgStatus* __restrict__ status,
                                        const int* __restrict__ cand_keys, int* __restrict__ out, int max_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = min(status->n_new, max_out);
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
    VbgStatus* status;     // size, overflow
    int capacity;
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
    if (r == kResFull) a.status->overflow = 1;
}
// pass 2: winners pop a slot (CUDAHashBackendBufferAccessor.h:80-83 heap_top), publish key + slot.
__global__ void activate_commit_kernel(MapArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    const int b = a.bucket_of_input[i];
    if (b < 0) return;
    const int slot = atomicAdd(&a.status->size, 1);
    if (slot >= a.capacity) {
        atomicSub(&a.status->size, 1);
        a.tab.table[b] = kTomb;
        if (a.masks) a.masks[i] = 0;
        a.status->overflow = 1;
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
    // fused mode (status != nullptr): exist_list ++ new_list, commit on the fly
    const int* exist_list;
    const int2* new_list;
    const int* cand_keys;
    VbgStatus* status;       // the volume's record: read at the start, updated and re-armed by the last CTA
    VbgStatus* ring;         // pinned host memory, kStatusRing records: the frame's status, written by the last CTA
    int* table;
    int* keys_rw;
    int* stamp;
    int* frame_slots;        // [max] slots of this frame's frustum blocks (Model::frustum_block_coords_)
    unsigned long long* exec_ns;   // fused integrate16_kernel only: [0] earliest CTA start of this launch (re-armed by the last
                                   // CTA), [1] sum over launches of (last CTA end - earliest start), [2] launches — %globaltimer,
                                   // unperturbed by events
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


// What every CTA of an integrate launch knows about its frame.  List mode: n_total = n_blocks, nothing else.
struct Frame {
    int n_exist, n_new;   // touched committed blocks, keys first seen (fused mode)
    int size0;            // size before the frame: new block i takes slot size0 + i
    int n_total;          // blocks to integrate
    bool drop;
};

// Start of an integrate launch, after pdl_wait.  Fused mode: ONE decision for every CTA (all the values it reads are
// final once the touch kernel has finished): a frame whose new blocks do not fit, whose lists overflowed, or that
// follows a dropped frame, is dropped as a whole — nothing integrated, its provisional table entries released — and
// reported by the host.
__device__ __forceinline__ Frame frame_begin(const IntegrateArgs& a) {
    Frame f{0, 0, 0, a.n_blocks, false};
    if (!a.status) return f;
    f.n_exist = a.status->n_exist;
    f.n_new = a.status->n_new;
    f.size0 = a.status->size;
    f.drop = a.status->overflow != 0 || f.size0 + f.n_new > a.capacity;
    f.n_total = f.drop ? 0 : f.n_exist + f.n_new;
    if (f.drop) {
        // no committed key's probe chain passes over a bucket that was empty when the frame began, so emptying every
        // bucket this frame claimed restores the table exactly
        const int n_roll = min(f.n_new, a.max_list);
        for (int i = blockIdx.x * kT + threadIdx.x; i < n_roll; i += gridDim.x * kT) a.table[a.new_list[i].x] = kEmpty;
    }
    return f;
}

// Slot of block b of the launch, and in *key its block coordinate, for work unit `unit` of the block.  Fused mode:
// the frame's touched committed blocks, then the keys it saw first, which take slots size0, size0 + 1, ...; unit 0 of
// a new block commits it (key, stamp, table entry), and unit 0 of every block records its slot in frame_slots.
__device__ __forceinline__ int unit_block(const IntegrateArgs& a, const Frame& f, int b, int unit, const int*& key) {
    int slot;
    if (!a.status) {
        slot = a.buf_indices[b];
        key = a.block_keys + 3 * (size_t)slot;
    } else if (b < f.n_exist) {
        slot = a.exist_list[b];
        key = a.block_keys + 3 * (size_t)slot;
    } else {
        const int2 nl = a.new_list[b - f.n_exist];
        slot = f.size0 + (b - f.n_exist);
        key = a.cand_keys + 3 * (size_t)nl.y;
        if (unit == 0) {
            a.keys_rw[3 * (size_t)slot] = key[0];
            a.keys_rw[3 * (size_t)slot + 1] = key[1];
            a.keys_rw[3 * (size_t)slot + 2] = key[2];
            a.stamp[slot] = a.frame_id;
            a.table[nl.x] = slot;
        }
    }
    if (a.status && unit == 0) a.frame_slots[b] = slot;
    return slot;
}

// The last CTA of a fused frame publishes the frame's status straight into pinned HOST memory (a posted write over
// PCIe): entry frame_index % kStatusRing of the ring, seq last.  The host therefore learns sizes without a
// device-to-host copy or an event in the stream — the frame's two kernels stay adjacent, which programmatic
// dependent launch needs.
__device__ __forceinline__ void publish_status(const IntegrateArgs& a, const Frame& f) {
    volatile VbgStatus* r = a.ring + (a.frame_index & (kStatusRing - 1));
    r->size = f.drop ? f.size0 : f.size0 + f.n_new;
    r->n_new = f.n_new;
    r->overflow = f.drop ? 1 : 0;
    r->frame_count = f.n_total;
    r->max_new = a.status->max_new;
    r->dropped_need = a.status->dropped_need;
    r->dropped_frame = a.status->dropped_frame;
    __threadfence_system();
    r->seq = a.frame_index + 1;
}

// End of a fused integrate launch: the last CTA to finish updates the status, re-arms the per-frame counters and
// publishes the frame.
__device__ __forceinline__ void frame_end(const IntegrateArgs& a, const Frame& f) {
    __shared__ int s_last;
    if (!a.status) return;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(&a.status->ticket, 1) == (int)gridDim.x - 1;
    __syncthreads();
    if (!s_last || threadIdx.x != 0) return;
    VbgStatus* s = a.status;
    if (f.drop) {
        if (s->dropped_frame == 0) {          // first dropped frame: what it needed, and which one it was
            s->dropped_need = f.size0 + f.n_new;
            s->dropped_frame = a.frame_index + 1;
        }
        s->overflow = 1;                      // sticky: later frames are dropped too until the host reserves
    } else {
        s->size = f.size0 + f.n_new;
    }
    s->frame_count = f.n_total;
    if (f.n_new > s->max_new) s->max_new = f.n_new;
    s->n_exist = 0;
    s->n_new = 0;
    s->ticket = 0;
    s->work = 0;
    if (a.exec_ns) {
        const unsigned long long now = global_ns();
        a.exec_ns[1] += now - a.exec_ns[0];
        a.exec_ns[2] += 1;
        a.exec_ns[0] = ~0ull;
    }
    publish_status(a, f);
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
    pdl_wait();
    pdl_launch_dependents();
    const Frame f = frame_begin(a);
    // work unit = one quarter of a 16^3 block (whole block for other resolutions)
    constexpr bool kVec = sizeof(weight_t) == 2;     // the vectorised quarter-block path is the u16 / u16 layout's
    const int upb = (kVec && a.resolution == 16) ? 4 : 1;
    for (int wu = blockIdx.x; wu < f.n_total * upb; wu += gridDim.x) {
        const int b = wu / upb, unit = wu % upb;
        if (threadIdx.x == 0) {
            const int* k;
            const int slot = unit_block(a, f, b, unit, k);
            s_slot = slot;
            if (slot >= 0) {
                s_key[0] = k[0];
                s_key[1] = k[1];
                s_key[2] = k[2];
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
    frame_end(a, f);
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
    constexpr int kTileCols = kTileRowBytes / (int)sizeof(depth_t);
    const int tid = threadIdx.x;
    if (tid == 0) {
        mbar_init(&s_mbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    pdl_wait();                 // the touch kernel's lists / counters, the previous frame's size
    pdl_launch_dependents();
    if (a.exec_ns && tid == 0) atomicMin(&a.exec_ns[0], (unsigned long long)global_ns());
    const Frame f = frame_begin(a);
    const int n_units = f.n_total * 4;

    auto fetch = [&](int wu, int buf) {    // one thread: metadata of work unit wu
        const int* k;
        s_meta[buf][0] = unit_block(a, f, wu >> 2, wu & 3, k);
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
            int next = a.status ? (int)gridDim.x + atomicAdd(&a.status->work, 1) : wu + (int)gridDim.x;
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
    frame_end(a, f);
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

// verify_fast_scale, run once per scale and thread: a sequence of frames keeps its scale, so the 65536-value check is
// paid once, and each thread keeps its own answer.
static bool fast_scale_ok(float s) {
    thread_local float last = 0.f;
    thread_local bool ok = false;   // == verify_fast_scale(0.f)
    if (s != last) {
        last = s;
        ok = verify_fast_scale(s);
    }
    return ok;
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

// Allocates and clears the map m of v's shape for `capacity` blocks.
static int alloc_map(const o3db_vbg* v, VbgMap& m, int64_t capacity, cudaStream_t st) {
    m.capacity = capacity;
    m.nbuckets = pow2_at_least(2 * capacity);
    const size_t r3 = res3(v);
    if (int rc = dev_alloc(m.table, m.nbuckets, st)) return rc;
    if (int rc = dev_alloc(m.keys, (size_t)capacity * 3, st)) return rc;
    if (int rc = dev_alloc(m.stamp, (size_t)capacity, st)) return rc;
    if (int rc = dev_alloc(m.tsdf, (size_t)capacity * r3, st)) return rc;
    if (int rc = dev_alloc(m.weight, (size_t)capacity * r3, st)) return rc;
    if (v->with_color)
        if (int rc = dev_alloc(m.color, (size_t)capacity * r3 * 3, st)) return rc;
    O3DB_CUDA_CHECK(cudaMemsetAsync(m.table.get(), 0xff, (size_t)m.nbuckets * sizeof(int), st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(m.keys.get(), 0, (size_t)capacity * 3 * sizeof(int), st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(m.stamp.get(), 0xff, (size_t)capacity * sizeof(int), st));
    // value buffers are zero-initialised at allocation (CUDAHashBackendBufferAccessor.h:56-57)
    O3DB_CUDA_CHECK(cudaMemsetAsync(m.tsdf.get(), 0, (size_t)capacity * r3 * sizeof(float), st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(m.weight.get(), 0, (size_t)capacity * r3 * sizeof(uint16_t), st));
    if (v->with_color) O3DB_CUDA_CHECK(cudaMemsetAsync(m.color.get(), 0, (size_t)capacity * r3 * 3 * sizeof(uint16_t), st));
    return O3DB_OK;
}

static int ensure_frame_scratch(o3db_vbg* v, int rows, int cols, cudaStream_t st) {
    const int64_t need = (int64_t)(rows / kStride) * (cols / kStride) * kSamples;   // VoxelBlockGrid.cpp:225-227
    if (need <= v->frustum_cap) return O3DB_OK;
    v->frustum_cap = 0;   // until every buffer has its new size
    for (GridPtr<int>* p : {&v->cand_keys, &v->exist_list, &v->frame_slots, &v->ftable}) free_on(*p, st);
    free_on(v->new_list, st);
    const unsigned fbuckets = pow2_at_least(2 * need);
    if (int rc = dev_alloc(v->cand_keys, (size_t)need * 3, st)) return rc;
    if (int rc = dev_alloc(v->exist_list, (size_t)need, st)) return rc;
    if (int rc = dev_alloc(v->new_list, (size_t)need, st)) return rc;
    if (int rc = dev_alloc(v->frame_slots, (size_t)need, st)) return rc;
    if (int rc = dev_alloc(v->ftable, fbuckets, st)) return rc;
    v->frustum_cap = need;
    v->fbuckets = fbuckets;
    return O3DB_OK;
}

// Builds the grown map in m: the live slots keep their indices, only the table is rebuilt.
static int fill_grown_map(const o3db_vbg* v, VbgMap& m, int64_t new_capacity, int size, cudaStream_t st) {
    int rc = alloc_map(v, m, new_capacity, st);
    if (rc || size == 0) return rc;
    const VbgMap& old = v->map;
    const size_t r3 = res3(v);
    O3DB_CUDA_CHECK(cudaMemcpyAsync(m.keys.get(), old.keys.get(), (size_t)size * 3 * sizeof(int), cudaMemcpyDeviceToDevice, st));
    O3DB_CUDA_CHECK(cudaMemcpyAsync(m.stamp.get(), old.stamp.get(), (size_t)size * sizeof(int), cudaMemcpyDeviceToDevice, st));
    O3DB_CUDA_CHECK(cudaMemcpyAsync(m.tsdf.get(), old.tsdf.get(), (size_t)size * r3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    O3DB_CUDA_CHECK(cudaMemcpyAsync(m.weight.get(), old.weight.get(), (size_t)size * r3 * sizeof(uint16_t), cudaMemcpyDeviceToDevice, st));
    if (v->with_color)
        O3DB_CUDA_CHECK(cudaMemcpyAsync(m.color.get(), old.color.get(), (size_t)size * r3 * 3 * sizeof(uint16_t), cudaMemcpyDeviceToDevice, st));
    rehash_kernel<<<(unsigned)ceil_div(size, kT), kT, 0, st>>>(m.table.get(), m.nbuckets - 1, m.keys.get(), size);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

static int grow(o3db_vbg* v, int64_t new_capacity, cudaStream_t st) {
    // HashMap::Reserve (HashMap.cpp:47-77): upstream re-inserts active entries into
    // new buffers; here slots keep their indices, only the table is rebuilt.
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    int size = 0;
    O3DB_CUDA_CHECK(cudaMemcpy(&size, &v->status->size, sizeof(int), cudaMemcpyDeviceToHost));
    VbgMap m;
    const int rc = fill_grown_map(v, m, new_capacity, size, st);
    if (rc == O3DB_OK) std::swap(v->map, m);
    m.free_on(st);   // the old map, or on failure the partial new one: v is then as it was
    return rc;
}

static int absorb_status(o3db_vbg* v, const VbgStatus& s) {
    v->known_size = s.size;
    v->max_new_seen = std::max<int64_t>(v->max_new_seen, s.max_new);
    if (s.overflow) {
        // Frames are atomic and ordered on the device: a frame whose new blocks did not fit (HashMap::Activate would
        // have grown the map, HashMap.cpp:166-181) and every frame after it were dropped whole — nothing integrated,
        // the table restored — so the volume is exactly the state before that frame.
        set_last_error("voxel block hash map capacity (%lld blocks) exceeded: fused frame #%d needed %d blocks; that frame "
                       "and all later ones were dropped (volume unchanged).  Call o3db_vbg_reserve with a larger capacity "
                       "and resubmit from that frame.",
                       (long long)v->map.capacity, s.dropped_frame - 1, s.dropped_need);
        return O3DB_ERR_CAPACITY;
    }
    return O3DB_OK;
}

// Copies the device status into h_status[0] and waits for it.
static int copy_status(o3db_vbg* v, cudaStream_t st) {
    O3DB_CUDA_CHECK(cudaMemcpyAsync(&v->h_status[0], v->status.get(), sizeof(VbgStatus), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    return O3DB_OK;
}

int read_status(o3db_vbg* v, cudaStream_t st) {
    if (int rc = copy_status(v, st)) return rc;
    return absorb_status(v, v->h_status[0]);
}

// The status fused frame f published into its ring entry, once the entry's seq says that frame wrote it.  The device
// writes the entry while the host reads it: every field is read from volatile memory, seq first.
static bool ring_status(const o3db_vbg* v, int64_t f, VbgStatus& s) {
    const volatile VbgStatus* e = &v->h_status[1 + (f & (kStatusRing - 1))];
    if (e->seq != (int)(f + 1)) return false;
    s.size = e->size;
    s.n_new = e->n_new;
    s.overflow = e->overflow;
    s.frame_count = e->frame_count;
    s.max_new = e->max_new;
    s.dropped_need = e->dropped_need;
    s.dropped_frame = e->dropped_frame;
    return true;
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

// Launches the integrate kernel of the input dtypes and value layout (VoxelBlockGridCUDA.cu:238-244).  u16 weight /
// u16 colour: the 16^3 fast path with its TMA-staged depth tile, or the generic-resolution kernel; f32 weight / f32
// colour: the generic kernel.  Fused frames take the persistent grid, block lists one CTA per work unit up to it.
template <typename depth_t, typename color_in_t, bool HAS_COLOR>
static int launch_integrate_typed(IntegrateArgs& a, int depth_dtype, bool f32_values, cudaStream_t st) {
    if (f32_values) {
        const unsigned grid = (unsigned)std::min<int64_t>(a.n_blocks, (int64_t)num_sms() * 8);
        O3DB_CUDA_CHECK(launch_pdl_ex(integrate_kernel<depth_t, color_in_t, HAS_COLOR, float, float>, {grid, kT}, st, a));
        return O3DB_OK;
    }
    const unsigned grid = a.status ? integrate_grid() : (unsigned)std::min<int64_t>((int64_t)a.n_blocks * 4, integrate_grid());
    if (a.resolution == 16 && a.rows <= 32767 && a.cols <= 65535) {
        CUtensorMap map;
        a.use_tile = make_depth_tensor_map(&map, a.depth, depth_dtype, a.rows, a.cols) ? 1 : 0;
        if (!a.use_tile) memset(&map, 0, sizeof(map));
        O3DB_CUDA_CHECK(launch_pdl_ex(integrate16_kernel<depth_t, color_in_t, HAS_COLOR>, {grid, kT}, st, a, map));
    } else {
        a.exec_ns = nullptr;   // o3db_vbg_exec_stats times integrate16_kernel only
        O3DB_CUDA_CHECK(launch_pdl_ex(integrate_kernel<depth_t, color_in_t, HAS_COLOR>, {grid, kT}, st, a));
    }
    return O3DB_OK;
}

// has_color: a.color is set.  Depth dtypes other than u16 / f32 were rejected by check_images.
static int launch_integrate(IntegrateArgs& a, int depth_dtype, int color_dtype, bool f32_values, cudaStream_t st) {
    const bool u16 = depth_dtype == O3DB_DEPTH_U16, has_color = a.color != nullptr;
    if (has_color && color_dtype != (u16 ? O3DB_COLOR_U8 : O3DB_COLOR_F32)) {
        if (f32_values) set_last_error("Unsupported input data type combination. Expected (float, float) or (uint16, uint8)");
        else if (u16) set_last_error("u16 depth requires u8 color (kernel/VoxelBlockGrid.cpp:107-146)");
        else set_last_error("f32 depth requires f32 color (kernel/VoxelBlockGrid.cpp:107-146)");
        return O3DB_ERR_INVALID;
    }
    if (u16)
        return has_color ? launch_integrate_typed<uint16_t, uint8_t, true>(a, depth_dtype, f32_values, st)
                         : launch_integrate_typed<uint16_t, uint8_t, false>(a, depth_dtype, f32_values, st);
    return has_color ? launch_integrate_typed<float, float, true>(a, depth_dtype, f32_values, st)
                     : launch_integrate_typed<float, float, false>(a, depth_dtype, f32_values, st);
}

// Arguments common to the handle and the stateless entry points.
static IntegrateArgs base_integrate_args(float voxel_size, int resolution, const void* depth, const void* color,
                                         int color_dtype, int rows, int cols, const double* dK, const double* cK,
                                         const double* E, float depth_scale, float depth_max, float trunc_mult) {
    IntegrateArgs a{};
    a.depth = depth;
    a.color = color;
    a.rows = rows;
    a.cols = cols;
    a.dcam = make_cam(dK, E, voxel_size);                           // VoxelBlockGridImpl.h:184
    const double eye[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    a.ccam = make_cam(cK ? cK : dK, eye, 1.0f);                     // :185-187
    a.sdf_trunc = voxel_size * trunc_mult;                          // VoxelBlockGrid.cpp:325
    a.depth_scale = depth_scale;
    a.depth_max = depth_max;
    a.color_multiplier = color_dtype == O3DB_COLOR_F32 ? 255.0f : 1.0f;   // VoxelBlockGridImpl.h:216-218
    a.resolution = resolution;
    a.fast_scale = fast_scale_ok(depth_scale) ? 1 : 0;
    a.inv_scale = 1.0f / depth_scale;
    // colour intrinsics identical to the depth intrinsics (what slam::Model passes) and sane: interior pixels map to
    // themselves (integrate16_kernel); anything else takes the reference's unproject / project per voxel
    a.same_k = (a.ccam.fx == a.dcam.fx && a.ccam.fy == a.dcam.fy && a.ccam.cx == a.dcam.cx && a.ccam.cy == a.dcam.cy &&
                a.dcam.fx > 1e-3f && a.dcam.fy > 1e-3f && std::isfinite(a.dcam.fx) && std::isfinite(a.dcam.fy) &&
                fabsf(a.dcam.cx) < 1e5f && fabsf(a.dcam.cy) < 1e5f && rows <= 16384 && cols <= 16384)
                       ? 1 : 0;
    return a;
}

static IntegrateArgs vbg_integrate_args(o3db_vbg* v, const void* depth, const void* color, int color_dtype, int rows,
                                        int cols, const double* dK, const double* cK, const double* E,
                                        float depth_scale, float depth_max, float trunc_mult) {
    IntegrateArgs a = base_integrate_args(v->voxel_size, v->resolution, depth, color, color_dtype, rows, cols, dK, cK,
                                          E, depth_scale, depth_max, trunc_mult);
    a.block_keys = v->map.keys.get();
    a.tsdf = v->map.tsdf.get();
    a.weight = v->map.weight.get();
    a.color_buf = v->map.color.get();
    a.capacity = (int)v->map.capacity;
    a.max_list = (int)v->frustum_cap;
    a.inv_w = v->inv_w;
    return a;
}

static int check_images(const void* depth, int depth_dtype, const void* color, int color_dtype, int rows, int cols) {
    O3DB_REQUIRE(depth != nullptr && rows > 0 && cols > 0, "depth image is empty");
    O3DB_REQUIRE(depth_dtype == O3DB_DEPTH_U16 || depth_dtype == O3DB_DEPTH_F32, "Unsupported depth image dtype");
    O3DB_REQUIRE(color == nullptr || color_dtype == O3DB_COLOR_U8 || color_dtype == O3DB_COLOR_F32,
                 "Unsupported color image dtype");
    return O3DB_OK;
}

// Geometry of a touch launch; the caller adds the table, the lists and the status record.
static TouchArgs make_touch_args(const void* depth, int rows, int cols, const double* K, const double* E,
                                 float block_size, float sdf_trunc, float depth_scale, float depth_max) {
    TouchArgs t{};
    double pose[16];
    inverse_transformation(E, pose);               // VoxelBlockGridCUDA.cu:119
    t.depth = depth;
    t.rows = rows;
    t.cols = cols;
    t.cam = make_cam(K, pose, 1.0f);               // :120
    t.block_size = block_size;                     // :143
    t.sdf_trunc = sdf_trunc;
    t.depth_scale = depth_scale;
    t.depth_max = depth_max;
    return t;
}

// Touch arguments on the handle's frame scratch.
static TouchArgs vbg_touch_args(o3db_vbg* v, const void* depth, int rows, int cols, const double* K, const double* E,
                                float depth_scale, float depth_max, float trunc_mult) {
    TouchArgs t = make_touch_args(depth, rows, cols, K, E, v->voxel_size * v->resolution,
                                  v->voxel_size * trunc_mult,   // VoxelBlockGrid.cpp:241
                                  depth_scale, depth_max);
    t.cand_keys = v->cand_keys.get();
    t.new_list = v->new_list.get();
    t.exist_list = v->exist_list.get();
    t.status = v->status.get();
    t.max_list = (int)v->frustum_cap;
    return t;
}

static int launch_touch(const TouchArgs& t, int depth_dtype, cudaStream_t st) {
    const int64_t nthreads = (int64_t)(t.rows / kStride) * (t.cols / kStride) * kSamples;
    const unsigned nb = (unsigned)std::max<int64_t>(1, ceil_div(nthreads, kT));
    O3DB_CUDA_CHECK(depth_dtype == O3DB_DEPTH_U16 ? launch_pdl_ex(touch_kernel<uint16_t>, {nb, kT}, st, t)
                                                  : launch_pdl_ex(touch_kernel<float>, {nb, kT}, st, t));
    return O3DB_OK;
}

// GetUniqueBlockCoordinates (VoxelBlockGrid.cpp:225-244) on t's frustum table, which only ever holds provisional
// entries: clears the table and the touch counters, runs the touch kernel and emits the keys it saw first.
static int unique_block_keys(const TouchArgs& t, int depth_dtype, int32_t* out, int64_t max_out, int64_t* num_host,
                             cudaStream_t st) {
    O3DB_CUDA_CHECK(cudaMemsetAsync(t.tab.table, 0xff, ((size_t)t.tab.mask + 1) * sizeof(int), st));   // frustum_hashmap_->Clear()
    O3DB_CUDA_CHECK(cudaMemsetAsync(&t.status->n_exist, 0, 2 * sizeof(int), st));                        // n_exist, n_new
    if (int rc = launch_touch(t, depth_dtype, st)) return rc;
    int n_new = 0;
    O3DB_CUDA_CHECK(cudaMemcpyAsync(&n_new, &t.status->n_new, sizeof(int), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    const int64_t n = n_new;
    if (num_host) *num_host = n;
    if (n == 0) {  // VoxelBlockGridCUDA.cu:193-198
        set_last_error("No block is touched in TSDF volume, abort integration. Please check specified parameters, "
                       "especially depth_scale and voxel_size");
        return O3DB_ERR_NO_BLOCKS;
    }
    if (out) {
        O3DB_REQUIRE(max_out >= n, "block_coords buffer too small: %lld < %lld", (long long)max_out, (long long)n);
        emit_unique_keys_kernel<<<(unsigned)ceil_div(n, kT), kT, 0, st>>>(t.new_list, t.status, t.cand_keys, out, (int)max_out);
        O3DB_LAUNCH_CHECK();
    }
    return O3DB_OK;
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
    std::unique_ptr<o3db_vbg, HandleDestroy<o3db_vbg_destroy>> v(new (std::nothrow) o3db_vbg());
    O3DB_REQUIRE(v != nullptr, "out of host memory");
    v->voxel_size = voxel_size;
    v->resolution = block_resolution;
    v->with_color = with_color != 0;
    if (int rc = alloc_map(v.get(), v->map, block_count, st)) return rc;
    if (int rc = dev_alloc(v->status, 1, st)) return rc;
    O3DB_CUDA_CHECK(cudaMemsetAsync(v->status.get(), 0, sizeof(VbgStatus), st));
    v->h_status = pinned_block<VbgStatus[]>(1 + kStatusRing);
    if (!v->h_status) {
        set_last_error("o3db_vbg_create: out of pinned host memory");
        return O3DB_ERR_CUDA;
    }
    memset(v->h_status.get(), 0, (1 + kStatusRing) * sizeof(VbgStatus));
    if (dev_alloc(v->exec_ns, 3) == O3DB_OK) {   // optional: without it o3db_vbg_exec_stats reports zeros
        const unsigned long long init[3] = {~0ull, 0ull, 0ull};
        cudaMemcpy(v->exec_ns.get(), init, sizeof(init), cudaMemcpyHostToDevice);
    }
    v->inv_w = inv_weight_table();
    if (!v->inv_w) {
        set_last_error("o3db_vbg_create: could not build the weight table: %s", cudaGetErrorString(cudaGetLastError()));
        return O3DB_ERR_CUDA;
    }
    *out = v.release();
    return O3DB_OK;
}

void o3db_vbg_destroy(o3db_vbg* v) {
    if (!v) return;
    cudaDeviceSynchronize();   // before the buffer owners free with cudaFree
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

int64_t o3db_vbg_capacity(const o3db_vbg* v) { return v ? v->map.capacity : 0; }

int o3db_vbg_reserve(o3db_vbg* v, int64_t capacity, void* stream) {
    O3DB_REQUIRE(v != nullptr, "o3db_vbg_reserve: null handle");
    cudaStream_t st = (cudaStream_t)stream;
    if (capacity > v->map.capacity)
        if (int rc = grow(v, capacity, st)) return rc;
    // a reserve acknowledges dropped frames (absorb_status): re-arm the device flag and forget the stale
    // read-backs, so that the caller can resubmit from the first dropped frame
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    VbgStatus* s = v->status.get();
    for (int* field : {&s->overflow, &s->dropped_need, &s->dropped_frame})
        O3DB_CUDA_CHECK(cudaMemsetAsync(field, 0, sizeof(int), st));
    for (int i = 0; i < 1 + kStatusRing; ++i) {
        VbgStatus& h = v->h_status[i];
        h.overflow = h.dropped_need = h.dropped_frame = 0;
    }
    v->sync_next_frame = true;
    return O3DB_OK;
}

int32_t* o3db_vbg_key_buffer(o3db_vbg* v) { return v ? v->map.keys.get() : nullptr; }
float* o3db_vbg_tsdf_buffer(o3db_vbg* v) { return v ? v->map.tsdf.get() : nullptr; }
uint16_t* o3db_vbg_weight_buffer(o3db_vbg* v) { return v ? v->map.weight.get() : nullptr; }
uint16_t* o3db_vbg_color_buffer(o3db_vbg* v) { return v ? v->map.color.get() : nullptr; }

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
    if (new_size > v->map.capacity) {
        rc = grow(v, std::max(new_size, 2 * v->map.capacity), st);
        if (rc) return rc;
    }
    DevPtr<int> scratch;
    rc = dev_alloc(scratch, (size_t)n, st);
    if (rc) return rc;
    MapArgs a{};
    a.tab = Table{v->map.table.get(), v->map.nbuckets - 1, v->map.keys.get()};
    a.keys_rw = v->map.keys.get();
    a.in_keys = keys_dev;
    a.n = (int)n;
    a.buf_indices = buf_indices_dev;
    a.masks = masks_dev;
    a.bucket_of_input = scratch.get();
    a.status = v->status.get();
    a.capacity = (int)v->map.capacity;
    const unsigned nb = (unsigned)ceil_div(n, kT);
    activate_claim_kernel<<<nb, kT, 0, st>>>(a);
    O3DB_LAUNCH_CHECK();
    activate_commit_kernel<<<nb, kT, 0, st>>>(a);
    O3DB_LAUNCH_CHECK();
    if (buf_indices_dev) {
        find_kernel<<<nb, kT, 0, st>>>(a, false);
        O3DB_LAUNCH_CHECK();
    }
    return O3DB_OK;
}

int o3db_vbg_find(o3db_vbg* v, const int32_t* keys_dev, int64_t n, int32_t* buf_indices_dev, uint8_t* masks_dev,
                  void* stream) {
    O3DB_REQUIRE(v != nullptr && n >= 0 && n < INT_MAX && (n == 0 || keys_dev), "o3db_vbg_find: bad arguments");
    if (n == 0) return O3DB_OK;
    MapArgs a{};
    a.tab = Table{v->map.table.get(), v->map.nbuckets - 1, v->map.keys.get()};
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
    TouchArgs t = vbg_touch_args(v, depth_dev, rows, cols, K, E, depth_scale, depth_max, trunc_mult);
    t.tab = Table{v->ftable.get(), v->fbuckets - 1, nullptr};
    rc = unique_block_keys(t, depth_dtype, block_coords_dev, max_blocks, num_blocks_host, st);
    // the touch counters are the fused frames' too, and the next frame expects them zero
    if (rc != O3DB_ERR_CUDA) O3DB_CUDA_CHECK(cudaMemsetAsync(&v->status->n_exist, 0, 2 * sizeof(int), st));
    return rc;
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
    DevPtr<int> buf;
    rc = dev_alloc(buf, (size_t)num_blocks, st);
    if (rc) return rc;
    // VoxelBlockGrid.cpp:313-315: Activate, then Find
    rc = o3db_vbg_activate(v, block_coords_dev, num_blocks, buf.get(), nullptr, st);
    if (rc) return rc;
    IntegrateArgs a = vbg_integrate_args(v, depth_dev, has_color ? color_dev : nullptr, color_dtype, rows, cols, dK, cK,
                                         E, depth_scale, depth_max, trunc_mult);
    a.buf_indices = buf.get();
    a.n_blocks = (int)num_blocks;
    return launch_integrate(a, depth_dtype, color_dtype, false, st);
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
    // scratch of one call: candidate keys, winners, a frustum-sized table (VoxelBlockGrid.cpp:225-234), counters
    const int64_t need = (int64_t)(rows / kStride) * (cols / kStride) * kSamples;
    const unsigned fbuckets = pow2_at_least(2 * need);
    DevPtr<int> cand, ftable;
    DevPtr<int2> winners;
    DevPtr<VbgStatus> status;
    rc = dev_alloc(cand, (size_t)need * 3, st);
    if (rc) return rc;
    rc = dev_alloc(winners, (size_t)need, st);
    if (rc) return rc;
    rc = dev_alloc(ftable, fbuckets, st);
    if (rc) return rc;
    rc = dev_alloc(status, 1, st);
    if (rc) return rc;
    TouchArgs t = make_touch_args(depth_dev, rows, cols, K, E, voxel_size * block_resolution, sdf_trunc, depth_scale,
                                  depth_max);
    t.cand_keys = cand.get();
    t.new_list = winners.get();
    t.status = status.get();
    t.max_list = (int)need;
    t.tab = Table{ftable.get(), fbuckets - 1, nullptr};
    return unique_block_keys(t, depth_dtype, block_coords_dev, max_blocks, num_blocks_host, st);
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
    const bool has_color = color_dev != nullptr && color_buf_dev != nullptr;     // VoxelBlockGridImpl.h:202-203
    const float* inv_w = inv_weight_table();
    O3DB_REQUIRE(inv_w != nullptr, "o3db_integrate_blocks: could not build the weight table");
    IntegrateArgs a = base_integrate_args(voxel_size, block_resolution, depth_dev, has_color ? color_dev : nullptr,
                                          color_dtype, rows, cols, dK, cK, E, depth_scale, depth_max, 1.0f);
    a.block_keys = block_keys_dev;
    a.tsdf = tsdf_dev;
    a.weight = (uint16_t*)weight_dev;
    a.color_buf = (uint16_t*)color_buf_dev;
    a.inv_w = inv_w;
    a.sdf_trunc = sdf_trunc;      // the reference passes the truncation itself (VoxelBlockGrid.h:369-381)
    a.capacity = INT_MAX;
    a.buf_indices = block_indices_dev;
    a.n_blocks = (int)num_blocks;
    return launch_integrate(a, depth_dtype, color_dtype, value_layout == O3DB_VALUES_F32, (cudaStream_t)stream);
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
        VbgStatus s{};
        const auto t0 = std::chrono::steady_clock::now();
        while (!ring_status(v, f, s)) {
            if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(20)) {
                const cudaError_t e = cudaStreamQuery(st);
                set_last_error("fused frame #%lld never reported its status (%s)", (long long)f,
                               e == cudaSuccess || e == cudaErrorNotReady ? "timeout" : cudaGetErrorString(e));
                return O3DB_ERR_CUDA;
            }
        }
        rc = absorb_status(v, s);
        if (rc) return rc;
    }
    const int64_t per_frame = std::max<int64_t>(2 * v->max_new_seen, 2048);
    if (v->known_size + 3 * per_frame > v->map.capacity) {
        rc = read_status(v, st);
        if (rc) return rc;
        if (v->known_size + 3 * per_frame > v->map.capacity) {
            rc = grow(v, std::max<int64_t>(2 * v->map.capacity, v->known_size + 6 * per_frame), st);
            if (rc) return rc;
        }
    }
    const bool has_color = color_dev != nullptr && v->with_color;
    const bool prof = v->prof_on && (size_t)(3 * v->prof_frames + 2) < v->prof_ev.size();
    if (prof) cudaEventRecord(v->prof_ev[3 * v->prof_frames], st);
    auto touch = [&]() -> int {
        v->frame_id += 1;
        TouchArgs t = vbg_touch_args(v, depth_dev, rows, cols, K, E, depth_scale, depth_max, trunc_mult);
        t.tab = Table{v->map.table.get(), v->map.nbuckets - 1, v->map.keys.get()};
        t.stamp = v->map.stamp.get();
        t.frame_id = v->frame_id;
        return launch_touch(t, depth_dtype, st);
    };
    rc = touch();
    if (rc) return rc;
    if (v->frames == 0 || v->sync_next_frame) {
        // Nothing is known yet about how many blocks a frame of this sequence adds (first frame, or the first one
        // after a reserve that followed a dropped frame): size the map from the touch kernel's own count before
        // integrating, as HashMap::Activate does (HashMap.cpp:166-181).  One host synchronisation, once.  The status
        // is not absorbed here: a frame whose touch overflowed goes on to the integrate kernel, which drops it and
        // releases the buckets it claimed.
        v->sync_next_frame = false;
        rc = copy_status(v, st);
        if (rc) return rc;
        const VbgStatus& s = v->h_status[0];
        const int64_t need = (int64_t)s.size + s.n_new;
        if (need > v->map.capacity && !s.overflow) {
            rc = grow(v, std::max<int64_t>(2 * v->map.capacity, need + std::max<int64_t>(need / 2, 2048)), st);
            if (rc) return rc;
            // the provisional entries lived in the old table: discover the frame again in the new one
            O3DB_CUDA_CHECK(cudaMemsetAsync(&v->status->n_exist, 0, 2 * sizeof(int), st));
            rc = touch();
            if (rc) return rc;
        }
    }
    if (prof) cudaEventRecord(v->prof_ev[3 * v->prof_frames + 1], st);
    IntegrateArgs a = vbg_integrate_args(v, depth_dev, has_color ? color_dev : nullptr, color_dtype, rows, cols, K, K, E,
                                         depth_scale, depth_max, trunc_mult);
    a.exist_list = v->exist_list.get();
    a.new_list = v->new_list.get();
    a.cand_keys = v->cand_keys.get();
    a.status = v->status.get();
    a.ring = &v->h_status[1];
    a.table = v->map.table.get();
    a.keys_rw = v->map.keys.get();
    a.stamp = v->map.stamp.get();
    a.frame_slots = v->frame_slots.get();
    a.frame_id = v->frame_id;
    a.frame_index = (int)v->frames;
    a.exec_ns = v->exec_ns.get();
    rc = launch_integrate(a, depth_dtype, color_dtype, false, st);
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
        v->d_depth[slot].reset();
        v->d_depth_bytes[slot] = 0;
        rc = dev_alloc(v->d_depth[slot], dbytes);
        if (rc) return rc;
        v->d_depth_bytes[slot] = dbytes;
    }
    if (cbytes > v->d_color_bytes[slot]) {
        O3DB_CUDA_CHECK(cudaStreamSynchronize(v->copy_stream));
        v->d_color[slot].reset();
        v->d_color_bytes[slot] = 0;
        rc = dev_alloc(v->d_color[slot], cbytes);
        if (rc) return rc;
        v->d_color_bytes[slot] = cbytes;
    }
    O3DB_CUDA_CHECK(cudaMemcpyAsync(v->d_depth[slot].get(), depth_host, dbytes, cudaMemcpyHostToDevice, v->copy_stream));
    if (cbytes) O3DB_CUDA_CHECK(cudaMemcpyAsync(v->d_color[slot].get(), color_host, cbytes, cudaMemcpyHostToDevice, v->copy_stream));
    O3DB_CUDA_CHECK(cudaEventRecord(v->copied[slot], v->copy_stream));
    O3DB_CUDA_CHECK(cudaStreamWaitEvent(st, v->copied[slot], 0));
    const int rc2 = o3db_vbg_integrate_frame(v, v->d_depth[slot].get(), depth_dtype, cbytes ? v->d_color[slot].get() : nullptr, color_dtype,
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
        O3DB_CUDA_CHECK(cudaMemcpy(h, v->exec_ns.get(), sizeof(h), cudaMemcpyDeviceToHost));
        if (reset) {
            const unsigned long long init[3] = {~0ull, 0ull, 0ull};
            O3DB_CUDA_CHECK(cudaMemcpy(v->exec_ns.get(), init, sizeof(init), cudaMemcpyHostToDevice));
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
    const int64_t n = v->h_status[0].frame_count;
    const int64_t m = std::min(n, max_blocks);
    if (m > 0 && block_coords_dev) {
        gather_keys_kernel<<<(unsigned)ceil_div(m, kT), kT, 0, st>>>(v->map.keys.get(), v->frame_slots.get(), (int)m, block_coords_dev);
        O3DB_LAUNCH_CHECK();
    }
    return n;
}

}  // extern "C"
