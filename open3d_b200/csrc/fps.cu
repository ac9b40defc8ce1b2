// fps.cu — farthest-point down-sampling on the device: PointCloud::FarthestPointDownSample (t/geometry/PointCloud.cpp:
// 612-648) in one persistent cooperative launch.  DESIGN.md §4.20.
//
// Upstream runs one round per sample on the host: five tensor kernels and a device-to-host read of the ArgMax.  Here
// one CTA per SM owns a contiguous slice of the cloud for the whole call.  The first kFpsOnChip points of a slice keep
// their positions in shared memory and their running minimum distances in registers; the rest of the slice (a cloud
// above the on-chip capacity) is read from and written back to global memory every round, by the same loop body.
// A round:
//   update   d[j] = min(d[j], |p_j - p_f|^2) for every point of the slice, the selected point f itself set to -1;
//   argmax   each thread's largest d in ascending index order (strict >, so the lowest index wins a tie), a warp and a
//            CTA maximum over 64-bit keys (d bits << 32 | 0xFFFFFFFF - index), one atomicMax into the round's slot;
//   barrier  one grid-wide synchronisation, after which every CTA reads the winner from the slot.
// Selected points carry d = -1, which no min ever raises and no argmax ever picks, so every index is selected at most
// once even where the cloud has fewer distinct positions than samples.
#include <cooperative_groups.h>

#include <climits>
#include <cmath>

#include "common.cuh"

namespace o3db {

namespace cg = cooperative_groups;

constexpr int kFpsThreads = 512;
constexpr int kFpsPerThread = 36;                                  // registers of running minima per thread
constexpr int kFpsOnChip = kFpsThreads * kFpsPerThread;            // points per CTA held on chip: 18432
constexpr size_t kFpsSmem = 3 * sizeof(float) * kFpsOnChip;        // their x, y and z: 221184 bytes

struct FpsArgs {
    const float* pts;            // [n,3]
    int64_t n;
    int64_t slice;               // points per CTA
    int num_samples;
    int start;
    float* rem_d;                // [grid][slice - kFpsOnChip]: running minima of the points past the on-chip part
    unsigned long long* slot;    // [num_samples], zero on entry: [0] non-finite flag, [r] round r's winning key
    int32_t* selected;           // [num_samples]
};

// upstream's f32 distance: diff = p - selected, (diff * diff).Sum({1}) in the order x, y, z, each op rounded, no FMA
__device__ __forceinline__ float fps_dist2(float x, float y, float z, float fx, float fy, float fz) {
    const float dx = __fsub_rn(x, fx), dy = __fsub_rn(y, fy), dz = __fsub_rn(z, fz);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ bool fps_finite(float x, float y, float z) {
    return isfinite(x) && isfinite(y) && isfinite(z);
}

__device__ __forceinline__ unsigned long long fps_warp_max(unsigned long long k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) k = max(k, __shfl_xor_sync(0xffffffffu, k, o));
    return k;
}

__global__ void __launch_bounds__(kFpsThreads, 1) fps_kernel(FpsArgs a) {
    extern __shared__ float fps_smem[];
    float* sx = fps_smem;
    float* sy = fps_smem + kFpsOnChip;
    float* sz = fps_smem + 2 * kFpsOnChip;
    __shared__ unsigned long long wkey[kFpsThreads / 32];
    cg::grid_group grid = cg::this_grid();
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int64_t lo = min(a.n, (int64_t)blockIdx.x * a.slice);
    const int64_t hi = min(a.n, lo + a.slice);
    const int on = (int)min(hi - lo, (int64_t)kFpsOnChip);
    const int rows = (on + kFpsThreads - 1) / kFpsThreads;
    const int64_t rem_lo = lo + on;
    float* rd = a.rem_d + (size_t)blockIdx.x * (size_t)max(a.slice - (int64_t)kFpsOnChip, (int64_t)0);

    // stage: positions to shared memory, d = +inf (-1 past the slice: never picked), non-finite coordinates flagged
    float d[kFpsPerThread];
    bool bad = false;
#pragma unroll
    for (int k = 0; k < kFpsPerThread; ++k) {
        const int l = t + k * kFpsThreads;
        float x = 0.f, y = 0.f, z = 0.f;
        if (l < on) {
            const float* p = a.pts + 3 * (lo + l);
            x = __ldg(p);
            y = __ldg(p + 1);
            z = __ldg(p + 2);
            bad |= !fps_finite(x, y, z);
        }
        sx[l] = x;
        sy[l] = y;
        sz[l] = z;
        d[k] = l < on ? INFINITY : -1.f;
    }
    for (int64_t j = rem_lo + t; j < hi; j += kFpsThreads) {
        const float* p = a.pts + 3 * j;
        bad |= !fps_finite(__ldg(p), __ldg(p + 1), __ldg(p + 2));
        rd[j - rem_lo] = INFINITY;
    }
    if (__syncthreads_or(bad) && t == 0) atomicOr(&a.slot[0], 1ull);
    grid.sync();
    if (__ldcg(&a.slot[0])) return;

    int f = a.start;
    if (blockIdx.x == 0 && t == 0) a.selected[0] = f;
    for (int r = 1; r < a.num_samples; ++r) {
        const float* pf = a.pts + 3 * (int64_t)f;
        const float fx = __ldg(pf), fy = __ldg(pf + 1), fz = __ldg(pf + 2);
        // f's row in this thread's registers: rel == k * kFpsThreads, or -1 when f is not on this CTA's chip part
        const int rel = (f >= lo && f < rem_lo) ? (int)(f - lo) - t : -1;
        float best = -1.f;
        int64_t bj = -1;
        int bl = -1;
#pragma unroll
        for (int k = 0; k < kFpsPerThread; ++k) {
            if (k < rows) {
                const int l = t + k * kFpsThreads;
                const float e = fps_dist2(sx[l], sy[l], sz[l], fx, fy, fz);
                d[k] = rel == k * kFpsThreads ? -1.f : fminf(d[k], e);
                if (d[k] > best) {
                    best = d[k];
                    bl = l;
                }
            }
        }
        if (bl >= 0) bj = lo + bl;
        for (int64_t j = rem_lo + t; j < hi; j += kFpsThreads) {
            const float* p = a.pts + 3 * j;
            const float e = fps_dist2(__ldg(p), __ldg(p + 1), __ldg(p + 2), fx, fy, fz);
            const float dj = j == f ? -1.f : fminf(rd[j - rem_lo], e);
            rd[j - rem_lo] = dj;
            if (dj > best) {
                best = dj;
                bj = j;
            }
        }
        // d >= +0 orders like its bits; 0 is no candidate (a real key's low word is at least 2^31)
        unsigned long long key =
                bj >= 0 ? ((unsigned long long)__float_as_uint(best) << 32) | (0xffffffffu - (unsigned)bj) : 0ull;
        key = fps_warp_max(key);
        if (lane == 0) wkey[warp] = key;
        __syncthreads();
        if (warp == 0) {
            key = fps_warp_max(lane < kFpsThreads / 32 ? wkey[lane] : 0ull);
            if (lane == 0 && key) atomicMax(&a.slot[r], key);
        }
        grid.sync();
        f = (int)(0xffffffffu - (unsigned)__ldcg(&a.slot[r]));
        if (blockIdx.x == 0 && t == 0) a.selected[r] = f;
    }
}

}  // namespace o3db

using namespace o3db;

extern "C" {

int o3db_farthest_point_down_sample(const float* positions_dev, int64_t n, int64_t num_samples, int64_t start_index,
                                    int32_t* selected_dev, void* stream) {
    O3DB_REQUIRE(positions_dev != nullptr && selected_dev != nullptr,
                 "o3db_farthest_point_down_sample: null positions or selected");
    O3DB_REQUIRE(n >= 0 && n < INT_MAX, "o3db_farthest_point_down_sample: bad point count (%lld)", (long long)n);
    O3DB_REQUIRE(num_samples >= 1 && num_samples <= n,
                 "FarthestPointDownSample: Illegal number of samples: %lld, must <= point size: %lld",
                 (long long)num_samples, (long long)n);
    O3DB_REQUIRE(start_index >= 0 && start_index < n,
                 "FarthestPointDownSample: Illegal start index: %lld, must < point size: %lld", (long long)start_index,
                 (long long)n);
    cudaStream_t st = (cudaStream_t)stream;
    configure_memory_pool();
    int dev = 0, sms = 0, coop = 0, per_sm = 0;
    O3DB_CUDA_CHECK(cudaGetDevice(&dev));
    O3DB_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    O3DB_CUDA_CHECK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    O3DB_CUDA_CHECK(cudaFuncSetAttribute(fps_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFpsSmem));
    O3DB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fps_kernel, kFpsThreads, kFpsSmem));
    if (!coop || per_sm < 1) {
        set_last_error("FarthestPointDownSample: the device cannot run fps_kernel cooperatively (%d CTAs per SM)",
                       per_sm);
        return O3DB_ERR_CUDA;
    }
    // every CTA gets at least a row of points: a small cloud pays for fewer CTAs at each barrier
    const int64_t grid = std::min<int64_t>((int64_t)per_sm * sms, ceil_div(n, kFpsThreads));
    const int64_t slice = ceil_div(n, grid);
    const int64_t rem = std::max<int64_t>(slice - kFpsOnChip, 0);
    DevPtr<unsigned long long> slot;
    DevPtr<float> rem_d;
    if (int rc = dev_alloc(slot, (size_t)num_samples, st)) return rc;
    if (rem > 0)
        if (int rc = dev_alloc(rem_d, (size_t)(grid * rem), st)) return rc;
    O3DB_CUDA_CHECK(cudaMemsetAsync(slot.get(), 0, (size_t)num_samples * sizeof(unsigned long long), st));
    FpsArgs args{positions_dev, n, slice, (int)num_samples, (int)start_index, rem_d.get(), slot.get(), selected_dev};
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(kFpsThreads);
    cfg.dynamicSmemBytes = kFpsSmem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    count_launch();
    O3DB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, fps_kernel, args));
    unsigned long long nonfinite = 0;
    O3DB_CUDA_CHECK(cudaMemcpyAsync(&nonfinite, slot.get(), sizeof(nonfinite), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    O3DB_REQUIRE(!nonfinite, "FarthestPointDownSample: the point cloud has non-finite coordinates");
    return O3DB_OK;
}

}  // extern "C"
