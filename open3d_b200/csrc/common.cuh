// common.cuh — shared helpers of the sm_90a kernels (error plumbing, launch
// accounting, warp primitives).  Product code; never includes anything from
// oracle/.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "../../include/open3d_b200.h"

namespace o3db {

void set_last_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launch_count;

inline void count_launch(uint64_t n = 1) { g_launch_count.fetch_add(n, std::memory_order_relaxed); }

#define O3DB_CUDA_CHECK(expr)                                                              \
    do {                                                                                   \
        cudaError_t e__ = (expr);                                                          \
        if (e__ != cudaSuccess) {                                                          \
            ::o3db::set_last_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), \
                                   __FILE__, __LINE__);                                    \
            return O3DB_ERR_CUDA;                                                          \
        }                                                                                  \
    } while (0)

#define O3DB_LAUNCH_CHECK()                                                                 \
    do {                                                                                    \
        ::o3db::count_launch();                                                             \
        cudaError_t e__ = cudaGetLastError();                                               \
        if (e__ != cudaSuccess) {                                                           \
            ::o3db::set_last_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(e__), \
                                   __FILE__, __LINE__);                                     \
            return O3DB_ERR_CUDA;                                                           \
        }                                                                                   \
    } while (0)

#define O3DB_REQUIRE(cond, ...)                 \
    do {                                        \
        if (!(cond)) {                          \
            ::o3db::set_last_error(__VA_ARGS__); \
            return O3DB_ERR_INVALID;            \
        }                                       \
    } while (0)

inline int num_sms() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return 132;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
            sms = 132;
    }
    return sms;
}

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Keep freed stream-ordered allocations cached in the device's default memory pool (the
// default release threshold of 0 hands everything back to the driver at every synchronise,
// which makes each create/destroy cycle re-map hundreds of MB).
void configure_memory_pool();

// Small pinned host blocks (result read-back) recycled through a process-wide free list:
// cudaMallocHost / cudaFreeHost cost ~1 ms each and would otherwise dominate short calls.
void* pinned_acquire(size_t bytes);     // bytes <= 4096
void pinned_release(void* p);

#ifdef __CUDACC__
// Programmatic dependent launch: a kernel launched through launch_pdl_ex may become resident while its predecessor
// on the stream drains; it must call pdl_wait() before touching anything the predecessor wrote.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Launch shape of launch_pdl_ex.  cluster > 0: thread-block clusters of `cluster` CTAs along x.
struct PdlLaunch {
    dim3 grid;
    unsigned block;
    size_t smem = 0;
    unsigned cluster = 0;
};

// Every kernel of the library that is ordered by griddepcontrol.wait is launched here, with the
// programmatic-stream-serialization attribute.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_ex(void (*kernel)(KArgs...), const PdlLaunch& l, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = l.grid;
    cfg.blockDim = dim3(l.block);
    cfg.dynamicSmemBytes = l.smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = l.cluster;
    attr[1].val.clusterDim.y = 1;
    attr[1].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = l.cluster > 0 ? 2 : 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// %globaltimer: nanoseconds, comparable across the SMs of a device.
__device__ __forceinline__ long long global_ns() {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// mbarrier (sm_90) helpers shared by the TMA pipelines of icp.cu and tsdf.cu.
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* b, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* b, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* b, unsigned parity) {
    unsigned done;
    do {
        asm volatile(
                "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                : "=r"(done)
                : "r"(smem_u32(b)), "r"(parity)
                : "memory");
    } while (!done);
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// Order-preserving float <-> uint mapping for atomicMin/atomicMax on floats.
__device__ __forceinline__ unsigned float_to_ordered(float f) {
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ordered_to_float(unsigned u) {
    u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}
#endif

}  // namespace o3db
