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
#include <memory>
#include <mutex>
#include <random>
#include <type_traits>

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

// The library's one process-global random engine, utility::random's RandomContext (utility/Random.cpp:15-50): seeded
// from std::random_device until o3db_random_seed replaces it with std::mt19937(seed).  Hold random_mutex() while
// drawing from it.
std::mt19937& random_engine();
std::mutex& random_mutex();

// Keep freed stream-ordered allocations cached in the device's default memory pool (the
// default release threshold of 0 hands everything back to the driver at every synchronise,
// which makes each create/destroy cycle re-map hundreds of MB).
void configure_memory_pool();

// Small pinned host blocks (result read-back) recycled through a process-wide free list:
// cudaMallocHost / cudaFreeHost cost ~1 ms each and would otherwise dominate short calls.
void* pinned_acquire(size_t bytes);     // bytes <= 4096
void pinned_release(void* p);

// ------------------------------------------------------------------------ owners of host-side allocations
// Every device buffer and pinned block the host code allocates has one of these owners, so that each path out of a
// call, error paths included, frees exactly what the call allocated.

// Frees in stream order on the stream the buffer was allocated on: the scratch of one call, and the buffers of the
// handles that keep their creation stream (o3db_icp, o3db_nns).
struct StreamFree {
    cudaStream_t stream = nullptr;
    StreamFree(cudaStream_t st = nullptr) : stream(st) {}
    void operator()(void* p) const { cudaFreeAsync(p, stream); }
};
// Frees with cudaFree, which synchronises the device: buffers an o3db_vbg keeps across calls.  Its entry points each
// take the caller's stream, so the buffer must not remember one; o3db_vbg_destroy synchronises the device before the
// owners go, and a buffer replaced during a call is handed to free_on instead.
struct DeviceFree {
    DeviceFree(cudaStream_t = nullptr) {}
    void operator()(void* p) const { cudaFree(p); }
};
template <typename T, typename D = StreamFree>
using DevPtr = std::unique_ptr<T, D>;

int alloc_failed(cudaError_t e, size_t bytes);   // clears the runtime's error, sets last_error, returns O3DB_ERR_CUDA

// Allocates count elements into p, stream-ordered on st (cudaMallocAsync), or without a stream through cudaMalloc.
// What p held before is released by its deleter; on failure p is unchanged and the runtime's last error is cleared, so
// that the next launch check does not report it against an unrelated kernel.
template <typename T, typename D>
int dev_alloc(DevPtr<T, D>& p, size_t count, cudaStream_t st) {
    void* q = nullptr;
    const cudaError_t e = cudaMallocAsync(&q, count * sizeof(T), st);
    if (e != cudaSuccess) return alloc_failed(e, count * sizeof(T));
    p = DevPtr<T, D>(static_cast<T*>(q), D(st));
    return O3DB_OK;
}
template <typename T>
int dev_alloc(DevPtr<T, DeviceFree>& p, size_t count) {
    void* q = nullptr;
    const cudaError_t e = cudaMalloc(&q, count * sizeof(T));
    if (e != cudaSuccess) return alloc_failed(e, count * sizeof(T));
    p = DevPtr<T, DeviceFree>(static_cast<T*>(q));
    return O3DB_OK;
}
// Releases a buffer held across calls in stream order on the current call's stream, without a device synchronise.
template <typename T>
void free_on(DevPtr<T, DeviceFree>& p, cudaStream_t st) {
    if (p) cudaFreeAsync(p.release(), st);
}

struct PinnedRelease {
    void operator()(void* p) const { pinned_release(p); }
};
template <typename T>
using PinnedPtr = std::unique_ptr<T, PinnedRelease>;
// A pinned block from the free list for one T, or for count elements when T is an array type; null when none could
// be allocated.
template <typename T>
PinnedPtr<T> pinned_block(size_t count = 1) {
    using E = std::remove_extent_t<T>;
    return PinnedPtr<T>(static_cast<E*>(pinned_acquire(count * sizeof(E))));
}

// Owner of a handle created through the C ABI: calls its destroy function.
template <auto Destroy>
struct HandleDestroy {
    template <typename H>
    void operator()(H* h) const { Destroy(h); }
};

// Cross-stream order of a handle that outlives its create call (o3db_knn, o3db_nns, o3db_icp).  Its buffers are
// allocated on the creation stream ("home"), and its destroy drains that stream and frees them on it.  A call may use
// the handle on another stream: it then records `ready` on home and waits on it, so that it runs after everything
// queued on home so far (the tail of create included), and afterwards records `used` on its own stream and makes home
// wait on that, so that home, and with it destroy's frees, come after every use.  The two events are created on the
// first such call; on the creation stream none of this is needed and nothing is done.  One call at a time per handle
// (the header's one-handle-per-host-thread rule): the events are shared by the handle's calls.
struct HandleEvents {
    mutable cudaEvent_t ready = nullptr;
    mutable cudaEvent_t used = nullptr;
    HandleEvents() = default;
    HandleEvents(const HandleEvents&) = delete;
    HandleEvents& operator=(const HandleEvents&) = delete;
    ~HandleEvents();
};
// Scope of one call on a handle: the wait on home when st is not home (check status()), and on every way out of the
// scope the `used` record that orders home after st.
class HandleUse {
  public:
    HandleUse(const HandleEvents& e, cudaStream_t home, cudaStream_t st);
    ~HandleUse();
    int status() const { return status_; }
    HandleUse(const HandleUse&) = delete;
    HandleUse& operator=(const HandleUse&) = delete;

  private:
    const HandleEvents& e_;
    cudaStream_t home_, st_;
    int status_ = O3DB_OK;
};

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
// programmatic-stream-serialization attribute.  Counts the launch, whether it succeeds or not.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_ex(void (*kernel)(KArgs...), const PdlLaunch& l, cudaStream_t st, Args&&... args) {
    count_launch();
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
