// common.cu — last-error storage, version, launch counter.
#include "common.cuh"

#include <mutex>
#include <vector>

namespace o3db {

static thread_local char g_last_error[1024] = "";
std::atomic<uint64_t> g_launch_count{0};

void set_last_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
    va_end(ap);
}

const char* last_error() { return g_last_error; }

std::mt19937& random_engine() {
    static std::mt19937 engine((int)std::random_device{}());   // upstream's Seed(rd()) takes an int
    return engine;
}

std::mutex& random_mutex() {
    static std::mutex mu;
    return mu;
}

int alloc_failed(cudaError_t e, size_t bytes) {
    (void)cudaGetLastError();
    set_last_error("device allocation of %zu bytes failed: %s", bytes, cudaGetErrorString(e));
    return O3DB_ERR_CUDA;
}

void configure_memory_pool() {
    static thread_local int configured_device = -1;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev == configured_device) return;
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
        unsigned long long keep = ~0ull;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    cudaGetLastError();
    configured_device = dev;
}

HandleEvents::~HandleEvents() {
    if (ready) cudaEventDestroy(ready);
    if (used) cudaEventDestroy(used);
}

static cudaError_t wait_for_home(const HandleEvents& e, cudaStream_t home, cudaStream_t st) {
    cudaError_t err = cudaSuccess;
    if (!e.ready && (err = cudaEventCreateWithFlags(&e.ready, cudaEventDisableTiming)) != cudaSuccess) return err;
    if (!e.used && (err = cudaEventCreateWithFlags(&e.used, cudaEventDisableTiming)) != cudaSuccess) return err;
    if ((err = cudaEventRecord(e.ready, home)) != cudaSuccess) return err;
    return cudaStreamWaitEvent(st, e.ready, 0);
}

HandleUse::HandleUse(const HandleEvents& e, cudaStream_t home, cudaStream_t st) : e_(e), home_(home), st_(st) {
    if (st_ == home_) return;
    const cudaError_t err = wait_for_home(e_, home_, st_);
    if (err != cudaSuccess) {
        (void)cudaGetLastError();
        set_last_error("ordering the call after the handle's creation stream failed: %s", cudaGetErrorString(err));
        status_ = O3DB_ERR_CUDA;
        st_ = home_;   // nothing was ordered after the wait, so there is nothing to order home after either
    }
}

HandleUse::~HandleUse() {
    if (st_ == home_) return;
    // (a handle's destroy ignores errors too: there is no caller left to report them to)
    if (cudaEventRecord(e_.used, st_) == cudaSuccess) cudaStreamWaitEvent(home_, e_.used, 0);
}

static std::mutex g_pinned_mu;
static std::vector<void*> g_pinned_free;

void* pinned_acquire(size_t bytes) {
    if (bytes > 4096) return nullptr;
    {
        std::lock_guard<std::mutex> lk(g_pinned_mu);
        if (!g_pinned_free.empty()) {
            void* p = g_pinned_free.back();
            g_pinned_free.pop_back();
            return p;
        }
    }
    void* p = nullptr;
    if (cudaMallocHost(&p, 4096) != cudaSuccess) return nullptr;
    return p;
}

void pinned_release(void* p) {
    if (!p) return;
    std::lock_guard<std::mutex> lk(g_pinned_mu);
    g_pinned_free.push_back(p);
}

}  // namespace o3db

extern "C" {
const char* o3db_last_error(void) { return o3db::last_error(); }
int o3db_version(void) { return O3DB_VERSION_MAJOR * 1000 + O3DB_VERSION_MINOR; }
uint64_t o3db_kernel_launch_count(void) { return o3db::g_launch_count.load(); }
}
